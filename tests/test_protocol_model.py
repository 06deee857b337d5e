"""Exhaustive interleaving check of the device engine's epoch-flag protocol (CPU only).

The reference has no race detection (SURVEY.md §5); here every mode's flag protocol is model-checked, and each
"mutant" (one wait deleted) must be caught — otherwise the checker would prove nothing.
"""
import pytest

from pytorch_ps_mpi_b200.parallel import protocol_model as pm


@pytest.mark.parametrize("mode,n,epochs,kw", [
    ("ps", 2, 3, {}),
    ("ps", 3, 2, {}),
    ("ps", 4, 1, {}),
    ("ps_unpipelined", 3, 2, {}),
    ("allgather", 2, 3, {}),
    ("allgather", 3, 2, {}),
    ("allgather_unpipelined", 3, 2, {}),
    # with >= 2 pipelined chunks the in-order comm streams already imply the CONSUMED wait (it is load-bearing for 1 chunk)
    ("allgather", 2, 2, {"drop": "consumed"}),
    ("async", 2, 3, {}),
    ("async", 3, 2, {"quota": 1}),
    ("async", 3, 2, {"quota": 2}),
    ("async", 2, 2, {"consistent": True}),
    ("async", 2, 3, {"consistent": True}),
    # the reader's BEGIN == VERSION pre-check is an optimisation, not a safety requirement
    ("async", 2, 2, {"consistent": True, "drop": "begin"}),
])
def test_protocol_holds(mode, n, epochs, kw):
    res = pm.check(mode, n, epochs, **kw)
    assert res.finals >= 1 and res.states > 10


@pytest.mark.parametrize("mode,n,epochs,kw,kinds", [
    # workers start the next forward without waiting for the broadcast
    ("ps", 2, 2, {"drop": "params_ready"}, {"race", "version"}),
    # the server sums before the workers' gradients are in their arenas
    ("ps", 2, 2, {"drop": "grad_ready"}, {"race", "version"}),
    # the last encode launch does not wait for backward to finish
    ("ps", 2, 1, {"drop": "bwd_event"}, {"race", "version"}),
    # pipelined: the server updates chunk A / chunk B before every rank's flag carries that chunk's progress value
    ("ps", 2, 2, {"drop": "grad_ready_a"}, {"race", "version"}),
    ("ps", 2, 2, {"drop": "progress_off_by_one"}, {"race", "version"}),
    # pipelined: chunk A is encoded and flagged before backward produced its gradients
    ("ps", 2, 1, {"drop": "mid_event"}, {"race", "version"}),
    ("ps_unpipelined", 2, 2, {"drop": "params_ready"}, {"race", "version"}),
    ("ps_unpipelined", 2, 2, {"drop": "grad_ready"}, {"race", "version"}),
    # a rank re-encodes while a peer still reads its previous wire tiles
    ("allgather_unpipelined", 2, 2, {"drop": "consumed"}, {"race", "version"}),
    ("allgather_unpipelined", 2, 2, {"drop": "grad_ready"}, {"race", "version"}),
    ("allgather", 2, 2, {"drop": "grad_ready"}, {"race", "version"}),
    ("allgather", 2, 2, {"drop": "grad_ready_a"}, {"race", "version"}),
    # async: re-encode before the server consumed the previous gradient
    ("async", 2, 2, {"drop": "ack"}, {"race", "version", "final", "ack"}),
    # async: DONE posted before the last gradient was consumed → the gradient is lost
    ("async", 2, 2, {"drop": "final_ack"}, {"final", "ack"}),
    # consistent reads: a sequence lock without its second check adopts torn copies
    ("async", 2, 2, {"consistent": True, "drop": "recheck"}, {"torn-snapshot", "version"}),
    ("async", 2, 2, {"consistent": True, "drop": "server_begin"}, {"torn-snapshot", "version"}),
])
def test_mutants_are_caught(mode, n, epochs, kw, kinds):
    with pytest.raises(pm.Violation) as ei:
        pm.check(mode, n, epochs, **kw)
    assert ei.value.kind in kinds, str(ei.value)
    assert ei.value.trace, "a violation carries the interleaving that reaches it"


def test_cli(capsys):
    assert pm.main(["--mode", "ps", "--ranks", "2", "--epochs", "2"]) == 0
    assert "ok:" in capsys.readouterr().out
    assert pm.main(["--mode", "ps", "--ranks", "2", "--epochs", "2", "--drop", "params_ready"]) == 1
    assert "VIOLATION" in capsys.readouterr().out


@pytest.mark.parametrize("mode,tiles", [("stem_pipeline", 6), ("stem_wgrad_pipeline", 6)])
def test_kernel_pipelines_hold(mode, tiles):
    """The mbarrier / named-barrier hand-offs inside the fused-stem kernels (double-buffered patch / A / gy / staging)."""
    res = pm.check(mode, 1, tiles)
    assert res.finals == 1


@pytest.mark.parametrize("mode,drop", [("stem_pipeline", "a_empty"), ("stem_pipeline", "store_wait"), ("stem_pipeline", "staging_bar"),
                                       ("stem_wgrad_pipeline", "empty"), ("stem_wgrad_pipeline", "g_full")])
def test_kernel_pipeline_mutants_are_caught(mode, drop):
    with pytest.raises(pm.Violation) as ei:
        pm.check(mode, 1, 5, drop=drop)
    assert ei.value.kind in {"race", "version"}, str(ei.value)
