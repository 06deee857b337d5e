"""``mode='sharded'``: the parameter server split over every rank.

Each rank gathers, updates and publishes its own contiguous share of every pipeline chunk, keeps optimizer state for those tiles
only, and adds 1 to every rank's PARAMS_READY when it is done; the next forward waits for ``epoch * N``.  The mode computes what
``mode='ps'`` computes, so most checks here are bit-for-bit comparisons of the two:

* the protocol model (``build_sharded``) and its mutants;
* N ranks of the real device engine over the real ``bindings.cpp`` and the emulated kernels (``tests/_cuda_emu.py``), against
  ``mode='ps'``, with the launch log showing which tiles each rank updated;
* checkpoints across the two modes, the compact state size, a stalled peer and ``recover()``;
* the host engine at 2 and 3 spawned CPU ranks;
* on the H100 (``-m gpu``): 2 and 3 ranks on one GPU, the gated ``BcastLinear``, and N >= 2 GPUs when present."""
import contextlib
import threading

import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200 import runtime
from pytorch_ps_mpi_b200.codings import TILE
from pytorch_ps_mpi_b200.launch import spawn
from pytorch_ps_mpi_b200.parallel import device_engine as de
from pytorch_ps_mpi_b200.parallel import protocol_model as pm
from tests import _cuda_emu
from tests import test_multirank_engine_emulation as H
from tests.test_device_engine_control_flow import FakeEvent, FakeStream

ONE_GPU = {"PSB200_PG_BACKEND": "gloo", "CUDA_VISIBLE_DEVICES": "0", "PSB200_DEVICE_TIMEOUT": "20"}


# ---------------------------------------------------------------------------------------------------------------------
# 1. protocol model
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 3])
def test_sharded_protocol_holds(n):
    pm.check("sharded", n, 2)


@pytest.mark.parametrize("drop", ["params_ready", "count_short", "grad_ready", "signal_server_only"])
def test_sharded_protocol_mutants_are_caught(drop):
    with pytest.raises(pm.Violation):
        pm.check("sharded", 3, 2, drop=drop)


@pytest.mark.parametrize("mode", ["ps", "allgather", "async", "ps_accumulate"])
def test_other_protocol_models_still_hold(mode):
    pm.check(mode, 2, 2)


def test_protocol_cli_sharded(capsys):
    assert pm.main(["--mode", "sharded", "--ranks", "3", "--epochs", "2"]) == 0
    assert "ok: mode=sharded" in capsys.readouterr().out


# ---------------------------------------------------------------------------------------------------------------------
# 2. N ranks of the device engine on the emulated kernels, through the real bindings
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def emu(monkeypatch):
    ext = _cuda_emu.build_extension()
    if ext is None:
        pytest.skip("no g++")
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    ext.emu.emu_set_sm_count(1)              # update grid = 3 CTAs: grid-stride loops over several tiles
    monkeypatch.setattr(H, "_EXT", ext)
    H._tls.world, H._tls.m = H.World(H.Cluster(ext.emu, 1), 0), None
    monkeypatch.setattr(runtime, "world", lambda: H._tls.world)
    monkeypatch.setattr(de.ext, "cuda", lambda: H._tls.m)
    monkeypatch.setattr(de, "SymmetricArena", H.SharedArena)
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    monkeypatch.setenv("PSB200_CHUNK_BYTES", str(TILE * 4))      # one parameter per chunk (fp32)
    yield ext.emu
    torch.set_num_threads(n)


_rng = threading.Lock()


def _model(dtype=torch.float32):
    """Six parameters of 6, 1, 4, 1, 1 and 1 tiles: chunks that split over the ranks and one-tile chunks that one rank serves."""
    with _rng:
        torch.manual_seed(0)
        return torch.nn.Sequential(torch.nn.Linear(40, 260), torch.nn.Tanh(), torch.nn.Linear(260, 24), torch.nn.Tanh(),
                                   torch.nn.Linear(24, 10)).to(dtype)


def _data(rank, step, dtype, micro=0, width=40):
    g = torch.Generator().manual_seed(1000 * rank + 10 * step + micro)
    return torch.randn(8, width, generator=g).to(dtype), torch.randint(0, 10, (8,), generator=g)


def _loss(model, x, y, skip_head):
    h = model[:-1](x)
    out = h[:, :10] if skip_head else model[-1](h)
    return torch.nn.functional.cross_entropy(out.float(), y)


CODINGS = {"identity": ps.Identity, "scale": lambda: ps.Scale("int8"), "topk": lambda: ps.TopK(ratio=0.25),
           "topk_ef": lambda: ps.TopK(ratio=0.25, error_feedback=True), "qsgd": lambda: ps.QSGD(7, blockwise=True)}
HYPER = {"sgd": dict(lr=0.05, momentum=0.9, weight_decay=1e-3, nesterov=True),
         "adam": dict(lr=1e-2, weight_decay=1e-2, amsgrad=True)}


def _train(lib, n, mode, *, optim="sgd", coding="identity", dtype=torch.float32, steps=4, pipeline=True, skip_until=0,
           micro=1, reduce="p2p", multicast=False, body=None, narrow=False):
    """``steps`` steps at ``n`` ranks; returns per rank: final parameters, the launch log, the engine's shard facts.
    ``narrow``: five one-tile parameters instead (every chunk has one server)."""
    width = 20 if narrow else 40

    def rank_main(rank, w):
        model = (H._model if narrow else _model)(dtype)
        cls = ps.SGD if optim == "sgd" else ps.Adam
        opt = cls(model.named_parameters(), model.parameters(), engine="host", mode=mode, code=CODINGS[coding](),
                  pipeline=pipeline, **HYPER[optim])
        H._attach(opt, reduce=reduce)
        eng = opt._engine
        if body is not None:
            return body(rank, w, model, opt, eng)
        for s in range(steps):
            opt.zero_grad(set_to_none=True)
            for i in range(micro):
                with opt.no_sync() if i < micro - 1 else contextlib.nullcontext():
                    _loss(model, *_data(rank, s, dtype, i, width), skip_head=s < skip_until).backward()
            _, data = opt.step()
            assert data["micro_batches"] == micro
        eng.check()
        w.barrier()
        out = dict(params=[p.detach().clone() for p in model.parameters()], log=list(H._tls.m.log),
                   sig=list(H._words(eng.arena.local_ptr)), nchunks=eng.nchunks, chunk_tiles=list(eng.chunk_tiles),
                   shards=getattr(eng, "shards", None), state_tiles=eng.state_tiles, reduce=eng.reduce,
                   buf0=None if eng.buf0 is None else eng.buf0.numel())
        opt.close()
        return out

    return H.run_ranks(lib, n, rank_main, multicast=multicast)


def _same(a, b, what):
    for ra, rb in zip(a, b):
        for x, y in zip(ra["params"], rb["params"]):
            assert torch.equal(x, y), (what, float((x.float() - y.float()).abs().max()))


def _check_shards(res, n, steps, pipeline=True, mode="sharded"):
    """Every rank updated exactly its plan ranges, with the plan's completion signal on the step's last launch, and keeps state
    for exactly those tiles.  ``mode='sharded'``: the ranges of each chunk cover it once and the counted PARAMS_READY == e * N;
    ``ps``: rank 0 serves whole chunks and PARAMS_READY == e; ``allgather``: every rank serves whole chunks and CONSUMED == e."""
    spans = res[0]["chunk_tiles"] if pipeline else [(0, res[0]["chunk_tiles"][-1][1])]
    for k, (lo, hi) in enumerate(spans):
        if mode == "sharded":
            got = sorted(tuple(r["shards"][k][q]) for q, r in enumerate(res))
            assert got[0][0] == lo and got[-1][1] == hi and all(a[1] == b[0] for a, b in zip(got, got[1:])), (k, got)
            sizes = [e - b for b, e in res[0]["shards"][k]]
            assert max(sizes) - min(sizes) <= 1
        else:
            servers = range(n) if mode == "allgather" else [0]
            assert [r["shards"][k][q] for q, r in enumerate(res)] == [(lo, hi) if q in servers else None for q in range(n)]
    done = de.SIGNAL_NONE if n == 1 else {"ps": de.SIGNAL_PARAMS_READY, "allgather": de.SIGNAL_CONSUMED,
                                          "sharded": H._EXT.SIGNAL_PARAMS_READY_ADD}[mode]
    for q, r in enumerate(res):
        ups = [(e[1], e[2], e[3]) for e in r["log"] if e[0] == "update"]
        mine = [(sh[q], k == len(spans) - 1) for k, sh in enumerate(r["shards"]) if sh[q] is not None and sh[q][1] > sh[q][0]]
        assert ups == [(b, e, done if last else de.SIGNAL_NONE) for (b, e), last in mine] * steps
        assert r["state_tiles"] == sum(e - b for (b, e), _ in mine)
        if n > 1 and mode == "allgather":
            assert list(r["sig"][H.M.SIG_CONSUMED: H.M.SIG_CONSUMED + n]) == [steps] * n
        elif n > 1:
            assert r["sig"][H.M.SIG_PARAMS_READY] == steps * (n if mode == "sharded" else 1)
        if r["shards"][-1][q] is not None and r["shards"][-1][q][1] == r["shards"][-1][q][0]:   # the counted signal alone
            assert sum(1 for e in r["log"] if e[0] == "signal" and e[1] == H.M.SIG_PARAMS_READY) == steps


CASES = {
    "identity_fp32_sgd": dict(),
    "identity_bf16_adam": dict(optim="adam", dtype=torch.bfloat16),
    "scale_sgd": dict(coding="scale"),
    "topk_adam": dict(optim="adam", coding="topk"),
    "topk_ef_sgd": dict(coding="topk_ef"),
    "qsgd_sgd": dict(coding="qsgd"),
    "inactive_late": dict(skip_until=2),
    "unpipelined": dict(pipeline=False),
    "no_sync_3": dict(micro=3, optim="adam"),
}


@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("case", sorted(CASES))
def test_sharded_p2p_equals_ps_p2p(emu, n, case):
    kw = CASES[case]
    want = _train(emu, n, "ps", **kw)
    got = _train(emu, n, "sharded", **kw)
    _same(got, want, case)
    _check_shards(got, n, 4, pipeline=kw.get("pipeline", True))
    _check_shards(want, n, 4, pipeline=kw.get("pipeline", True), mode="ps")
    for r in got:                                   # ranks bit-identical
        for a, b in zip(r["params"], got[0]["params"]):
            assert torch.equal(a, b)


def test_a_rank_with_an_empty_share_of_the_last_chunk(emu):
    """One tile per chunk: at 3 ranks each chunk has one server, the last chunk's two others add their 1 by the signal kernel."""
    got = _train(emu, 3, "sharded", optim="adam", narrow=True)
    _same(got, _train(emu, 3, "ps", optim="adam", narrow=True), "empty share")
    last = [tuple(r["shards"][-1][q]) for q, r in enumerate(got)]
    assert sum(1 for b, e in last if e == b) == 2
    _check_shards(got, 3, 4)


def test_compact_state_is_one_nth_of_the_arena(emu):
    """Per rank the optimizer state holds exactly its tiles; the ranks' tiles add up to the arena."""
    got = _train(emu, 3, "sharded", optim="adam", steps=1)
    # chunks (one parameter each) of 1, 1, 1, 4, 1, 6 tiles; the remainder of chunk k goes to ranks k % 3, k % 3 + 1, ...
    assert [e - b for b, e in got[0]["chunk_tiles"]] == [1, 1, 1, 4, 1, 6]
    assert [r["shards"] for r in got] == [got[0]["shards"]] * 3          # one static plan on every rank
    assert [[e - b for b, e in sh] for sh in got[0]["shards"]] == [[1, 0, 0], [0, 1, 0], [0, 0, 1], [2, 1, 1], [0, 1, 0], [2, 2, 2]]
    assert [r["state_tiles"] for r in got] == [5, 5, 4]                  # of 14 arena tiles
    for r in got:
        assert r["buf0"] == r["state_tiles"] * TILE


def _plan_facts(rank, w, model, opt, eng):
    out = dict(chunk_tiles=list(eng.chunk_tiles), shards=eng.shards, state_tiles=eng.state_tiles, ntiles=eng.layout.ntiles,
               buf0=None if eng.buf0 is None else eng.buf0.numel())
    opt.close()
    return out


@pytest.mark.parametrize("mode", ["ps", "allgather", "async"])
def test_serve_plan_and_state_size_in_the_other_modes(emu, mode):
    """The same serve plan outside mode='sharded': a serving rank gets whole spans and holds every tile's state, a worker gets
    ``None`` and holds none.  Read from the engines without training (an async engine trains differently)."""
    got = _train(emu, 3, mode, optim="adam", body=_plan_facts)
    servers = [0, 1, 2] if mode == "allgather" else [0]
    spans = got[0]["chunk_tiles"] if mode != "async" else [(0, got[0]["ntiles"])]      # async never pipelines
    for q, r in enumerate(got):
        assert r["shards"] == [[sp if p in servers else None for p in range(3)] for sp in spans]
        assert r["state_tiles"] == (r["ntiles"] if q in servers else 0)
        assert r["buf0"] == (r["state_tiles"] * TILE if q in servers else None)


@pytest.mark.parametrize("optim", ["sgd", "adam"])
def test_nvls_sharded_equals_ps_nvls(emu, optim):
    """The switch reduction on emulated multicast windows at 4 ranks: each server's multimem.ld_reduce covers its range only."""
    kw = dict(optim=optim, dtype=torch.bfloat16, reduce="auto", multicast=True)
    want = _train(emu, 4, "ps", **kw)
    got = _train(emu, 4, "sharded", **kw)
    assert got[0]["reduce"] == de.REDUCE_NVLS and want[0]["reduce"] == de.REDUCE_NVLS
    _same(got, want, "nvls")


# ---- checkpoints ------------------------------------------------------------------------------------------------------
def _only_step_counts(opt):
    """mode='sharded': after state_dict() / load_state_dict() no full-size state tensor stays behind in ``opt.state`` (the
    engine's compact buffers are the state; a full copy on every rank would undo the 1/N)."""
    assert opt.state and all(set(st) == {"step"} for st in opt.state.values()), [sorted(st) for st in opt.state.values()]


@pytest.mark.parametrize("first,second", [("ps", "sharded"), ("sharded", "ps")])
def test_checkpoint_across_modes(emu, first, second):
    """2 steps in ``first`` + state_dict + load into ``second`` + 2 steps == 4 straight steps, bit for bit (bf16 parameters with
    fp32 masters, Adam, a parameter that first fires late)."""
    import copy
    n = 3

    def body(mode_a, mode_b):
        def run(rank, w, model, opt, eng):
            for s in range(2):
                opt.zero_grad(set_to_none=True)
                _loss(model, *_data(rank, s, torch.bfloat16), skip_head=s < 1).backward()
                opt.step()
            sd = copy.deepcopy(opt.state_dict())            # collective in mode='sharded': every rank calls it
            if mode_a == "sharded":
                _only_step_counts(opt)
            sd = w.broadcast_object(sd, src=0)                # a checkpoint is written once (rank 0) and loaded everywhere
            msd = {k: v.clone() for k, v in model.state_dict().items()}
            opt.close()
            model2 = _model(torch.bfloat16)
            model2.load_state_dict(msd)
            opt2 = ps.Adam(model2.named_parameters(), model2.parameters(), engine="host", mode=mode_b, **HYPER["adam"])
            H._attach(opt2)
            opt2.load_state_dict(sd)
            if mode_b == "sharded":
                _only_step_counts(opt2)
            for s in range(2, 4):
                opt2.zero_grad(set_to_none=True)
                _loss(model2, *_data(rank, s, torch.bfloat16), skip_head=False).backward()
                opt2.step()
            opt2._engine.check()
            w.barrier()
            out = dict(params=[p.detach().clone() for p in model2.parameters()], keys=sorted(sd["state"][min(sd["state"])]))
            opt2.close()
            return out
        return run

    def straight(rank, w, model, opt, eng):
        for s in range(4):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s, torch.bfloat16), skip_head=s < 1).backward()
            opt.step()
        w.barrier()
        out = dict(params=[p.detach().clone() for p in model.parameters()])
        opt.close()
        return out

    want = _train(emu, n, "ps", optim="adam", dtype=torch.bfloat16, body=straight)
    got = _train(emu, n, first, optim="adam", dtype=torch.bfloat16, body=body(first, second))
    assert got[0]["keys"] == ["exp_avg", "exp_avg_sq", "master_param", "max_exp_avg_sq", "step"]
    _same(got, want, f"{first} -> {second}")


def test_stalled_peer_then_recover(emu, monkeypatch):
    """Rank 1 sits step 1 out: its peers' bounded waits time out, ``check()`` raises, ``recover()`` realigns the ranks and the
    count, and training continues to the same parameters on every rank."""
    monkeypatch.setenv("PSB200_DEVICE_TIMEOUT", "0.3")

    def run(rank, w, model, opt, eng):
        raised = None
        for s in range(4):
            if s == 1:
                if rank != 1:
                    opt.zero_grad(set_to_none=True)
                    _loss(model, *_data(rank, s, torch.float32), skip_head=False).backward()
                    opt.step()
                    try:
                        eng.check()
                        raised = False
                    except RuntimeError as exc:
                        raised = "timed out" in str(exc)
                w.barrier()
                eng.recover()
                assert H._words(eng.arena.local_ptr)[H.M.SIG_ERROR] == 0 and eng._epoch == 0
                continue
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s, torch.float32), skip_head=False).backward()
            opt.step()
        eng.check()
        w.barrier()
        out = dict(raised=raised, params=[p.detach().clone() for p in model.parameters()],
                   count=H._words(eng.arena.local_ptr)[H.M.SIG_PARAMS_READY])
        opt.close()
        return out

    res = _train(emu, 3, "sharded", body=run)
    assert res[0]["raised"] is True and res[2]["raised"] is True and res[1]["raised"] is None
    assert all(r["count"] == 2 * 3 for r in res)                     # two steps since recover(), three servers each
    for r in res:
        for a, b in zip(r["params"], res[0]["params"]):
            assert torch.equal(a, b)


# ---- direct gradient placement on the package's ResNet --------------------------------------------------------------
def _resnet(extm, n, steps):
    from tests.test_model_integration_emulation import ModelM, _batch, _tiny_resnet
    cluster = H.Cluster(extm.emu, n)
    out, errs = [None] * n, []

    def main(rank):
        H._tls.world, H._tls.m = H.World(cluster, rank), ModelM(cluster, extm)
        try:
            model = _tiny_resnet()
            named = list(model.named_parameters())
            opt = ps.SGD(named, [p for _, p in named], lr=0.05, momentum=0.9, weight_decay=1e-4, mode="sharded", engine="device")
            eng = opt._engine
            model.attach(opt)
            for s in range(steps):
                x, y = _batch(rank, s)
                opt.zero_grad(set_to_none=True)
                torch.nn.functional.cross_entropy(model(x).float(), y).backward()
                opt.step()
            eng.ensure_params()
            eng.check()
            H._tls.world.barrier()
            out[rank] = dict(params=[p.detach().clone() for p in model.parameters()], direct_n=eng.direct_grads,
                             gates=[e for e in H._tls.m.log if e[0] == "gate"])
            opt.close()
        except BaseException as exc:       # noqa: BLE001
            errs.append(exc)
            cluster.fail(exc)

    ts = [threading.Thread(target=main, args=(r,), daemon=True) for r in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in ts), "a rank thread is stuck"
    if errs:
        real = [e for e in errs if "another rank" not in str(e) and not isinstance(e, threading.BrokenBarrierError)]
        raise (real or errs)[0]
    return out


def test_resnet_direct_placement_equals_encode_path(emu, monkeypatch):
    """Two ranks, three steps of the tiny ResNet in mode='sharded' with the stem gate attached: producers we own write their
    gradients into the wire arena; with ``PSB200_DIRECT_GRAD=0`` the same gradients are encoded.  Bit for bit the same."""
    from pytorch_ps_mpi_b200.ops import ext as ops_ext
    monkeypatch.setattr(ops_ext, "cuda", lambda: H._tls.m)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setenv("PSB200_CHUNK_BYTES", str(2048 * 2 * 8))
    ext = _cuda_emu.build_extension()
    a = _resnet(ext, 2, 3)
    monkeypatch.setenv("PSB200_DIRECT_GRAD", "0")
    b = _resnet(ext, 2, 3)
    assert a[0]["direct_n"] > 0 and b[0]["direct_n"] == 0
    for ra, rb in zip(a, b):
        for x, y in zip(ra["params"], rb["params"]):
            assert torch.equal(x, y)
    for r in a:                                   # every rank (rank 0 too) acquired the counted flag through the stem gate
        assert [g[1] for g in r["gates"]] == [2, 4]


# ---------------------------------------------------------------------------------------------------------------------
# 3. host engine
# ---------------------------------------------------------------------------------------------------------------------
def host_ranks(rank, size):
    w = runtime.init()
    assert (w.rank, w.size) == (rank, size)
    finals = {}
    for mode in ("ps", "sharded"):
        for optim in ("sgd", "adam"):
            model = _model()
            cls = ps.SGD if optim == "sgd" else ps.Adam
            opt = cls(model.named_parameters(), model.parameters(), engine="host", mode=mode, **HYPER[optim])
            for s in range(3):
                opt.zero_grad(set_to_none=True)
                _loss(model, *_data(rank, s, torch.float32), skip_head=s < 1).backward()
                opt.step()
            sd = opt.state_dict()                      # collective in mode='sharded'; rank 0 holds everything in 'ps'
            if mode == "sharded":                      # only the parameters this rank serves keep state here
                assert {i for i, p in enumerate(model.parameters()) if p in opt.state} == \
                    {i for i in range(len(sd["state"])) if i % size == rank}
                opt.load_state_dict(sd)
                assert {i for i, p in enumerate(model.parameters()) if p in opt.state} == \
                    {i for i in range(len(sd["state"])) if i % size == rank}
            finals[mode, optim] = ([p.detach().clone() for p in model.parameters()],
                                   {i: {k: v.clone() if torch.is_tensor(v) else v for k, v in st.items()}
                                    for i, st in sd["state"].items()})
            opt.close()
    for optim in ("sgd", "adam"):
        for a, b in zip(finals["ps", optim][0], finals["sharded", optim][0]):
            assert torch.equal(a, b), optim
        if rank == 0:
            sp, ss = finals["ps", optim][1], finals["sharded", optim][1]
            assert sorted(sp) == sorted(ss)
            for i in sp:
                for k, v in sp[i].items():
                    assert torch.equal(v, ss[i][k]) if torch.is_tensor(v) else v == ss[i][k], (optim, i, k)
    with pytest.raises(ValueError, match="coalesce"):
        ps.SGD(_model().named_parameters(), lr=0.1, engine="host", mode="sharded", coalesce=True)
    w.barrier()


@pytest.mark.parametrize("n", [2, 3])
def test_host_engine_sharded_equals_ps(n):
    spawn(host_ranks, n, env={"PSB200_TRANSPORT": "shm"}, timeout=240)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the H100
# ---------------------------------------------------------------------------------------------------------------------
def gpu_ranks(rank, size, optim, dtype_name, pull=-1, gate=1):
    """Device engine, one process per rank: ``mode='ps'`` then ``mode='sharded'`` (reduce='p2p') from the same start; the
    parameters must agree bit for bit.  ``pull >= 0``: the first layer is the gated ``BcastLinear`` (``pull=1``: its weight
    tiles are read from rank 0's arena); with ``gate=1`` every rank, rank 0 included, acquires the counted PARAMS_READY in that
    GEMM instead of the wait kernel."""
    w = runtime.init()
    from pytorch_ps_mpi_b200.models import mnist_mlp
    from pytorch_ps_mpi_b200.ops.linear import convert_first_linear
    dev = w.device
    dtype = {"fp32": torch.float32, "bf16": torch.bfloat16}[dtype_name]
    hyper = HYPER[optim]
    finals = {}
    for mode in ("ps", "sharded"):
        torch.manual_seed(0)
        model = mnist_mlp(hidden=256).to(dev).to(dtype)
        cls = ps.SGD if optim == "sgd" else ps.Adam
        opt = cls(model.named_parameters(), model.parameters(), mode=mode, engine="device", reduce="p2p", **hyper)
        eng = opt._engine
        assert eng is not None and eng.sharded == (mode == "sharded")
        if pull >= 0:
            convert_first_linear(model, opt, relu=True, pull=bool(pull), gate=bool(gate))
        for s in range(5):
            g = torch.Generator().manual_seed(100 * rank + s)
            x = torch.randn(128, 784, generator=g).to(dev).to(dtype)
            y = torch.randint(0, 10, (128,), generator=g).to(dev)
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(model(x).float(), y).backward()
            opt.step()
        eng.ensure_params()
        eng.check()
        torch.cuda.synchronize()
        if mode == "sharded":
            assert int(eng.signal[eng.m.SIG_PARAMS_READY].item()) == 5 * size
            assert eng.state_tiles < eng.layout.ntiles
        finals[mode] = torch.cat([p.detach().float().reshape(-1) for p in model.parameters()]).cpu()
        opt.close()
    if pull < 0 or not gate:
        assert torch.equal(finals["ps"], finals["sharded"]), float((finals["ps"] - finals["sharded"]).abs().max())
    else:
        # The gated GEMM (the consumer acquires PARAMS_READY inside its TMA producer instead of the wait kernel) is not
        # run-to-run reproducible in EITHER mode: two mode='ps' runs of this very loop differ by up to 2 bf16 ulps in a few
        # hundred elements of fc1 / fc2, while the same GEMM ungated (gate=0, the case above) is bit-identical across runs and
        # across the two modes.  So the two modes can only be compared to that spread here (DESIGN.md §7).
        assert torch.allclose(finals["ps"], finals["sharded"], rtol=0, atol=2e-3), \
            float((finals["ps"] - finals["sharded"]).abs().max())
    allp = w.all_gather_object(finals["sharded"])
    for f in allp:
        assert torch.equal(f, allp[0]), "ranks diverged"
    if rank == 0:
        print("sharded ok", size, optim, dtype_name, pull, flush=True)


@pytest.mark.gpu
@pytest.mark.parametrize("n,optim,dtype", [(2, "sgd", "fp32"), (2, "adam", "bf16"), (3, "adam", "bf16"), (3, "sgd", "bf16")])
def test_sharded_equals_ps_one_gpu(n, optim, dtype):
    spawn(gpu_ranks, n, (optim, dtype), env=dict(ONE_GPU, PSB200_CHUNK_BYTES="65536"), timeout=300)


@pytest.mark.gpu
@pytest.mark.parametrize("pull,gate", [(0, 0), (0, 1), (1, 1)])
def test_sharded_bcast_linear_gate_one_gpu(pull, gate):
    spawn(gpu_ranks, 2, ("sgd", "bf16", pull, gate), env=ONE_GPU, timeout=300)


@pytest.mark.gpu
def test_sharded_multi_gpu():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    spawn(gpu_ranks, min(n, 8), ("adam", "bf16"), env={"PSB200_DEVICE_TIMEOUT": "20"}, timeout=300)
