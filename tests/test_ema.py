"""Weight average (``ema_decay``, DESIGN.md rule E1) and ``opt.ema_weights()`` on both engines.

* the rule (a numpy replay) against ``torch._foreach_lerp_``, bit for bit, NaN and +-Inf included;
* ``psb_ema_kernel`` and ``psb_publish_kernel`` through the real bindings against the replay, bit for bit (CPU emulator of the
  same source, and the GPU with ``-m gpu``);
* the device engine on the emulator at 2-3 ranks: the average equals the replay over the engine's own weights, ``sharded``
  equals ``ps``, ``ema_weights()``, checkpoints and async;
* the host engine against torch SGD + ``AveragedModel(get_ema_multi_avg_fn(d))``, bit for bit."""
import copy

import numpy as np
import pytest
import torch
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200 import runtime
from pytorch_ps_mpi_b200.codings import TILE
from pytorch_ps_mpi_b200.launch import spawn
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout
from tests import _cuda_emu
from tests.test_adamw import F32, fma32, same_bits
from tests.test_multirank_engine_emulation import _attach, _data, _loss, _model, emu, run_ranks  # noqa: F401  (emu: fixture)

DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
GDT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
BCAST_LOCAL, BCAST_UNICAST, BCAST_MULTICAST = 0, 1, 2
DECAYS = [0.3, 0.7, 0.999, 0.9999]


# ---------------------------------------------------------------------------------------------------------------------
# the rule (DESIGN.md, rule E1) in numpy
# ---------------------------------------------------------------------------------------------------------------------
def weight(decay):
    return F32(1.0 - decay)                       # formed in double, rounded once


def e1(e, w, decay):
    """One average: ``e <- w`` at the first (``e is None``), else torch's ``lerp(e, w, a)`` in fp32."""
    w = np.asarray(w, F32)
    if e is None:
        return w.copy()
    a = weight(decay)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (w - e).astype(F32)
        if a < 0.5:
            return fma32(a, d, e)
        return fma32(F32(a - F32(1)), d, w)


def special(rng, n):
    x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 6, n)).astype(F32)
    x[rng.integers(0, n, 20)] = np.nan
    x[rng.integers(0, n, 20)] = np.inf
    x[rng.integers(0, n, 20)] = -np.inf
    return x


@pytest.mark.parametrize("decay", DECAYS)
def test_rule_against_torch(decay):
    rng = np.random.default_rng(int(decay * 1e4))
    n = 1 << 15
    e = None
    ref = None
    for t in range(5):
        w = special(rng, n) if t == 3 else (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(F32)
        e = e1(e, w, decay)
        if ref is None:
            ref = torch.from_numpy(w.copy())
        else:
            torch._foreach_lerp_([ref], [torch.from_numpy(w)], 1 - decay)
        assert np.array_equal(np.isnan(e), np.isnan(ref.numpy())), t
        assert same_bits(e, ref.numpy()), (decay, t)


# ---------------------------------------------------------------------------------------------------------------------
# the kernels through the real bindings
# ---------------------------------------------------------------------------------------------------------------------
BACKENDS = ["emu", pytest.param("gpu", marks=pytest.mark.gpu)]


def _ext(be):
    if be == "gpu":
        from pytorch_ps_mpi_b200.ops import ext
        return ext.cuda(), torch.device("cuda", 0)
    m = _cuda_emu.build_extension()
    if m is None:
        pytest.skip("no g++")
    return m, torch.device("cpu")


def _sync(be):
    if be == "gpu":
        torch.cuda.synchronize()


def _stem_layout():
    """A ResNet-stem-like [64,3,7,7] weight in its zero-padded [64,176] placement, between two plain parameters."""
    stem = torch.nn.Parameter(torch.zeros(64, 3, 7, 7))
    stem.ps_arena_layout = ((176, 1, 24, 3), 64 * 176)
    params = [torch.nn.Parameter(torch.zeros(3 * TILE + 77)), stem, torch.nn.Parameter(torch.zeros(9))]
    L = FlatLayout([{"params": params}], {id(p): f"p{i}" for i, p in enumerate(params)})
    real = torch.zeros(L.numel_padded, dtype=torch.bool)
    for s in L.slots:
        s.view(real[s.offset: s.offset + s.numel]).fill_(True)
    return L, real.numpy()


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("pname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("master", [True, False])
@pytest.mark.parametrize("decay,lo,hi", [(0.999, 0, None), (0.3, 2, None), (0.7, 1, 4)])
def test_ema_kernel_bits(be, pname, master, decay, lo, hi):
    """Copy, then three lerps, over tiles [lo, hi) with the compact state of a launch with state_shift = lo: from the fp32
    master or from the parameter arena widened exactly; NaN / Inf propagate; every padding lane (the stem's interior padding
    included) stays +0; tiles outside the range are untouched."""
    m, dev = _ext(be)
    dtype = GDT[pname]
    L, real = _stem_layout()
    nt, npad = L.ntiles, L.numel_padded
    hi = nt if hi is None else hi
    rng = np.random.default_rng(hash((pname, master, decay, lo)) % 2 ** 32)
    ns = (nt - lo) * TILE
    ema = torch.full((ns,), 7.0, dtype=torch.float32, device=dev)          # outside [lo, hi): a marker that must survive
    ema[(lo - lo) * TILE: (hi - lo) * TILE] = 0.0
    want = ema.cpu().numpy().copy()
    e = None
    for t in range(4):
        w = np.where(real, rng.standard_normal(npad) * 10.0 ** rng.uniform(-2, 2, npad), 0).astype(F32)
        if t == 2:
            w[5], w[TILE + 9], w[3 * TILE + 2] = np.nan, np.inf, -np.inf
        w = torch.from_numpy(w).to(dtype).float().numpy()                   # what the parameter dtype can hold
        arena = torch.from_numpy(w).to(dtype).to(dev).clone()
        mast = torch.from_numpy(w[lo * TILE:]).to(dev) if master else None
        m.ema(mast.data_ptr() if master else 0, 0 if master else arena.data_ptr(), DT[dtype], ema.data_ptr(), nt, lo, hi,
              lo, float(1.0 - decay), t == 0)
        _sync(be)
        e = e1(e, w, decay)
        want[: (hi - lo) * TILE] = e[lo * TILE: hi * TILE]
        got = ema.cpu().numpy()
        assert same_bits(got, want), (t, np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))[:5].tolist())
        pad = ~real[lo * TILE: hi * TILE]
        assert (got[: (hi - lo) * TILE][pad].view(np.uint32) == 0).all(), "padding must stay +0"


def _publish_case(be, pname, bcast, nranks):
    m, dev = _ext(be)
    dtype = GDT[pname]
    L, real = _stem_layout()
    nt, npad, lo = L.ntiles, L.numel_padded, 1
    rng = np.random.default_rng(11)
    live = np.where(real, rng.standard_normal(npad), 0).astype(F32)
    live[TILE + 3] = np.nan
    arenas = [torch.from_numpy(live).to(dtype).to(dev).clone() for _ in range(nranks)]
    bits0 = [a.cpu().view(torch.int16 if dtype != torch.float32 else torch.int32).clone() for a in arenas]
    ema = torch.from_numpy(np.where(real, rng.standard_normal(npad), 0).astype(F32)[lo * TILE:]).to(dev)
    saved = arenas[0][lo * TILE:].clone()
    mc = 0
    if bcast == BCAST_MULTICAST:                          # the emulator's multicast window over every rank's arena
        import ctypes
        m.emu.emu_mc_clear()
        window = torch.zeros(npad * arenas[0].element_size() + 64, dtype=torch.uint8)
        ptrs = (ctypes.c_void_p * nranks)(*[a.data_ptr() for a in arenas])
        assert m.emu.emu_mc_register(ctypes.c_void_p(window.data_ptr()), ctypes.c_size_t(window.numel() - 64), nranks, ptrs) >= 0
        mc = window.data_ptr()
    kw = dict(param_dst=[a.data_ptr() for a in arenas] if bcast == BCAST_UNICAST else [], param_mc=mc,
              param_local=arenas[0].data_ptr())
    m.publish(ema.data_ptr(), 0, lo, nt, lo, nt, DT[dtype], bcast, **kw)
    _sync(be)
    rounded = torch.from_numpy(ema.cpu().numpy()).to(dtype)
    targets = range(nranks) if bcast != BCAST_LOCAL else [0]
    for r in range(nranks):
        got = arenas[r].cpu()
        if r in targets:
            assert torch.equal(got[lo * TILE:].view(bits0[r].dtype), rounded.view(bits0[r].dtype)), (bcast, r)
        else:
            assert torch.equal(got.view(bits0[r].dtype), bits0[r])
        assert torch.equal(got[: lo * TILE].view(bits0[r].dtype), bits0[r][: lo * TILE])     # outside the range: untouched
    m.publish(saved.data_ptr(), DT[dtype], lo, nt, lo, nt, DT[dtype], bcast, **kw)        # the saved bits come back
    _sync(be)
    for r in range(nranks):
        assert torch.equal(arenas[r].cpu().view(bits0[r].dtype), bits0[r]), (bcast, r)     # NaN payload included
    if bcast == BCAST_MULTICAST:
        m.emu.emu_mc_clear()


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("pname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("bcast", [BCAST_LOCAL, BCAST_UNICAST])
def test_publish_kernel(be, pname, bcast):
    _publish_case(be, pname, bcast, 3)


@pytest.mark.parametrize("pname", ["fp32", "bf16"])
def test_publish_kernel_multicast_emulated(pname):
    _publish_case("emu", pname, BCAST_MULTICAST, 3)


def test_bindings_check_their_inputs():
    m, dev = _ext("emu")
    buf = torch.zeros(4 * TILE + 8, dtype=torch.float32)
    p, e = buf.data_ptr(), buf.data_ptr()
    ok = dict(master=p, param=0, param_dt=0, ema=e, ntiles=4, tile_begin=1, tile_end=3, state_shift=1, weight=0.001, first=True)
    m.ema(**ok)
    for bad, what in [(dict(tile_begin=3, tile_end=3), "tile range"), (dict(tile_end=5), "tile range"),
                      (dict(state_shift=2), "state_shift"), (dict(param_dt=3), "dtype"), (dict(ema=e + 4), "aligned"),
                      (dict(weight=0.0), "weight"), (dict(weight=1.0), "weight"), (dict(weight=float("nan")), "weight"),
                      (dict(master=0), "missing")]:
        with pytest.raises(RuntimeError, match=what):
            m.ema(**dict(ok, **bad))
    okp = dict(src=p, src_dt=0, src_shift=0, ntiles=4, tile_begin=0, tile_end=4, param_dt=1, bcast=BCAST_LOCAL, param_local=p)
    m.publish(**okp)
    for bad, what in [(dict(src_dt=2), "fp32 or the parameter dtype"), (dict(tile_begin=-1), "tile range"),
                      (dict(src_shift=1), "state_shift"), (dict(src=p + 8), "aligned"), (dict(bcast=BCAST_UNICAST), "unicast"),
                      (dict(bcast=BCAST_MULTICAST), "multicast"), (dict(bcast=7), "publication mode"),
                      (dict(param_local=0), "missing")]:
        with pytest.raises(RuntimeError, match=what):
            m.publish(**dict(okp, **bad))


# ---------------------------------------------------------------------------------------------------------------------
# the device engine on the emulator (real bindings)
# ---------------------------------------------------------------------------------------------------------------------
HYPER = dict(lr=0.05, momentum=0.9, weight_decay=1e-3)
DECAY = 0.7                                        # the lerp's second branch; the kernel tests cover both


def _weights(model):
    return [p.detach().clone() for p in model.parameters()]


def _ema_of(sd, n):
    return [sd["state"][i]["ema"].clone() for i in range(n)]


def _ema_everywhere(rank, w, opt, n):
    """Rank 0's average (``state_dict()`` is collective in ``sharded``; in ``ps`` only rank 0 holds the state)."""
    sd = copy.deepcopy(opt.state_dict())
    return w.broadcast_object(_ema_of(sd, n) if rank == 0 else None, src=0)


def _replay(history, decay=DECAY):
    e = None
    for ws in history:
        e = [torch.from_numpy(e1(None if e is None else e[i].numpy(), w.numpy(), decay)) for i, w in enumerate(ws)]
    return e


def _run(emu, n, mode, steps=3, pipeline=True, coding=None, body=None, decay=DECAY, **kw):
    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode=mode, pipeline=pipeline,
                     code=coding() if coding else None, ema_decay=decay, **kw, **HYPER)
        _attach(opt, reduce="p2p")
        if body is not None:
            return body(rank, w, model, opt)
        hist = []
        for s in range(steps):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=s == 1).backward()      # step 1: the head gets no gradient
            opt.step()
            hist.append(_weights(model))
        sd = copy.deepcopy(opt.state_dict())
        opt._engine.check()
        w.barrier()
        opt.close()
        return hist, sd

    return run_ranks(emu, n, rank_main)


CODINGS = {"identity": None, "sign": lambda: ps.Sign()}


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("coding", ["identity", "sign"])
@pytest.mark.parametrize("pipeline", [True, False])
@pytest.mark.parametrize("n,mode", [(2, "ps"), (3, "allgather")])
def test_engine_average_is_the_replay(emu, n, mode, pipeline, coding):
    """The average in ``state_dict()`` is the E1 replay over the weights the engine produced, bit for bit (a parameter without a
    gradient in step 1 included); ranks agree; ``sharded`` gives the same bits as ``ps``."""
    res = _run(emu, n, mode, pipeline=pipeline, coding=CODINGS[coding])
    hist, sd = res[0]
    for r in res[1:]:
        for a, b in zip(r[0][-1], hist[-1]):
            assert torch.equal(a, b)
    want = _replay(hist)
    got = _ema_of(sd, len(want))
    for g, x in zip(got, want):
        assert g.dtype == torch.float32 and torch.equal(g, x)
    if mode == "ps":
        sh = _run(emu, n, "sharded", pipeline=pipeline, coding=CODINGS[coding])
        for r in sh:
            for a, b in zip(_ema_of(r[1], len(want)), got):
                assert torch.equal(a, b)
            for a, b in zip(r[0][-1], hist[-1]):
                assert torch.equal(a, b)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_sgd_weights_match_torch_sgd(emu):
    """The weights themselves stay those of torch SGD on the summed gradient (within fp32 rounding): the average changes no
    update."""
    hist, _ = _run(emu, 2, "ps", decay=0.9)[0]
    model = _model()
    ref = torch.optim.SGD(model.parameters(), **HYPER)
    for s in range(3):
        tot = None
        for r in range(2):
            model.zero_grad(set_to_none=True)
            _loss(model, *_data(r, s), skip_head=s == 1).backward()
            gs = [None if p.grad is None else p.grad.clone() for p in model.parameters()]
            tot = gs if tot is None else [a if b is None else a + b for a, b in zip(tot, gs)]
        for p, g in zip(model.parameters(), tot):
            p.grad = g
        ref.step()
    for a, b in zip(hist[-1], model.parameters()):
        assert torch.allclose(a, b.detach(), rtol=2e-5, atol=2e-6)


def _ema_weights_body(steps_before, check):
    def body(rank, w, model, opt):
        for s in range(steps_before):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=False).backward()
            opt.step()
        out = check(rank, w, model, opt)
        opt._engine.check()
        w.barrier()
        opt.close()
        return out
    return body


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("n,mode", [(2, "ps"), (3, "sharded"), (2, "allgather")])
def test_ema_weights_swaps_and_restores(emu, n, mode):
    """Inside the block every rank's parameters are round(ema); after it they are bit-identical to before; a run that enters
    the block between steps ends bit-identical to one that never does."""
    def check(rank, w, model, opt):
        before = _weights(model)
        ema = _ema_everywhere(rank, w, opt, len(before))
        with opt.ema_weights():
            inside = _weights(model)
            with pytest.raises(RuntimeError, match="inside ema_weights"):
                opt.step()
        for a, b in zip(_weights(model), before):
            assert torch.equal(a, b)
        for i, (a, e) in enumerate(zip(inside, ema)):
            assert torch.equal(a, e.to(a.dtype)), (rank, i, float((a - e).abs().max()))
        for s in range(2, 4):                                  # training goes on
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=False).backward()
            opt.step()
        return _weights(model), _ema_everywhere(rank, w, opt, len(before))

    def straight(rank, w, model, opt):
        for s in range(2, 4):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=False).backward()
            opt.step()
        return _weights(model), _ema_everywhere(rank, w, opt, len(list(model.parameters())))

    got = _run(emu, n, mode, body=_ema_weights_body(2, check))
    want = _run(emu, n, mode, body=_ema_weights_body(2, straight))
    for r in range(n):
        for a, b in zip(got[r][0] + got[r][1], want[r][0] + want[r][1]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_ema_weights_refusals(emu):
    def check(rank, w, model, opt):
        with pytest.raises(RuntimeError, match="no average"):
            with opt.ema_weights():
                pass
        opt.zero_grad(set_to_none=True)
        _loss(model, *_data(rank, 0), skip_head=False).backward()
        with pytest.raises(RuntimeError, match="between backward"):
            with opt.ema_weights():
                pass
        opt.step()
        with opt.no_sync():
            _loss(model, *_data(rank, 1), skip_head=False).backward()
        with pytest.raises(RuntimeError, match="accumulation"):
            with opt.ema_weights():
                pass
        opt.step()
        with opt.ema_weights():
            with pytest.raises(RuntimeError, match="inside opt.ema_weights"):
                _loss(model, *_data(rank, 2), skip_head=False).backward()
        return True

    assert _run(emu, 2, "ps", body=_ema_weights_body(0, check)) == [True, True]


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("first,second", [("ps", "ps"), ("ps", "sharded"), ("sharded", "ps")])
def test_engine_checkpoint_resume(emu, first, second):
    """Two steps, ``state_dict()``, a fresh optimizer in the other mode loads it, two more steps: the same weights and average
    bits as four straight steps.  torch's SGD loads the dict."""
    def straight(rank, w, model, opt):
        for s in range(4):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=False).backward()
            opt.step()
        return _weights(model), _ema_everywhere(rank, w, opt, 6)

    def resumed(rank, w, model, opt):
        for s in range(2):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=False).backward()
            opt.step()
        sd = w.broadcast_object(copy.deepcopy(opt.state_dict()), src=0)
        assert all(sd["state"][i]["ema"].dtype == torch.float32 for i in range(6))
        msd = {k: v.clone() for k, v in model.state_dict().items()}
        opt.close()
        tm = _model()
        torch.optim.SGD(tm.parameters(), **HYPER).load_state_dict(copy.deepcopy(sd))     # the extra key is harmless there
        model2 = _model()
        model2.load_state_dict(msd)
        opt2 = ps.SGD(model2.named_parameters(), model2.parameters(), engine="host", mode=second, ema_decay=DECAY, **HYPER)
        _attach(opt2, reduce="p2p")
        opt2.load_state_dict(sd)
        for s in range(2, 4):
            opt2.zero_grad(set_to_none=True)
            _loss(model2, *_data(rank, s), skip_head=False).backward()
            opt2.step()
        out = _weights(model2), _ema_everywhere(rank, w, opt2, 6)
        opt2._engine.check()
        w.barrier()
        opt2.close()
        return out

    want = _run(emu, 2, "ps", body=_ema_weights_body(0, straight))
    got = _run(emu, 2, first, body=resumed)
    for r in range(2):
        for a, b in zip(got[r][0] + got[r][1], want[r][0] + want[r][1]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_checkpoint_without_average_restarts_it(emu):
    """A checkpoint without ``ema`` restarts the average: the next step copies.  One with ``ema`` on some parameters raises."""
    def body(rank, w, model, opt):
        opt.zero_grad(set_to_none=True)
        _loss(model, *_data(rank, 0), skip_head=False).backward()
        opt.step()
        sd = copy.deepcopy(opt.state_dict())
        for st in sd["state"].values():
            st.pop("ema", None)
        opt.load_state_dict(sd)
        opt.zero_grad(set_to_none=True)
        _loss(model, *_data(rank, 1), skip_head=False).backward()
        opt.step()
        got = _ema_of(copy.deepcopy(opt.state_dict()), 6)
        after = _weights(model)
        bad = copy.deepcopy(opt.state_dict())
        bad["state"][0].pop("ema")
        with pytest.raises(ValueError, match="some parameters only"):
            opt.load_state_dict(bad)
        opt._engine.check()
        w.barrier()
        opt.close()
        return got, after

    got, after = _run(emu, 1, "ps", body=body)[0]
    for a, b in zip(got, after):
        assert torch.equal(a, b)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_async_server_average(emu):
    """Async, one worker, quota 1: the server's average is the replay over its weights after each applied update; the final
    select, which finds no contributor, does not average."""
    def body(rank, w, model, opt):
        if rank == 0:
            hist = []
            for _ in range(3):
                opt.step()
                # read right after the server's step: correct only because the emulator runs every stream in program order
                # (each launch completes before the call returns).  On a GPU the update is still queued here: a GPU version
                # would have to synchronise with the comm stream (or harvest the iteration) before reading the weights.
                hist.append(_weights(model))
            opt.serve()
            sd = copy.deepcopy(opt.state_dict())
            with pytest.raises(RuntimeError, match="async"):
                with opt.ema_weights():
                    pass
            opt.close()
            return hist, sd
        for s in range(3):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(1, s), skip_head=False).backward()
            opt.step()
        opt.close()
        return None

    res = _run(emu, 2, "async", body=body, quota=1)
    hist, sd = res[0]
    for g, x in zip(_ema_of(sd, 6), _replay(hist)):
        assert torch.equal(g, x)


def _bf16_run(emu, n, mode, optim, body=None, steps=3):
    """bf16 parameters with fp32 masters: the average's source is the master.  Returns per rank (masters after every step,
    final state dict, final bf16 weights) — the masters and the state from rank 0's (collective in ``sharded``) state dicts."""
    cls, hyper = {"sgd": (ps.SGD, HYPER), "adamw": (ps.AdamW, dict(lr=1e-2, weight_decay=0.05))}[optim]

    def rank_main(rank, w):
        model = _model(torch.bfloat16)
        opt = cls(model.named_parameters(), model.parameters(), engine="host", mode=mode, ema_decay=DECAY, **hyper)
        _attach(opt, reduce="p2p")
        assert opt._engine.master is not None or not opt._engine.is_server
        masters = []
        for s in range(steps):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s, torch.bfloat16), skip_head=s == 1).backward()
            opt.step()
            sd = w.broadcast_object(copy.deepcopy(opt.state_dict()), src=0)
            masters.append([sd["state"][i]["master_param"].float().cpu() for i in range(6)])
        out = body(rank, w, model, opt) if body is not None else None
        sd = w.broadcast_object(copy.deepcopy(opt.state_dict()), src=0)
        opt._engine.check()
        w.barrier()
        weights = _weights(model)
        opt.close()
        return masters, sd, weights, out

    return run_ranks(emu, n, rank_main)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("optim", ["sgd", "adamw"])
def test_engine_bf16_average_is_the_replay_over_the_masters(emu, optim):
    """bf16 parameters: the average is the replay over the fp32 masters, bit for bit (a parameter without a gradient in step 1
    included), for SGD and AdamW; ``sharded`` gives the same bits as ``ps``; inside ``ema_weights()`` every rank's parameters
    are the average rounded once to bf16, and they are bit-identical to before after it."""
    def swap(rank, w, model, opt):
        sd = w.broadcast_object(copy.deepcopy(opt.state_dict()), src=0)
        before = _weights(model)
        with opt.ema_weights():
            inside = _weights(model)
        for a, b in zip(_weights(model), before):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        for a, i in zip(inside, range(6)):
            assert a.dtype == torch.bfloat16 and torch.equal(a.view(torch.int16), sd["state"][i]["ema"].to(a.dtype).view(torch.int16))
        return True

    res = _bf16_run(emu, 3, "ps", optim, body=swap)
    masters, sd, _, _ = res[0]
    assert all(r[3] for r in res)
    for g, x in zip(_ema_of(sd, 6), _replay(masters)):
        assert g.dtype == torch.float32 and torch.equal(g, x)
    for r in _bf16_run(emu, 3, "sharded", optim):
        for a, b in zip(_ema_of(r[1], 6), _ema_of(sd, 6)):
            assert torch.equal(a, b)
        for a, b in zip(r[2], res[0][2]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_ema_weights_refusal_is_collective(emu):
    """A rank that refuses makes every rank refuse, instead of leaving the others in a barrier: in ``ps`` a worker that loads
    its own dict (which carries no average) while rank 0 loads one that does."""
    def body(rank, w, model, opt):
        opt.zero_grad(set_to_none=True)
        _loss(model, *_data(rank, 0), skip_head=False).backward()
        opt.step()
        sd = copy.deepcopy(opt.state_dict())
        assert ("ema" in sd["state"].get(0, {})) == (rank == 0)
        opt.load_state_dict(sd)
        with pytest.raises(RuntimeError, match="rank 1: ema_weights.*no average"):
            with opt.ema_weights():
                pass
        opt.load_state_dict(w.broadcast_object(sd if rank == 0 else None, src=0))    # rank 0's dict everywhere: fine
        with opt.ema_weights():
            pass
        opt._engine.check()
        w.barrier()
        opt.close()
        return True

    assert _run(emu, 2, "ps", body=body) == [True, True]


def test_ema_decay_validation():
    runtime.init()
    model = _model()
    for bad in (0.0, 1.0, -0.5, 1.5, float("nan"), "0.9"):
        with pytest.raises(ValueError, match="ema_decay"):
            ps.SGD(model.named_parameters(), model.parameters(), lr=0.1, engine="host", ema_decay=bad)


# ---------------------------------------------------------------------------------------------------------------------
# the host engine against torch SGD + AveragedModel
# ---------------------------------------------------------------------------------------------------------------------
def _host_oracle(n, steps, decay):
    model = _model()
    avg = AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(decay), use_buffers=False)
    ref = torch.optim.SGD(model.parameters(), **HYPER)
    for s in range(steps):
        tot = None
        for r in range(n):
            model.zero_grad(set_to_none=True)
            _loss(model, *_data(r, s), skip_head=s == 1).backward()
            gs = [None if p.grad is None else p.grad.clone() for p in model.parameters()]
            tot = gs if tot is None else [a if b is None else a + b for a, b in zip(tot, gs)]
        for p, g in zip(model.parameters(), tot):
            p.grad = g
        ref.step()
        avg.update_parameters(model)
    return [p.detach().clone() for p in avg.module.parameters()]


def host_ranks(rank, size):
    w = runtime.init()
    want = _host_oracle(size, 3, DECAY)
    for mode in ("ps", "sharded", "allgather"):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode=mode, ema_decay=DECAY, **HYPER)
        for s in range(3):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s), skip_head=s == 1).backward()
            opt.step()
        before = _weights(model)
        sd = opt.state_dict()
        if rank == 0 or mode != "ps":
            for i, x in enumerate(want):
                assert torch.equal(sd["state"][i]["ema"], x), (mode, i)
        with opt.ema_weights():
            for p, x in zip(model.parameters(), want):
                assert torch.equal(p.detach(), x), mode
        for a, b in zip(_weights(model), before):
            assert torch.equal(a, b)
        opt.close()
    w.barrier()


@pytest.mark.parametrize("n", [2, 3])
def test_host_engine_matches_averaged_model(n):
    spawn(host_ranks, n, env={"PSB200_TRANSPORT": "shm"}, timeout=240)


def test_host_engine_one_rank_checkpoint_and_torch():
    runtime.init()
    model, tm = _model(), _model()
    opt = ps.SGD(model.named_parameters(), model.parameters(), lr=0.05, momentum=0.9, engine="host", ema_decay=0.999)
    ref = torch.optim.SGD(tm.parameters(), lr=0.05, momentum=0.9)
    avg = AveragedModel(tm, multi_avg_fn=get_ema_multi_avg_fn(0.999), use_buffers=False)
    for s in range(4):
        for mdl, o in ((model, opt), (tm, ref)):
            o.zero_grad(set_to_none=True)
            _loss(mdl, *_data(0, s), skip_head=False).backward()
            o.step()
        avg.update_parameters(tm)
        if s == 1:                                              # resume from a checkpoint mid-run
            sd = copy.deepcopy(opt.state_dict())
            opt.close()
            opt = ps.SGD(model.named_parameters(), model.parameters(), lr=0.05, momentum=0.9, engine="host", ema_decay=0.999)
            opt.load_state_dict(sd)
    for p, q in zip(model.parameters(), avg.module.parameters()):
        assert torch.equal(opt.state[p]["ema"], q.detach())
    opt.close()


# ---------------------------------------------------------------------------------------------------------------------
# the GPU: two engine ranks on one H100
# ---------------------------------------------------------------------------------------------------------------------
def gpu_ranks(rank, size, mode, dtype_name):
    w = runtime.init()
    dev = w.device
    dtype = GDT[dtype_name]
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.Tanh(), torch.nn.Linear(256, 32)).to(dev, dtype)
    opt = ps.SGD(model.named_parameters(), model.parameters(), lr=0.05, momentum=0.9, mode=mode, engine="device",
                 ema_decay=0.9)
    eng = opt._engine
    assert eng is not None
    holds = mode != "ps" or rank == 0                      # the ranks whose state_dict() carries the state
    hist = []
    for s in range(4):
        opt.zero_grad(set_to_none=True)
        g = torch.Generator().manual_seed(100 * rank + s)
        x = torch.randn(16, 64, generator=g).to(dev, dtype)
        model(x).float().square().mean().backward()
        opt.step()
        eng.ensure_params()
        torch.cuda.synchronize()
        # the source of the average: the fp32 master of the server(s), gathered through the state dict
        sd = opt.state_dict()                              # collective in mode='sharded'
        if holds:
            src = [sd["state"][i]["master_param"] if "master_param" in sd["state"][i] else p.detach().float()
                   for i, p in enumerate(model.parameters())]
            hist.append([t.detach().float().cpu().clone() for t in src])
        if s == 2:
            before = [p.detach().clone() for p in model.parameters()]
            with opt.ema_weights():
                inside = [p.detach().clone() for p in model.parameters()]
            after = [p.detach().clone() for p in model.parameters()]
            assert all(torch.equal(a.view(torch.int16 if a.dtype != torch.float32 else torch.int32),
                                   b.view(torch.int16 if b.dtype != torch.float32 else torch.int32)) for a, b in zip(before, after))
            ema = w.broadcast_object([sd["state"][i]["ema"].cpu() for i in range(len(inside))] if rank == 0 else None, src=0)
            assert all(torch.equal(a.cpu(), e.to(a.dtype).cpu()) for a, e in zip(inside, ema)), "inside: round(ema)"
    sd = opt.state_dict()
    if holds:
        got = [sd["state"][i]["ema"].cpu() for i in range(len(hist[0]))]
        want = _replay(hist, decay=0.9)
        assert all(torch.equal(a, b) for a, b in zip(got, want)), "average != replay"
    eng.check()
    opt.close()
    w.barrier()


ONE_GPU = {"PSB200_PG_BACKEND": "gloo", "CUDA_VISIBLE_DEVICES": "0", "PSB200_DEVICE_TIMEOUT": "20"}


def gpu_state_right_after_step(rank, size, mode):
    """``state_dict()`` and ``load_state_dict()`` called the moment ``step()`` returns, with no synchronisation, on a rank that
    waits only for its own comm stream (N = 1, ``allgather``, rank 0 of ``ps``) and ``pipeline=False``, so the step's last
    average covers the whole arena: the dict holds the finished average, and a loaded average is not overwritten by it."""
    w = runtime.init()
    dev = w.device
    torch.manual_seed(0)
    # 134 M parameters: a long last average (about 0.6 ms on an H100).  On the H100 the host path of state_dict() /
    # load_state_dict() still outlasts it, so this checks the contract without provoking the overlap it guards against.
    model = torch.nn.Sequential(*[torch.nn.Linear(8192, 8192) for _ in range(2)]).to(dev, torch.bfloat16)
    opt = ps.SGD(model.named_parameters(), model.parameters(), lr=1e-3, momentum=0.9, mode=mode, engine="device",
                 pipeline=False, ema_decay=0.9)
    holds = mode != "ps" or rank == 0
    x = torch.randn(16, 8192, generator=torch.Generator().manual_seed(rank)).to(dev, torch.bfloat16)

    def step():
        opt.zero_grad(set_to_none=True)
        model(x).float().square().mean().backward()
        opt.step()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    w.barrier()
    saved = copy.deepcopy(opt.state_dict())
    for _ in range(3):
        step()
        now = copy.deepcopy(opt.state_dict())                       # no synchronisation between the two
        torch.cuda.synchronize()
        if holds:
            later = opt.state_dict()
            for i in range(len(list(model.parameters()))):
                assert torch.equal(now["state"][i]["ema"].cpu(), later["state"][i]["ema"].cpu()), ("state_dict", i)
        w.barrier()
    step()
    opt.load_state_dict(saved)                                      # no synchronisation between the two
    torch.cuda.synchronize()
    if holds:
        got = opt.state_dict()
        for i in range(len(list(model.parameters()))):
            assert torch.equal(got["state"][i]["ema"].cpu(), saved["state"][i]["ema"].cpu()), ("load_state_dict", i)
    opt._engine.check()
    opt.close()
    w.barrier()


@pytest.mark.gpu
@pytest.mark.parametrize("n,mode", [(1, "ps"), (2, "ps"), (2, "allgather")])
def test_gpu_state_dict_right_after_step(n, mode):
    spawn(gpu_state_right_after_step, n, (mode,), env=ONE_GPU, timeout=300)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,dtype_name", [("ps", "bf16"), ("sharded", "bf16"), ("allgather", "fp32")])
def test_gpu_engine_two_ranks_one_gpu(mode, dtype_name):
    spawn(gpu_ranks, 2, (mode, dtype_name), env=dict(ONE_GPU, PSB200_CHUNK_BYTES="16384"), timeout=300)


@pytest.mark.gpu
def test_gpu_multi_gpu():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    for mode in ("ps", "sharded"):
        spawn(gpu_ranks, min(n, 8), (mode, "bf16"), env={"PSB200_DEVICE_TIMEOUT": "20"}, timeout=300)
