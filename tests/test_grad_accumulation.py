"""Gradient accumulation over micro-batches (``MPI_PS.no_sync()``).

* ``psb_accumulate_kernel`` through the real ``accumulate`` binding: the carry is the fp32 sum of 1-5 micro-batches in order,
  bit for bit, for fp32 / bf16 / fp16 gradients, partial tiles, a custom (stem-like) strided span, NaN and +-Inf, more than
  ``PSB_ENCODE_MAX`` gradients; padding lanes stay 0.
* ``psb_encode_kernel`` with a carry, for every (kind, wire) of the dispatch table: the wire bytes and scales are those of the
  plain encode of the fp32 sum (whose bits ``test_wire_edges`` / ``test_qsgd_blockwise`` check against ``codings.py``), and the
  carry is left zero, or holds the leftover for error-feedback top-k.
* The device engine at 2-3 emulated ranks through the real bindings: ps / allgather / async, SGD / Adam, pipeline on and off,
  Identity / Cast / Scale / TopK (with and without error feedback) / block-wise QSGD against the gathered-gradient oracle fed
  each rank's micro-batch sum; patterns A and B bit-identical; parameters that fire only inside no_sync(); the errors; recover().
* The package's ResNet: direct gradient placement on plain steps only, and the wire-arena alias of ``zero_grad(set_to_none=False)``.
* The host engine at two spawned ranks over shm.
* On the H100 (``-m gpu``): the kernel cases, and two engine ranks on one GPU training a ResNet with micro-batches.
* The ``ps_accumulate`` protocol model, and which deleted waits it reports.
"""
from __future__ import annotations

import contextlib

import numpy as np
import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200.codings import KIND_DENSE, KIND_TOPK, TILE, WIRE_F32
from pytorch_ps_mpi_b200.parallel import protocol_model as pm
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout
from tests import _cuda_emu
from tests.test_model_integration_emulation import world  # noqa: F401  (fixture)
from tests.test_multirank_engine_emulation import _attach, _data, _loss, _model, emu, run_ranks  # noqa: F401  (emu: fixture)

GDT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
BACKENDS = ["emu", pytest.param("gpu", marks=pytest.mark.gpu)]


@pytest.fixture(autouse=True)
def _single_threaded_torch():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernels, through the real bindings (CPU emulator or the H100)
# ---------------------------------------------------------------------------------------------------------------------
class Kernels:
    """One arena of parameters: the ``accumulate`` / ``encode`` bindings over it, on the emulator or on the GPU."""

    def __init__(self, be, shapes, stem=False):
        if be == "gpu":
            from pytorch_ps_mpi_b200.ops import ext
            self.x, self.dev = ext.cuda(), torch.device("cuda")
        else:
            self.x, self.dev = _cuda_emu.build_extension(), torch.device("cpu")
            if self.x is None:
                pytest.skip("no g++")
        self.params = [torch.nn.Parameter(torch.zeros(s)) for s in shapes]
        if stem:   # the ResNet stem's placement: [64,3,7,7] as a zero-padded [64,176] span
            p = torch.nn.Parameter(torch.zeros(64, 3, 7, 7))
            p.ps_arena_layout = ((176, 49, 7, 1), 64 * 176)
            self.params.append(p)
        self.L = FlatLayout([{"params": self.params}], {id(p): f"p{i}" for i, p in enumerate(self.params)})
        self.slots = self.L.slots
        self.tiles = self.L.tile_table_fast().to(self.dev)
        self.carry = torch.zeros(self.L.numel_padded, dtype=torch.float32, device=self.dev)

    def sync(self):
        if self.dev.type == "cuda":
            torch.cuda.synchronize()

    def spans(self, rng, gdt, specials=True):
        """One gradient per slot as the engine hands it to the kernels: the slot's span (padding of a custom placement zero)."""
        out = []
        for s in self.slots:
            v = rng.standard_normal(s.numel).astype(np.float32) * np.float32(rng.choice([1e-3, 1.0, 1e3]))
            if specials:
                idx = rng.choice(s.numel, size=min(6, s.numel), replace=False)
                v[idx] = np.array([np.nan, np.inf, -np.inf, -0.0, 3e38, -3e38], dtype=np.float32)[: len(idx)]
            t = torch.from_numpy(v).to(gdt)
            if s.strides is not None:
                span = torch.zeros(s.numel, dtype=gdt)
                s.view(span).copy_(s.view(t))
                t = span
            out.append(t.to(self.dev))
        return out

    def accumulate(self, grads):
        self.x.accumulate(grads, [s.first_tile for s in self.slots], [s.ntiles for s in self.slots],
                          [s.index for s in self.slots], self.tiles.data_ptr(), self.carry.data_ptr())
        self.sync()

    def arena(self, grads):
        """The gradients laid out as the fp32 arena (padding lanes 0)."""
        a = torch.zeros(self.L.numel_padded, dtype=torch.float32)
        for s, g in zip(self.slots, grads):
            a[s.offset: s.offset + s.numel] = g.cpu().float()
        return a

    def encode(self, code, grads, carry=None, keep_leftover=True):
        spec = code.device_spec()
        gdt = grads[0].dtype
        wire, bpt = spec.resolved_wire(gdt), spec.bytes_per_tile(gdt)
        wires = torch.zeros(self.L.ntiles * bpt, dtype=torch.uint8, device=self.dev)
        scales = torch.zeros(self.L.nparams, dtype=torch.float32, device=self.dev)
        amax = torch.zeros(self.L.nparams, dtype=torch.int32, device=self.dev)
        qsgd = dict(seed=spec.seed, step=3, rank=1, levels=spec.levels) if spec.levels else {}
        self.x.encode(spec.kind, wire, grads, [s.first_tile for s in self.slots], [s.ntiles for s in self.slots],
                      [s.index for s in self.slots], self.tiles.data_ptr(), wires.data_ptr(), scales.data_ptr(), amax.data_ptr(),
                      0 if carry is None else carry.data_ptr(), bpt, spec.tile_capacity(), float(spec.ratio), **qsgd,
                      **({} if keep_leftover else {"keep_leftover": False}))
        self.sync()
        return wires.cpu(), scales.cpu()


def _bits(t):
    return t.view(torch.int32)


def _np_sum(arenas):
    """fp32 sum in micro-batch order, the first add into a +0 carry."""
    c = np.zeros_like(arenas[0].numpy())
    for a in arenas:
        c = c + a.numpy()
    return torch.from_numpy(c)


def _same_floats(got, want):
    """Bit-equal, any NaN matching any NaN (a NaN's payload is not part of the contract)."""
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    assert torch.equal(_bits(got)[~nan], _bits(want)[~nan])


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("micro", [1, 2, 5])
def test_accumulate_is_the_fp32_sum_in_order(be, gname, micro):
    K = Kernels(be, [(3 * TILE + 5,), (700,), (TILE,)], stem=True)
    rng = np.random.default_rng(micro * 10 + len(gname))
    arenas = []
    for _ in range(micro):
        gs = K.spans(rng, GDT[gname])
        K.accumulate(gs)
        arenas.append(K.arena(gs))
    got = K.carry.cpu()
    _same_floats(got, _np_sum(arenas))
    pad = torch.ones(K.L.numel_padded, dtype=torch.bool)
    for s in K.slots:
        pad[s.offset: s.offset + s.numel] = False
        if s.strides is not None:   # the span's own padding (elements the [64,3,7,7] view does not cover)
            cover = torch.zeros(s.numel, dtype=torch.bool)
            s.view(cover).fill_(True)
            pad[s.offset: s.offset + s.numel] = ~cover
    assert not _bits(got)[pad].any(), "padding lanes must stay +0"


@pytest.mark.parametrize("be", BACKENDS)
def test_accumulate_batches_more_than_one_launch(be):
    """70 gradients: two launches of PSB_ENCODE_MAX (64) and 6."""
    K = Kernels(be, [(37 + 5 * i,) for i in range(70)])
    rng = np.random.default_rng(7)
    arenas = []
    for _ in range(3):
        gs = K.spans(rng, torch.float32, specials=False)
        K.accumulate(gs)
        arenas.append(K.arena(gs))
    _same_floats(K.carry.cpu(), _np_sum(arenas))


def test_accumulate_rejects_bad_arguments():
    K = Kernels("emu", [(100,)])
    g = torch.zeros(100)
    with pytest.raises(RuntimeError, match="carry"):
        K.x.accumulate([g], [0], [1], [0], K.tiles.data_ptr(), 0)
    with pytest.raises(RuntimeError, match="mixed gradient dtypes"):
        K.x.accumulate([g, g.bfloat16()], [0, 0], [1, 1], [0, 0], K.tiles.data_ptr(), K.carry.data_ptr())
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        K.x.accumulate([torch.zeros(101)[1:]], [0], [1], [0], K.tiles.data_ptr(), K.carry.data_ptr())


# every (kind, wire) pair of psb_launch_encode's dispatch table, with the gradient dtype that selects it
ENCODE_CASES = [
    ("identity_f32", ps.Identity, "fp32"), ("identity_bf16", ps.Identity, "bf16"), ("identity_f16", ps.Identity, "fp16"),
    ("cast_bf16", lambda: ps.Cast("bf16"), "fp32"), ("cast_fp16", lambda: ps.Cast("fp16"), "fp32"),
    ("cast_e4m3", lambda: ps.Cast("fp8_e4m3"), "fp32"), ("cast_e5m2", lambda: ps.Cast("fp8_e5m2"), "bf16"),
    ("scale_i8", lambda: ps.Scale("int8"), "fp32"), ("scale_i8_bf16", lambda: ps.Scale("int8"), "bf16"),
    ("scale_e4m3", lambda: ps.Scale("fp8_e4m3"), "fp32"), ("scale_e5m2", lambda: ps.Scale("fp8_e5m2"), "fp16"),
    ("scale_f16", lambda: ps.Scale("fp16"), "fp32"),
    ("topk_f32", lambda: ps.TopK(ratio=0.1), "fp32"), ("topk_ef_f32", lambda: ps.TopK(ratio=0.1, error_feedback=True), "fp32"),
    ("topk_bf16", lambda: ps.TopK(ratio=0.1), "bf16"), ("topk_ef_bf16", lambda: ps.TopK(ratio=0.1, error_feedback=True), "bf16"),
    ("qsgd_i4", lambda: ps.QSGD(7, seed=5, blockwise=True), "fp32"), ("qsgd_i8", lambda: ps.QSGD(127, seed=5, blockwise=True), "bf16"),
]


def _plain_reference(K, code, s32, gname):
    """The encode of the fp32 sum by the paths that predate accumulation: top-k as a zero gradient plus the sum as its
    error-feedback residual (wire, scales, leftover); any other coding as the plain encode (no carry) of the sum as an fp32
    gradient (wire, scales), unless the wire is the gradient's own 16-bit dtype (None: rule 2, checked by the caller)."""
    spec = code.device_spec()
    if spec.kind == KIND_TOPK:
        res = s32.clone().to(K.dev)
        w, sc = K.encode(code, [torch.zeros(s.numel, dtype=GDT[gname], device=K.dev) for s in K.slots], carry=res)
        return w, sc, res.cpu()
    if spec.resolved_wire(torch.float32) != spec.resolved_wire(GDT[gname]):
        return None
    w, sc = K.encode(code, [s32[s.offset: s.offset + s.numel].clone().to(K.dev) for s in K.slots])
    return w, sc, None


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("case", [c[0] for c in ENCODE_CASES])
def test_encode_with_carry_encodes_the_fp32_sum(be, case):
    _, factory, gname = next(c for c in ENCODE_CASES if c[0] == case)
    code = factory()
    spec = code.device_spec()
    K = Kernels(be, [(2 * TILE + 300,), (700,)], stem=True)
    rng = np.random.default_rng(len(case))
    specials = spec.kind != KIND_TOPK          # top-k keys of NaN / Inf are covered by the plain encode's tests
    firsts = [K.spans(rng, GDT[gname], specials) for _ in range(2)]
    for gs in firsts:
        K.accumulate(gs)
    last = K.spans(rng, GDT[gname], specials)
    s32 = _np_sum([K.arena(g) for g in firsts + [last]])
    keep = spec.kind == KIND_TOPK and spec.error_feedback
    wires, scales = K.encode(code, last, carry=K.carry, keep_leftover=keep)
    left = K.carry.cpu()
    ref = _plain_reference(K, code, s32, gname)
    if ref is not None:
        if spec.kind == KIND_DENSE and spec.resolved_wire(GDT[gname]) == WIRE_F32:
            _same_floats(wires.view(torch.float32), ref[0].view(torch.float32))   # an exact copy: any NaN is a NaN (rule 4)
        else:
            assert torch.equal(wires, ref[0]), "wire bytes differ from the plain encode of the fp32 sum"
        assert torch.equal(_bits(scales), _bits(ref[1]))
        if keep:
            _same_floats(left, ref[2])
    else:   # a dense wire of the gradient's own (16-bit) dtype: the fp32 sum rounded once, Inf on overflow (rule 2)
        want = s32.to(GDT[gname]).view(torch.int16)
        esz = 2
        for s in K.slots:
            got = wires[s.first_tile * TILE * esz: (s.first_tile * TILE + s.numel) * esz].view(torch.int16)
            nan = torch.isnan(s32[s.offset: s.offset + s.numel])
            assert torch.equal(got[~nan], want[s.offset: s.offset + s.numel][~nan])
    if not keep:
        assert not _bits(left).any(), "the carry must be left zero"


# ---------------------------------------------------------------------------------------------------------------------
# 2. the device engine on the emulator (real bindings, 2-3 rank threads)
# ---------------------------------------------------------------------------------------------------------------------
CODINGS = {"identity": ps.Identity, "cast": lambda: ps.Cast("bf16"), "scale": lambda: ps.Scale("int8"),
           "topk": lambda: ps.TopK(ratio=0.25), "topk_ef": lambda: ps.TopK(ratio=0.25, error_feedback=True),
           "qsgd": lambda: ps.QSGD(7, seed=3, blockwise=True)}
TOL = {"identity": (3e-5, 3e-6)}
MICRO = 3


def _slots(eng, model):
    return [eng.layout.by_id[id(p)] for p in model.parameters()]


def _micro_step(opt, model, rank, s, pattern, skip=lambda i: False):
    """One step of MICRO micro-batches; returns each parameter's fp32 micro-batch sum (None: no gradient in the step)."""
    opt.zero_grad(set_to_none=True)
    sums = [None] * len(list(model.parameters()))
    for i in range(MICRO):
        last = i == MICRO - 1
        with (opt.no_sync() if pattern == "B" or not last else contextlib.nullcontext()):
            probe = _model()
            with torch.no_grad():
                for q, p in zip(probe.parameters(), model.parameters()):
                    q.copy_(p)
            _loss(probe, *_data(rank, 10 * s + i), skip_head=skip(i)).backward()
            for j, q in enumerate(probe.parameters()):
                if q.grad is not None:
                    sums[j] = q.grad.clone() if sums[j] is None else sums[j] + q.grad
            _loss(model, *_data(rank, 10 * s + i), skip_head=skip(i)).backward()
    return sums


def _train_sync(emu, n, mode, optim, coding, pipeline, pattern, steps=3):
    hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-4) if optim == "sgd" else dict(lr=1e-2, eps=1e-8)

    def rank_main(rank, w):
        model = _model()
        shadow = [torch.nn.Parameter(p.detach().float().clone()) for p in model.parameters()]
        cls = ps.SGD if optim == "sgd" else ps.Adam
        oracle = cls([(f"p{i}", q) for i, q in enumerate(shadow)], shadow, engine="host", use_mpi=False, **hyper)
        for h in oracle._hooks:
            h.remove()
        groups = oracle._group_of()
        opt = cls(model.named_parameters(), model.parameters(), engine="host", mode=mode, code=CODINGS[coding](),
                  pipeline=pipeline, **hyper)
        _attach(opt)
        eng = opt._engine
        slots = _slots(eng, model)
        codes = [CODINGS[coding]() for _ in range(n)]          # the oracle's coding state of every rank (error feedback)
        for s in range(steps):
            sums = _micro_step(opt, model, rank, s, pattern)
            _, data = opt.step()
            assert data["micro_batches"] == MICRO
            allg = w.all_gather_object(sums)
            with torch.no_grad():
                for i, q in enumerate(shadow):
                    total = torch.zeros_like(q)
                    for r in range(n):
                        kw = dict(step=s, rank=r, first_tile=slots[i].first_tile) if coding == "qsgd" else dict(name=f"p{i}")
                        total += codes[r].decode(codes[r].encode(allg[r][i], **kw)).reshape(q.shape).float()
                    oracle.optim_step(q, total, **oracle._hyper(groups[id(q)]))
        eng.check()
        w.barrier()
        assert not eng.accumulating
        assert coding == "topk_ef" or not eng.carry.any()              # every encode consumed its carry
        got = [p.detach().clone() for p in model.parameters()]
        opt.close()
        oracle.close()
        return got, [q.detach().clone() for q in shadow]

    return run_ranks(emu, n, rank_main)


SYNC_CASES = [
    (2, "ps", "sgd", "identity", True), (3, "ps", "adam", "scale", True), (2, "ps", "sgd", "qsgd", False),
    (3, "allgather", "sgd", "cast", True), (2, "allgather", "adam", "topk_ef", False), (2, "ps", "sgd", "topk", True),
    (2, "allgather", "adam", "identity", False), (2, "ps", "adam", "topk_ef", True), (3, "allgather", "sgd", "qsgd", True),
]


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("n,mode,optim,coding,pipeline", SYNC_CASES)
def test_sync_modes_match_the_summed_gradient_oracle(emu, n, mode, optim, coding, pipeline):
    res = _train_sync(emu, n, mode, optim, coding, pipeline, "A")
    rtol, atol = TOL.get(coding, (2e-4, 2e-5))
    for got, want in res:
        for a, b in zip(got, res[0][0]):
            assert torch.equal(a, b)                                   # ranks bit-identical
        for a, b in zip(got, want):
            assert torch.allclose(a, b, rtol=rtol, atol=atol), (coding, float((a - b).abs().max()))


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("mode,coding,pipeline", [("ps", "identity", True), ("allgather", "scale", False), ("ps", "topk", True),
                                                  ("ps", "qsgd", False)])
def test_patterns_a_and_b_give_the_same_bits(emu, mode, coding, pipeline):
    a = _train_sync(emu, 2, mode, "sgd", coding, pipeline, "A", steps=2)
    b = _train_sync(emu, 2, mode, "sgd", coding, pipeline, "B", steps=2)
    for (ga, _), (gb, _) in zip(a, b):
        for x, y in zip(ga, gb):
            assert torch.equal(x, y)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_async_worker_accumulates_then_posts_once(emu):
    nsteps, n, lr = 3, 2, 0.05

    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="async", quota=1, lr=lr)
        _attach(opt)
        sums = []
        if rank == 0:
            with opt.no_sync():                                # a no-op on the dedicated server
                assert not opt._engine._no_sync
            assert opt.serve() == nsteps
        else:
            for s in range(nsteps):
                sums.append(_micro_step(opt, model, rank, s, "A"))
                _, data = opt.step()
                assert data["micro_batches"] == MICRO
        opt.close()
        return [p.detach().clone() for p in model.parameters()], sums

    res = run_ranks(emu, n, rank_main)
    want = [p.detach().clone() for p in _model().parameters()]
    for gs in res[1][1]:
        for i, g in enumerate(gs):
            want[i] -= lr * g
    for a, b in zip(res[0][0], want):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), float((a - b).abs().max())


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_parameters_firing_only_inside_no_sync_count_and_silent_ones_are_skipped(emu):
    """Step 0: the head gets a gradient in the first micro-batch only (inside no_sync) and is updated from the carry alone.
    Step 1: the head gets none at all and keeps its value (the reference's ``p.grad is None`` skip)."""
    lr, n = 0.1, 2

    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="ps", lr=lr)
        _attach(opt)
        head = list(model.parameters())[-2:]
        before = [p.detach().clone() for p in head]
        sums = _micro_step(opt, model, rank, 0, "A", skip=lambda i: i > 0)
        opt.step()
        after0 = [p.detach().clone() for p in head]
        allg = w.all_gather_object(sums[-2:])
        _micro_step(opt, model, rank, 1, "A", skip=lambda i: True)
        _, data = opt.step()
        after1 = [p.detach().clone() for p in head]
        opt._engine.check()
        opt.close()
        return before, after0, after1, allg

    for before, after0, after1, allg in run_ranks(emu, n, rank_main):
        for j in range(2):
            want = before[j] - lr * (allg[0][j] + allg[1][j])
            assert torch.allclose(after0[j], want, rtol=1e-6, atol=1e-7)
            assert torch.equal(after1[j], after0[j])


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_errors_and_recover(emu):
    """step() inside no_sync() and state_dict() with an open accumulation raise; a second final gradient points at no_sync();
    recover() drops the carry and the next accumulated step starts from zero."""
    lr, n = 0.1, 2

    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="ps", lr=lr)
        _attach(opt)
        eng = opt._engine
        with opt.no_sync():
            _loss(model, *_data(rank, 0), skip_head=False).backward()
            with pytest.raises(RuntimeError, match="no_sync"):
                opt.step()
        with pytest.raises(RuntimeError, match="accumulation"):
            opt.state_dict()
        assert eng.grad_out(next(model.parameters())) is None
        eng.recover()
        assert not eng.accumulating and not eng.carry.any()
        opt.state_dict()
        before = [p.detach().clone() for p in model.parameters()]
        sums = _micro_step(opt, model, rank, 1, "A")
        opt.step()
        eng.check()
        after = [p.detach().clone() for p in model.parameters()]
        allg = w.all_gather_object(sums)
        # a plain step: a parameter's second gradient before step() names no_sync()
        opt.zero_grad(set_to_none=True)
        _loss(model, *_data(rank, 5), skip_head=False).backward()
        with pytest.raises(RuntimeError, match="no_sync"):
            _loss(model, *_data(rank, 6), skip_head=False).backward()
        opt.close()
        return before, after, allg

    for before, after, allg in run_ranks(emu, n, rank_main):
        for j, (b, a) in enumerate(zip(before, after)):
            assert torch.allclose(a, b - lr * (allg[0][j] + allg[1][j]), rtol=1e-6, atol=1e-7)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the package's ResNet at two ranks (direct gradient placement, the wire-arena alias)
# ---------------------------------------------------------------------------------------------------------------------
def _resnet_run(extm, plan, n=2):
    """``plan``: per step ("plain" | "accum", set_to_none).  Returns per rank: direct_grads after each step, the wire tiles and
    each parameter's fp32 micro-batch sum (from an engine-less copy of the model) after every accumulated step, final params."""
    import threading

    from tests import test_multirank_engine_emulation as H
    from tests.test_model_integration_emulation import ModelM, _batch, _tiny_resnet
    cluster = H.Cluster(extm.emu, n)
    out, errs = [None] * n, []

    def main(rank):
        H._tls.world, H._tls.m = H.World(cluster, rank), ModelM(cluster, extm)
        try:
            model = _tiny_resnet()
            named = list(model.named_parameters())
            opt = ps.SGD(named, [p for _, p in named], lr=0.05, momentum=0.9, mode="ps", engine="device")
            eng = opt._engine
            model.attach(opt)
            direct, wires = [], []
            for s, (kind, set_to_none) in enumerate(plan):
                opt.zero_grad(set_to_none=set_to_none)
                if s == 1 and not set_to_none:   # the hazard is really there: gradients that still view the wire arena
                    assert any(p.grad is not None and 0 <= p.grad.data_ptr() - eng._wire_ptr < eng.wire_arena.numel()
                               for _, p in named)
                nmb = 1 if kind == "plain" else MICRO
                sums = {}
                for i in range(nmb):
                    x, y = _batch(rank, 10 * s + i)
                    if kind == "accum":
                        probe = _tiny_resnet()
                        with torch.no_grad():
                            for q, (_, p) in zip(probe.parameters(), named):
                                q.copy_(p)
                        torch.nn.functional.cross_entropy(probe(x).float(), y).backward()
                        for (name, _), q in zip(named, probe.parameters()):
                            sums[name] = sums.get(name, torch.zeros(q.shape)) + q.grad.float()
                    with (opt.no_sync() if i < nmb - 1 else contextlib.nullcontext()):
                        torch.nn.functional.cross_entropy(model(x).float(), y).backward()
                opt.step()
                eng.ensure_params()
                eng.check()
                direct.append(eng.direct_grads)
                if kind == "accum":
                    got = {}
                    for name, p in named:
                        sl = eng.layout.by_id[id(p)]
                        flat = eng.wire_arena[sl.first_tile * eng.bpt: sl.first_tile * eng.bpt + sl.numel * eng.psz]
                        got[name] = sl.view(flat.view(eng.dtype)).clone()
                    wires.append((got, sums))
            H._tls.world.barrier()
            out[rank] = dict(direct=direct, wires=wires, params=[p.detach().clone() for p in model.parameters()],
                             names=set(eng.direct_names))
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
        raise [e for e in errs if "another rank" not in str(e)][0] if any("another rank" not in str(e) for e in errs) else errs[0]
    return out


def test_resnet_direct_placement_on_plain_steps_only_and_no_wire_alias(world, monkeypatch):
    """A direct-placement step, then an accumulated one after ``zero_grad(set_to_none=False)`` (``param.grad`` still views the
    wire arena), then a plain one.  ``direct_grads`` grows on the plain steps only.  The accumulated step's wire tiles are the
    micro-batch sums rounded once to bf16, and bit-identical to a run with ``set_to_none=True``; so are the final parameters."""
    # one tile per chunk: a parameter's encode runs inside its own hook, BEFORE AccumulateGrad, which would then add into the tile
    monkeypatch.setenv("PSB200_CHUNK_BYTES", str(TILE * 2))
    hazard = _resnet_run(world, [("plain", True), ("accum", False), ("plain", True)])
    clean = _resnet_run(world, [("plain", True), ("accum", True), ("plain", True)])
    for r in range(2):
        d = hazard[r]["direct"]
        per_step = len(hazard[r]["names"])
        assert per_step > 0 and d == [per_step, per_step, 2 * per_step], d
        got, sums = hazard[r]["wires"][0]
        ref, _ = clean[r]["wires"][0]
        for name in got:
            assert torch.equal(got[name], ref[name]), name
            # the engine-less copy computes the same gradients up to the stem / GEMM reference math's rounding
            assert torch.allclose(got[name].float(), sums[name].to(torch.bfloat16).float(), rtol=3e-2, atol=1e-3), name
        for a, b in zip(hazard[r]["params"], clean[r]["params"]):
            assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the host engine, two spawned ranks over shm
# ---------------------------------------------------------------------------------------------------------------------
def host_two_ranks(rank, size):
    """One process of ``test_host_engine_two_ranks``: for each (mode, coding), patterns A and B over two steps of three
    micro-batches: the summed-gradient oracle holds, ``micro_batches`` is reported, and both patterns give the same bits."""
    from pytorch_ps_mpi_b200 import runtime
    w = runtime.init()
    assert (w.rank, w.size) == (rank, size)
    hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-4)
    for mode, coding in (("ps", "identity"), ("allgather", "topk_ef"), ("ps", "scale")):
        finals = {}
        for pattern in "AB":
            model = _model()
            shadow = [torch.nn.Parameter(p.detach().float().clone()) for p in model.parameters()]
            oracle = ps.SGD([(f"p{i}", q) for i, q in enumerate(shadow)], shadow, engine="host", use_mpi=False, **hyper)
            for h in oracle._hooks:
                h.remove()
            groups = oracle._group_of()
            opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode=mode, code=CODINGS[coding](), **hyper)
            codes = [CODINGS[coding]() for _ in range(size)]
            for s in range(2):
                sums = _micro_step(opt, model, rank, s, pattern)
                with pytest.raises(RuntimeError, match="no_sync"):
                    with opt.no_sync():
                        opt.step()
                with pytest.raises(RuntimeError, match="accumulation"):
                    opt.state_dict()
                _, data = opt.step()
                assert data["micro_batches"] == MICRO
                allg = w.all_gather_object(sums)
                with torch.no_grad():
                    for i, q in enumerate(shadow):
                        total = sum(codes[r].decode(codes[r].encode(allg[r][i], name=f"p{i}")).reshape(q.shape).float()
                                    for r in range(size))
                        oracle.optim_step(q, total, **oracle._hyper(groups[id(q)]))
            for p, q in zip(model.parameters(), shadow):
                assert torch.allclose(p.detach(), q.detach(), rtol=2e-4, atol=2e-5), (mode, coding, float((p - q).abs().max()))
            finals[pattern] = [p.detach().clone() for p in model.parameters()]
            opt.close()
            oracle.close()
        for a, b in zip(finals["A"], finals["B"]):
            assert torch.equal(a, b), (mode, coding)
    w.barrier()


def test_host_engine_two_ranks():
    from pytorch_ps_mpi_b200.launch import spawn
    spawn(host_two_ranks, 2, env={"PSB200_TRANSPORT": "shm"}, timeout=240)


# ---------------------------------------------------------------------------------------------------------------------
# 5. the device engine on one H100, two ranks, the package's ResNet
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("coding", ["identity", "scale"])
def test_two_engine_ranks_one_gpu_resnet(coding):
    from pytorch_ps_mpi_b200.launch import spawn
    from tests.test_gpu_engine import ONE_GPU
    spawn(gpu_resnet_two_ranks, 2, (coding,), env=ONE_GPU, timeout=300)


def gpu_resnet_two_ranks(rank, size, coding):
    """One process of ``test_two_engine_ranks_one_gpu_resnet``: a bf16 ResNet (one BasicBlock per stage) in ``mode='ps'``,
    three steps of three micro-batches each.  The oracle: each rank's micro-batch gradients from an engine-less copy of the
    model, summed in fp32, coded per rank, summed in rank order and fed to SGD on fp32 shadows.  The copy's stem and GEMMs round
    differently from the engine's fused kernels, so the check is on the size of the update, not on bits; an update built from
    any one micro-batch alone is far outside it.  Ranks end bit-identical."""
    from pytorch_ps_mpi_b200 import models, runtime
    w = runtime.init()
    dev = w.device
    lr = 0.1

    def build():
        torch.manual_seed(0)
        return models.ResNet(models.resnet.BasicBlock, [1, 1, 1, 1], num_classes=10).to(dev).to(
            memory_format=torch.channels_last).bfloat16()

    model = build()
    named = list(model.named_parameters())
    w0 = [p.detach().float().clone() for _, p in named]
    shadow = [x.clone() for x in w0]
    opt = ps.SGD(named, [p for _, p in named], lr=lr, mode="ps", engine="device", code=CODINGS[coding]())
    eng = opt._engine
    assert eng is not None
    for s in range(3):
        opt.zero_grad(set_to_none=True)
        sums = [torch.zeros_like(x) for x in w0]
        for i in range(MICRO):
            g = torch.Generator().manual_seed(100 * rank + 10 * s + i)
            x = torch.randn(8, 3, 64, 64, generator=g).to(dev).bfloat16().contiguous(memory_format=torch.channels_last)
            y = torch.randint(0, 10, (8,), generator=g).to(dev)
            probe = build()
            with torch.no_grad():
                for q, (_, p) in zip(probe.parameters(), named):
                    q.copy_(p)
            torch.nn.functional.cross_entropy(probe(x).float(), y).backward()
            for j, q in enumerate(probe.parameters()):
                sums[j] += q.grad.float()
            with (opt.no_sync() if i < MICRO - 1 else contextlib.nullcontext()):
                torch.nn.functional.cross_entropy(model(x).float(), y).backward()
        _, data = opt.step()
        assert data["micro_batches"] == MICRO
        allg = w.all_gather_object([t.cpu() for t in sums])
        code = CODINGS[coding]()
        for j in range(len(shadow)):
            tot = sum(code.decode(code.encode(allg[r][j])).reshape(w0[j].shape).float() for r in range(size))
            shadow[j] -= lr * tot.to(dev)
    eng.check()
    torch.cuda.synchronize()
    got = [(opt.state[p]["master_param"] if eng.is_server else p).detach().float() for _, p in named]
    pub = w.all_gather_object([p.detach().cpu() for _, p in named])
    if eng.is_server:
        num = sum(float(((a - s_) ** 2).sum()) for a, s_ in zip(got, shadow))
        den = sum(float(((s_ - x) ** 2).sum()) for s_, x in zip(shadow, w0))
        assert den > 0 and (num / den) ** 0.5 < 0.05, (num / den) ** 0.5
        for a, b in zip(pub[0], pub[1]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    opt.close()
    w.barrier()


# ---------------------------------------------------------------------------------------------------------------------
# 6. the opt-in ``ps_accumulate`` protocol model: each chunk's carry is a resource (compute-stream accumulates write it, the
#    final comm-stream encode reads and zeroes it)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,epochs", [(2, 3), (3, 2)])
def test_ps_accumulate_model_holds(n, epochs):
    res = pm.check("ps_accumulate", n, epochs)
    assert res.finals >= 1 and res.states > 10


def test_wire_alias_left_in_place_is_a_race():
    """Without the hook's drop of a ``param.grad`` that views the wire tile, AccumulateGrad adds the final gradient into the
    tile while the encode writes it and the server reads it."""
    with pytest.raises(pm.Violation) as ei:
        pm.check("ps_accumulate", 2, 2, drop="alias")
    assert ei.value.kind in {"race", "version"} and ei.value.trace


def test_prev_done_wait_is_implied_in_ps_mode():
    """Deleting the first accumulate's wait on the previous step's ``done`` is not a race in ``ps`` mode: a worker's compute
    stream waits for PARAMS_READY, which the server raises only after every rank's last encode (and so its carry zeroing)
    finished, and the server's compute stream waits for ``done`` itself.  (An async worker waits for neither, which is why the
    engine keeps the wait.)  The carry's version checks still run: a mis-ordered accumulate would read a non-zeroed carry."""
    res = pm.check("ps_accumulate", 2, 3, drop="prev_done")
    assert res.finals >= 1
