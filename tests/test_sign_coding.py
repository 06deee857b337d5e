"""Block-wise scaled sign with error feedback (``ps.Sign``), bit for bit: the ``codings.py`` oracle, the encode and update kernels,
the error-feedback bookkeeping, the engines and a model with a custom arena placement.

The reference here is numpy, written from rules 13-16 of ``DESIGN.md`` (wire numerics): the real-element set of a tile, the
abs-max and the mean magnitude summed in the kernel's documented order, the NaN and FLT_MAX scales, the bit layout, the decode
and the residual.  Kernel cases go through the real bindings (``encode`` with ``real_mask=``, ``UpdatePlan.set_real_mask``): on
the CPU emulator of the same source by default, on the GPU with ``-m gpu``."""
import math

import numpy as np
import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200.codings import KIND_SIGN, TILE, WIRE_B1
from pytorch_ps_mpi_b200.ops.stem import STEM_K, STEM_STRIDES
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout
from tests import _cuda_emu
from tests.test_model_integration_emulation import ModelM, _batch, _tiny_resnet, world  # noqa: F401  (world: fixture)
from tests.test_multirank_engine_emulation import _attach, _data, _loss, _model, emu, run_ranks  # noqa: F401  (emu: fixture)

GDT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
F32 = np.float32
FMAX = F32(np.finfo(np.float32).max)
QNAN = np.array([0x7FFFFFFF], np.uint32).view(np.float32)[0]
BPT = TILE // 8 + 16
STEM = ((64, 3, 7, 7), (STEM_STRIDES, 64 * STEM_K))     # the ResNet stem weight in its zero-padded [64,176] placement


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def ref_real_span(shape, placement):
    """Real elements of a parameter's arena span: all of it, or the lanes of a custom strided placement."""
    n = math.prod(shape)
    if placement is None:
        return np.ones(n, bool)
    strides, span = placement
    idx = np.lib.stride_tricks.as_strided(np.arange(span), shape, [8 * s for s in strides])
    real = np.zeros(span, bool)
    real[idx.reshape(-1)] = True
    return real


def ref_tile(p, real):
    """(payload uint8[256], scale, decoded f32[2048], residual f32[2048]) of one tile ``p`` (f32) with real elements ``real``."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        if (~np.isfinite(p[real])).any():
            scale = QNAN
        else:
            m = np.abs(p[real]).max() if real.any() else F32(0)
            if m == 0:
                scale = F32(0)
            else:
                t = np.where(real, np.abs(p) / m, F32(0)).astype(F32).reshape(256, 8)
                s = np.zeros(256, F32)
                for j in range(8):                                   # per thread, index order, from +0
                    s = (s + t[:, j]).astype(F32)
                s = s.reshape(8, 32)
                for off in (16, 8, 4, 2, 1):                         # xor butterfly in every warp
                    s = (s + s[:, np.arange(32) ^ off]).astype(F32)
                tot = s[0, 0]
                for w in range(1, 8):                                # warps in index order
                    tot = F32(tot + s[w, 0])
                scale = F32(m * F32(tot / F32(real.sum())))
                if not scale <= FMAX:
                    scale = FMAX
        bits = np.signbit(p) & ~np.isnan(p) & real
        payload = (bits.reshape(256, 8).astype(np.uint32) << np.arange(8, dtype=np.uint32)).sum(axis=1).astype(np.uint8)
        dec = np.where(real, np.where(bits, -scale, scale), F32(0)).astype(F32)
        res = np.where(real, p - dec, F32(0)).astype(F32)
    return payload, scale, dec, res


def ref_span(p, real):
    """Wire rows [ntiles, 272], decoded and residual (f32, tile-padded) of one parameter span ``p`` (f32, any length)."""
    nt = max(1, -(-len(p) // TILE))
    pp = np.zeros(nt * TILE, F32)
    pp[:len(p)] = p
    rr = np.zeros(nt * TILE, bool)
    rr[:len(real)] = real
    rows, decs, ress = [], [], []
    for t in range(nt):
        sl = slice(t * TILE, (t + 1) * TILE)
        pay, scale, dec, res = ref_tile(pp[sl], rr[sl])
        head = np.zeros(4, F32)
        head[0] = scale
        rows.append(np.concatenate([pay, head.view(np.uint8)]))
        decs.append(dec)
        ress.append(res)
    return np.stack(rows), np.concatenate(decs), np.concatenate(ress)


def same_bits(a, b):
    return np.array_equal(np.asarray(a, F32).view(np.uint32), np.asarray(b, F32).view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _dtype_values(x, gname):
    """float32 values of ``x`` rounded to the gradient dtype (NaN, +-Inf and -0 kept)."""
    with np.errstate(over="ignore"):
        return torch.from_numpy(np.asarray(x, np.float64)).to(GDT[gname]).float().numpy()


def edge_values(gname, rng):
    """Tiles: randn; +-0 and subnormals among randn; all zero; +-max (FLT_MAX for fp32: the scale clamps); a NaN tile; an Inf
    tile; only subnormals; then a partial tile."""
    dmax = float(torch.finfo(GDT[gname]).max)
    sub = float(torch.finfo(GDT[gname]).smallest_normal) / 4
    tiles = [rng.standard_normal(TILE) * 1e-3]
    t = rng.standard_normal(TILE)
    t[:8] = [0.0, -0.0, sub, -sub, 3 * sub, -3 * sub, 1e-30, -1e-30]
    tiles.append(rng.permutation(t))
    tiles.append(np.zeros(TILE))
    tiles.append(np.where(rng.random(TILE) < 0.5, -dmax, dmax))
    t = rng.standard_normal(TILE)
    t[rng.integers(TILE)] = np.nan
    tiles.append(t)
    t = rng.standard_normal(TILE)
    t[rng.integers(TILE)] = -np.inf
    tiles.append(t)
    tiles.append(rng.integers(-5, 6, TILE) * sub / 8)
    tiles.append(rng.standard_normal(TILE - 613))
    return _dtype_values(np.concatenate(tiles), gname)


def stem_span(gname, rng, garbage=True):
    """A gradient span of the stem placement: randn on the real lanes, randn (or 0) on the padding (which must be ignored)."""
    real = ref_real_span(*STEM)
    x = rng.standard_normal(real.size) * np.where(real, 1.0, 1.0 if garbage else 0.0)
    return _dtype_values(x, gname), real


# ---------------------------------------------------------------------------------------------------------------------
# 1. the oracle (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_interface():
    spec = ps.Sign().device_spec()
    assert (spec.kind, spec.wire, spec.error_feedback) == (KIND_SIGN, WIRE_B1, True) == (4, 7, True)
    assert ps.Sign(error_feedback=False).device_spec().error_feedback is False
    assert all(spec.bytes_per_tile(dt) == 272 for dt in GDT.values())
    with pytest.raises(ValueError):
        ps.Sign().encode(torch.ones(3))                       # error feedback needs the parameter's name
    assert "Sign" in ps.__all__ and "error_feedback=True" in repr(ps.Sign())


@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
def test_oracle_matches_reference(gname):
    rng = np.random.default_rng(len(gname))
    x = edge_values(gname, rng)
    code = ps.Sign()
    enc = code.encode(torch.from_numpy(x).to(GDT[gname]), name="w")
    want, dec, res = ref_span(x, np.ones(len(x), bool))
    assert enc["wire"].dtype == torch.uint8 and tuple(enc["wire"].shape) == want.shape == (8, 272)
    assert np.array_equal(enc["wire"].numpy(), want)
    assert same_bits(code._residual["w"], res)
    scales = want[:, 256:260].copy().view(F32)[:, 0]
    assert (want[:, 260:] == 0).all() and np.isfinite(scales[[0, 1, 2, 3, 6, 7]]).all()
    assert scales[2] == 0 and scales[3] == FMAX if gname == "fp32" else np.isfinite(scales[3])
    assert (want[:, 256:260][[4, 5]].view(np.uint32) == 0x7FFFFFFF).all()            # NaN / Inf tile: NaN scale ...
    assert np.isfinite(scales[[3, 6]]).all()                                         # ... neighbours unaffected
    got = code.decode(enc).numpy()
    assert np.array_equal(got, dec[:len(x)], equal_nan=True) and got.shape == x.shape
    # the second step adds the residual
    y = _dtype_values(rng.standard_normal(len(x)), gname)
    enc2 = code.encode(torch.from_numpy(y).to(GDT[gname]), name="w")
    want2, _, _ = ref_span((y + res[:len(x)]).astype(F32), np.ones(len(x), bool))
    assert np.array_equal(enc2["wire"].numpy(), want2)
    noef = ps.Sign(error_feedback=False)
    assert np.array_equal(noef.encode(torch.from_numpy(y).to(GDT[gname]))["wire"].numpy(), ref_span(y, np.ones(len(y), bool))[0])
    assert noef._residual == {}


def test_oracle_custom_placement():
    """A real mask shaped like the stem's [64,176] placement: padding lanes carry garbage, get bit 0, count nowhere, decode to +0
    and keep a residual of 0."""
    rng = np.random.default_rng(3)
    x, real = stem_span("bf16", rng)
    code = ps.Sign()
    enc = code.encode(torch.from_numpy(x).to(torch.bfloat16), name="stem", real=torch.from_numpy(np.pad(real, (0, 6 * TILE - real.size))))
    want, dec, res = ref_span(x, real)
    assert np.array_equal(enc["wire"].numpy(), want)
    assert same_bits(code._residual["stem"], res) and (code._residual["stem"][:real.size][~real] == 0).all()
    got = code.decode(enc, real=np.pad(real, (0, 6 * TILE - real.size))).numpy()
    assert np.array_equal(got, dec[:real.size]) and (got[~real] == 0).all()


def test_oracle_error_feedback_identity():
    """Σ decoded + final residual == Σ gradients exactly over 50 steps.  Every real |p| lies in [1.25, 1.75] (so does the scale,
    their mean): p - decode is exact (Sterbenz), and each gradient is chosen as p - residual, which is exact too."""
    rng = np.random.default_rng(4)
    n = 2 * TILE + 300
    code = ps.Sign()
    tot_g, tot_d = np.zeros(n), np.zeros(n)
    res = np.zeros(n, F32)
    for _ in range(50):
        mag = 1.25 + rng.integers(0, 513, n) / 1024.0
        sign = np.where(res != 0, np.sign(res), rng.choice([-1.0, 1.0], n))
        g = (sign * mag - res.astype(np.float64)).astype(F32)
        assert (g.astype(np.float64) == sign * mag - res).all()
        enc = code.encode(torch.from_numpy(g), name="p")
        tot_g += g
        tot_d += code.decode(enc).numpy()
        res = code._residual["p"][:n]
    assert (tot_d + res == tot_g).all()


# ---------------------------------------------------------------------------------------------------------------------
# kernel harness: N virtual ranks over the real bindings (emulator: host tensors; GPU: device tensors)
# ---------------------------------------------------------------------------------------------------------------------
class Ranks:
    def __init__(self, be, specs, dtype, nranks, optim="sgd", ef=True):
        if be == "gpu":
            from pytorch_ps_mpi_b200.ops import ext
            self.m, self.dev = ext.cuda(), torch.device("cuda", 0)
        else:
            self.m, self.dev = _cuda_emu.build_extension(), torch.device("cpu")
            if self.m is None:
                pytest.skip("no g++")
        self.be, self.n, self.dtype, self.optim = be, nranks, dtype, optim
        self.params = []
        for shape, placement in specs:
            p = torch.nn.Parameter(torch.zeros(shape, dtype=dtype))
            if placement is not None:
                p.ps_arena_layout = placement
            self.params.append(p)
        self.L = L = FlatLayout([{"params": self.params}], {id(p): f"p{i}" for i, p in enumerate(self.params)})
        self.slots = [L.by_id[id(p)] for p in self.params]
        nt, npad = L.ntiles, L.numel_padded
        self.real = np.zeros(npad, bool)
        for (shape, placement), s in zip(specs, self.slots):
            r = ref_real_span(shape, placement)
            self.real[s.offset: s.offset + r.size] = r
        words = np.packbits(self.real, bitorder="little").view(np.int32)
        z = lambda k, dt: torch.zeros(k, dtype=dt, device=self.dev)      # noqa: E731
        self.mask = z(len(words), torch.int32).copy_(torch.from_numpy(words))
        self.tiles = L.tile_table_fast().to(self.dev)
        self.wires = [z(nt * BPT, torch.uint8) for _ in range(nranks)]
        self.scales = [z(L.nparams, torch.float32) for _ in range(nranks)]
        self.param_arenas = [z(npad, dtype) for _ in range(nranks)]
        self.signals = [z(512, torch.int64) for _ in range(nranks)]
        self.residuals = [z(npad, torch.float32) for _ in range(nranks)] if ef else None
        self.master = z(npad, torch.float32) if dtype != torch.float32 else None
        self.buf0, self.buf1, self.buf2 = z(npad, torch.float32), z(npad, torch.float32), z(npad, torch.float32)
        self.counters = z(8, torch.int32)
        P = self.m.UpdatePlan()
        P.kind, P.wire, P.opt = KIND_SIGN, WIRE_B1, 0 if optim == "sgd" else 1
        P.grid = min(nt, 3 if be == "emu" else self.m.update_max_grid(KIND_SIGN, WIRE_B1, P.opt))
        for r in range(nranks):
            P.set_rank_ptrs(r, self.wires[r].data_ptr(), self.scales[r].data_ptr(), self.param_arenas[r].data_ptr(),
                            self.signals[r].data_ptr())
        P.configure(nranks, 0, nt, BPT, TILE, DT[dtype], 1, 0, 0, 0, self.param_arenas[0].data_ptr(),
                    self.master.data_ptr() if self.master is not None else 0, self.buf0.data_ptr(), self.buf1.data_ptr(),
                    self.buf2.data_ptr(), self.tiles.data_ptr(), self.signals[0].data_ptr(), self.counters.data_ptr(),
                    self.counters.data_ptr() + 4)
        P.set_real_mask(self.mask.data_ptr())
        self.P = P

    def set_start(self, values):
        """Parameter arenas (every rank) and masters from per-slot f32 spans (non-real lanes must be 0)."""
        full = np.zeros(self.L.numel_padded, F32)
        for s, v in zip(self.slots, values):
            full[s.offset: s.offset + len(v)] = v
        t = torch.from_numpy(full)
        for a in self.param_arenas:
            a.copy_(t.to(self.dtype))
        if self.master is not None:
            self.master.copy_(t.to(self.dtype).float())

    def encode(self, r, spans, carry=None, keep=True):
        """Encode rank ``r``'s gradient spans; ``carry`` (f32, arena-shaped) is what the carry holds before the launch."""
        res = 0
        if carry is not None:
            self.residuals[r].copy_(torch.from_numpy(carry))
            res = self.residuals[r].data_ptr()
        grads = [torch.from_numpy(np.ascontiguousarray(x)).to(self.dtype).to(self.dev) for x in spans]
        S = self.slots
        self.m.encode(KIND_SIGN, WIRE_B1, grads, [s.first_tile for s in S], [s.ntiles for s in S], [s.index for s in S],
                      self.tiles.data_ptr(), self.wires[r].data_ptr(), 0, 0, res, BPT, 0, 1.0, keep_leftover=keep,
                      real_mask=self.mask.data_ptr())
        if self.be == "gpu":
            torch.cuda.synchronize()

    def update(self, hypers, contrib=None):
        self.P.launch(1, hypers, (1 << self.n) - 1 if contrib is None else contrib, 1.0, 0, 1, timeout_s=5.0)
        if self.be == "gpu":
            torch.cuda.synchronize()

    def wire_rows(self, r, s):
        return self.wires[r].cpu().numpy().copy()[s.first_tile * BPT:(s.first_tile + s.ntiles) * BPT].reshape(s.ntiles, BPT)

    def span(self, t, s):
        return t.cpu().float().numpy()[s.offset: s.offset + s.ntiles * TILE].copy()


BACKENDS = ["emu", pytest.param("gpu", marks=pytest.mark.gpu)]


# ---------------------------------------------------------------------------------------------------------------------
# 2. encode, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def _encode_specs(rng):
    """70 parameters (two encode launches): an edge-case one, the stem placement, and 68 small odd shapes."""
    odd = [((int(k),), None) for k in rng.integers(1, 3 * TILE, 66)] + [((7, 300), None), ((TILE,), None)]
    return [((8 * TILE - 613,), None), STEM] + odd


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("case", ["ef", "noef", "accumulate", "ef+accumulate"])
def test_encode_kernel_bits(be, gname, case):
    rng = np.random.default_rng(len(gname) * 13 + len(case))
    specs = _encode_specs(rng)
    V = Ranks(be, specs, GDT[gname], 2, ef=True)
    spans = [edge_values(gname, rng), stem_span(gname, rng, garbage=True)[0]]
    spans += [_dtype_values(rng.standard_normal(s.numel) * 10.0 ** rng.integers(-3, 3), gname) for s in V.slots[2:]]
    carry, keep = None, True
    if case != "noef":
        carry = np.zeros(V.L.numel_padded, F32)
        if case != "ef":
            carry[V.real] = rng.standard_normal(int(V.real.sum())).astype(F32)    # a carry is 0 outside the real lanes
        keep = case != "accumulate"
    V.encode(1, spans, carry=carry, keep=keep)
    got_res = V.residuals[1].cpu().numpy() if carry is not None else None
    for i, (s, x) in enumerate(zip(V.slots, spans)):
        p = x.astype(F32)
        p = np.pad(p, (0, s.ntiles * TILE - len(p)))
        if carry is not None:                                      # (-0 + 0 is +0: a carry changes the sign bit of -0)
            p = p + carry[s.offset: s.offset + s.ntiles * TILE]
        want, _, res = ref_span(p, V.real[s.offset: s.offset + s.ntiles * TILE])
        got = V.wire_rows(1, s)
        bad = np.flatnonzero((got != want).any(axis=1))
        assert not len(bad), (be, gname, case, i, bad.tolist(), np.flatnonzero(got[bad[0]] != want[bad[0]])[:8].tolist())
        if carry is not None:
            g = got_res[s.offset: s.offset + s.ntiles * TILE]
            if keep:
                assert np.array_equal(np.isnan(g), np.isnan(res)) and same_bits(g[~np.isnan(g)], res[~np.isnan(res)]), (case, i)
            else:
                assert (g == 0).all(), (case, i)                   # accumulation without error feedback: the carry is consumed


# ---------------------------------------------------------------------------------------------------------------------
# 3. decode + rank-ordered sum + optimizer + publication
# ---------------------------------------------------------------------------------------------------------------------
UPD_SPECS = [((3 * TILE + 99,), None), ((700,), None), STEM]


def _update_case(be, pname, world, optim, hyper):
    """One step from a random start: exact decode / rank-ordered sum (plain SGD, lr = 1, zero start) or a float64 reference of
    the optimizer (momentum, Nesterov, weight decay, Adam); every non-real lane of the parameter arena, the master and the state
    exactly 0."""
    rng = np.random.default_rng(world * 7 + len(pname) + len(optim))
    dtype = GDT[pname]
    V = Ranks(be, UPD_SPECS, dtype, world, optim=optim, ef=False)
    exact = optim == "sgd" and hyper == {}
    starts = []
    for s in V.slots:
        real = V.real[s.offset: s.offset + s.numel]
        starts.append(np.zeros(s.numel, F32) if exact else _dtype_values(np.where(real, rng.standard_normal(s.numel), 0), pname))
    V.set_start(starts)
    w0 = [V.span(V.master if V.master is not None else V.param_arenas[0], s) for s in V.slots]
    total = [np.zeros(s.ntiles * TILE, F32) for s in V.slots]
    for r in range(world):
        spans = []
        for i, s in enumerate(V.slots):
            x = _dtype_values(rng.standard_normal(s.numel) * (1 + r), pname)
            if r == world - 1 and i == 0:
                x[2 * TILE + 3] = np.nan                               # tile 2 of the first parameter: NaN update
            spans.append(x)
        V.encode(r, spans)
        for i, (s, x) in enumerate(zip(V.slots, spans)):
            real = V.real[s.offset: s.offset + s.ntiles * TILE]
            _, dec, _ = ref_span(x, real)
            with np.errstate(invalid="ignore"):
                total[i] = (total[i] + dec).astype(F32)                # rank order, fp32
    lr, mom, wd, nest = 0.05, 0.9, 1e-2, 1.0
    if optim == "sgd":
        h = [[1.0 if exact else lr, hyper.get("wd", 0.0), hyper.get("mom", 0.0), 0.0, 0, 0, 0, 0,
              float(hyper.get("nesterov", False)), 0, 1.0]]
    else:
        h = [[1e-2, wd, 0, 0, 0.9, 0.999, 1e-8, 1e-2 * math.sqrt(1 - 0.999) / (1 - 0.9), 0, 0, 1.0]]
    V.update(h)
    for i, s in enumerate(V.slots):
        real = V.real[s.offset: s.offset + s.ntiles * TILE]
        got = V.span(V.master if V.master is not None else V.param_arenas[0], s)
        g = total[i].astype(np.float64)
        nan = np.isnan(g)
        if i == 0:
            assert nan[real].any()
        assert np.isnan(got[real & nan]).all() and np.isfinite(got[real & ~nan]).all(), (be, "NaN tile → NaN update")
        ok = real & ~nan
        w = w0[i].astype(np.float64)
        if exact:
            assert same_bits(got[ok], -total[i][ok]), (be, pname, world, i)
        else:
            if optim == "sgd":
                gg = g + hyper.get("wd", 0.0) * w
                step = (gg + mom * gg) if hyper.get("nesterov") else gg
                want = w - lr * step
            else:
                gg = g + wd * w
                want = w - (1e-2 * math.sqrt(1 - 0.999) / (1 - 0.9)) * (0.1 * gg) / (np.sqrt(0.001 * gg * gg) + 1e-8)
            assert np.allclose(got[ok], want[ok], rtol=1e-5, atol=1e-6), float(np.abs(got[ok] - want[ok]).max())
        pad = ~real
        assert (got[pad] == 0).all() and (V.span(V.param_arenas[world - 1], s)[pad] == 0).all(), (be, "padding stays 0")
        for b in (V.buf0, V.buf1):
            assert (V.span(b, s)[pad] == 0).all()
        if dtype != torch.float32:
            for r in range(world):
                pub = V.span(V.param_arenas[r], s)
                assert np.array_equal(pub, torch.from_numpy(got).to(dtype).float().numpy(), equal_nan=True)


HYPERS = {"plain": {}, "momentum+wd": {"mom": 0.9, "wd": 1e-2}, "nesterov": {"mom": 0.9, "nesterov": True}}


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("world", [1, 2, 5, 16])
@pytest.mark.parametrize("pname", ["fp32", "bf16"])
def test_decode_sum_sgd(be, world, pname):
    _update_case(be, pname, world, "sgd", {})


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("world", [1, 2, 5, 16])
@pytest.mark.parametrize("hyper", ["momentum+wd", "nesterov", "adam"])
def test_optimizers(be, world, hyper):
    _update_case(be, "bf16" if world % 2 else "fp16", world, "adam" if hyper == "adam" else "sgd", HYPERS.get(hyper, {}))


# ---------------------------------------------------------------------------------------------------------------------
# 4.-7. the engines on the emulator, through the real bindings
# ---------------------------------------------------------------------------------------------------------------------
def _names(eng, model):
    names = {id(p): n for n, p in model.named_parameters()}
    return [(names[id(s.param)], s) for s in eng.layout.slots]


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_engine_error_feedback_identity(emu):
    """One rank of the device engine: Σ (decoded wire) + the engine's final residual == Σ gradients, exactly, over 50 steps."""
    n, steps = 2 * TILE + 300, 50

    def rank_main(rank, w):
        p = torch.nn.Parameter(torch.zeros(n))
        opt = ps.SGD([("p", p)], [p], engine="host", mode="ps", lr=0.0, code=ps.Sign())
        _attach(opt)
        eng = opt._engine
        rng = np.random.default_rng(9)
        tot_g, tot_d = np.zeros(n), np.zeros(n)
        for _ in range(steps):
            res = eng.residual.numpy()[:n].copy()
            mag = 1.25 + rng.integers(0, 513, n) / 1024.0
            sign = np.where(res != 0, np.sign(res), rng.choice([-1.0, 1.0], n))
            g = (sign * mag - res.astype(np.float64)).astype(F32)
            opt.zero_grad(set_to_none=True)
            (p * torch.from_numpy(g)).sum().backward()
            opt.step()
            tot_g += g
            tot_d += ps.Sign(error_feedback=False).decode({"wire": eng.wire_arena.view(-1, BPT).clone(), "shape": (n,)}).numpy()
        ok = bool((tot_d + eng.residual.numpy()[:n] == tot_g).all())
        opt.close()
        return ok

    assert run_ranks(emu, 1, rank_main) == [True]


def _sign_run(emu, n, mode, steps=3, optim="sgd", inactive_step=None, check_wires=True, **kw):
    """``n`` ranks of the device engine with ``Sign()`` on the tiny MLP.  Each step every rank's wire tiles must equal, byte for
    byte, what a per-rank oracle coding (its own residuals, keyed by name) encodes from that rank's gradients; its residual must
    equal the oracle's.  Returns per rank (parameters, is_server, residual per name before/after each step)."""
    hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-4) if optim == "sgd" else dict(lr=1e-2)

    def rank_main(rank, w):
        model = _model(torch.bfloat16)
        cls = ps.SGD if optim == "sgd" else ps.Adam
        opt = cls(model.named_parameters(), model.parameters(), engine="host", mode=mode, code=ps.Sign(), **hyper)
        _attach(opt, **kw)
        eng = opt._engine
        assert eng.kind == KIND_SIGN and eng.bpt == BPT and eng.reduce == 0
        oracle = ps.Sign()
        slots = _names(eng, model)
        hist = []
        for s in range(steps):
            opt.zero_grad(set_to_none=True)
            skip = inactive_step == s
            _loss(model, *_data(rank, s, torch.bfloat16), skip_head=skip).backward()
            grads = {name: sl.param.grad for name, sl in slots}
            before = eng.residual.clone()
            opt.step()
            if mode == "async" and rank == 0:
                continue
            hist.append((before, eng.residual.clone(), {name for name, g in grads.items() if g is None}))
            if check_wires:
                for name, sl in slots:
                    if grads[name] is None:
                        continue
                    enc = oracle.encode(grads[name], name=name)
                    got = eng.wire_arena[sl.first_tile * BPT:(sl.first_tile + sl.ntiles) * BPT].view(sl.ntiles, BPT)
                    assert torch.equal(got, enc["wire"]), (rank, s, name)
                    r = eng.residual[sl.offset: sl.offset + sl.ntiles * TILE].numpy()
                    assert same_bits(r, oracle._residual[name]), (rank, s, name)
        eng.check()
        w.barrier()
        out = ([p.detach().clone() for p in model.parameters()], eng.is_server, hist, slots)
        opt.close()
        return out

    return run_ranks(emu, n, rank_main)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("n,mode,optim", [(2, "ps", "sgd"), (3, "ps", "adam"), (2, "sharded", "sgd"), (3, "sharded", "adam"),
                                          (3, "allgather", "sgd")])
def test_sync_modes_wires_and_ranks(emu, n, mode, optim):
    """Every rank's wire tiles and residuals are bit-identical to the per-rank oracle every step; the published parameters are
    bit-identical on every rank, and equal what ps mode computes from the same wires."""
    res = _sign_run(emu, n, mode, optim=optim)
    for params, _, _, _ in res:
        for a, b in zip(params, res[0][0]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    if mode != "ps":
        ref = _sign_run(emu, n, "ps", optim=optim, check_wires=False)
        for a, b in zip(res[0][0], ref[0][0]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_inactive_parameter_keeps_its_residual(emu):
    """Step 1 skips the head (its hook does not fire): the head's residual is untouched, everyone else's moves."""
    res = _sign_run(emu, 2, "ps", steps=3, inactive_step=1)
    for _, _, hist, slots in res:
        before, after, skipped = hist[1]
        assert skipped == {"4.weight", "4.bias"}, skipped
        for name, sl in slots:
            sl_ = slice(sl.offset, sl.offset + sl.ntiles * TILE)
            assert torch.equal(before[sl_], after[sl_]) == (name in skipped), name
            assert bool(before[sl_].abs().sum() > 0)                      # there was a residual to keep


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_async_applies_each_coded_gradient_once(emu):
    """Async, one server and one worker: the server's parameters are w0 - lr * (sum of the decoded worker gradients), the
    decodes coming from an oracle with error feedback."""
    nsteps, lr = 3, 0.05

    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="async", quota=1, lr=lr, code=ps.Sign())
        _attach(opt)
        names = [n for n, _ in model.named_parameters()]
        grads = []
        if rank == 0:
            assert opt.serve() == nsteps
        else:
            for s in range(nsteps):
                opt.zero_grad(set_to_none=True)
                _loss(model, *_data(rank, s), skip_head=False).backward()
                grads.append([p.grad.detach().clone() for p in model.parameters()])
                opt.step()
        opt.close()
        return [p.detach().clone() for p in model.parameters()], grads, names

    res = run_ranks(emu, 2, rank_main)
    oracle = ps.Sign()
    want = [p.detach().clone() for p in _model().parameters()]
    for gs in res[1][1]:
        for i, g in enumerate(gs):
            want[i] -= lr * oracle.decode(oracle.encode(g, name=res[1][2][i])).reshape(g.shape)
    for a, b in zip(res[0][0], want):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), float((a - b).abs().max())


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_no_sync_last_micro_batch_outside_equals_all_inside(emu):
    """Three micro-batches inside ``no_sync()`` and the fourth outside give the same bits as all four inside and then
    ``step()``: the error-feedback residual is the carry in both."""

    def rank_main(rank, w):
        out = []
        for last_inside in (False, True):
            model = _model(torch.bfloat16)
            opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="ps", lr=0.05, momentum=0.9,
                         code=ps.Sign())
            _attach(opt)
            for s in range(2):
                opt.zero_grad(set_to_none=True)
                with opt.no_sync():
                    for mb in range(3 + last_inside):
                        _loss(model, *_data(rank, 10 * s + mb, torch.bfloat16), skip_head=False).backward()
                if not last_inside:
                    _loss(model, *_data(rank, 10 * s + 3, torch.bfloat16), skip_head=False).backward()
                opt.step()
            out.append(([p.detach().clone() for p in model.parameters()], opt._engine.residual.clone()))
            opt.close()
        return out

    for (pa, ra), (pb, rb) in run_ranks(emu, 2, rank_main):
        assert all(torch.equal(a.view(torch.int16), b.view(torch.int16)) for a, b in zip(pa, pb))
        assert same_bits(ra.numpy(), rb.numpy()) and bool(ra.abs().sum() > 0)


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_switch_reduction_refused_and_auto_is_p2p(emu):
    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="ps", lr=0.1, code=ps.Sign())
        with pytest.raises(ValueError, match="nvls"):
            _attach(opt, reduce="nvls")
        w.barrier()
        _attach(opt, reduce="auto")
        reduce = opt._engine.reduce
        opt.close()
        return reduce

    assert run_ranks(emu, 4, rank_main, multicast=True) == [0] * 4


# ---------------------------------------------------------------------------------------------------------------------
# 6. the package ResNet (stem weight in its [64,176] placement) at two emulated ranks
# ---------------------------------------------------------------------------------------------------------------------
def test_resnet_with_sign_keeps_stem_padding_zero(world):
    import threading

    from tests import test_multirank_engine_emulation as H
    n, steps = 2, 3
    cluster = H.Cluster(world.emu, n)
    out, errs = [None] * n, []

    def main(rank):
        H._tls.world, H._tls.m = H.World(cluster, rank), ModelM(cluster, world)
        try:
            model = _tiny_resnet()
            named = list(model.named_parameters())
            opt = ps.SGD(named, [p for _, p in named], lr=0.05, momentum=0.9, mode="ps", engine="device", code=ps.Sign())
            eng = opt._engine
            assert eng.kind == KIND_SIGN
            model.attach(opt)
            for s in range(steps):
                x, y = _batch(rank, s)
                opt.zero_grad(set_to_none=True)
                torch.nn.functional.cross_entropy(model(x).float(), y).backward()
                opt.step()
            eng.ensure_params()
            eng.check()
            H._tls.world.barrier()
            sl = eng.layout.by_id[id(model.conv1.weight)]
            assert sl.strides == STEM_STRIDES
            pad = ~ref_real_span(*STEM)
            span = slice(sl.offset, sl.offset + sl.numel)
            arenas = [eng.param_arena[span].float(), eng.residual[span]]
            if eng.is_server:
                arenas += [eng.master[span], eng.buf0[span]]
            out[rank] = ([p.detach().clone() for p in model.parameters()], [bool((a[torch.from_numpy(pad)] == 0).all()) for a in arenas],
                         bool(eng.residual[span][torch.from_numpy(~pad)].abs().sum() > 0))
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
        raise errs[0]
    for params, zero, moved in out:
        assert all(zero) and moved
        for a, b in zip(params, out[0][0]):
            assert torch.equal(a, b)
        assert all(torch.isfinite(p).all() for p in params)


# ---------------------------------------------------------------------------------------------------------------------
# 7. the host engine and training
# ---------------------------------------------------------------------------------------------------------------------
def host_two_ranks(rank, size):
    """One process of ``test_host_engine_two_ranks``: every message the host engine sends equals the oracle's bytes, and the
    server applies the sum of both ranks' decodes."""
    from pytorch_ps_mpi_b200 import runtime
    w = runtime.init()
    p = torch.nn.Parameter(torch.zeros(3000))
    code = ps.Sign()
    sent = []
    enc = code.encode

    def recording(grad, **kw):
        out = enc(grad, **kw)
        sent.append(out["wire"].clone())
        return out

    code.encode = recording
    opt = ps.SGD([("p", p)], [p], engine="host", mode="ps", lr=1.0, code=code)
    oracle, mine = ps.Sign(), []
    for s in range(2):
        gr = torch.randn(3000, generator=torch.Generator().manual_seed(10 * s + rank))
        mine.append(gr)
        opt.zero_grad(set_to_none=True)
        (p * gr).sum().backward()
        opt.step()
    assert len(sent) == 2
    for gr, wire in zip(mine, sent):
        assert torch.equal(wire, oracle.encode(gr, name="p")["wire"])
    allg = w.all_gather_object(mine)
    ref = [ps.Sign() for _ in range(size)]
    want = torch.zeros(3000)
    for s in range(2):
        want -= sum(ref[r].decode(ref[r].encode(allg[r][s], name="p")) for r in range(size))
    assert torch.allclose(p.detach(), want, rtol=1e-6, atol=1e-6), float((p.detach() - want).abs().max())
    opt.close()
    w.barrier()


def test_host_engine_two_ranks():
    from pytorch_ps_mpi_b200.launch import spawn
    spawn(host_two_ranks, 2, env={"PSB200_TRANSPORT": "shm"}, timeout=240)


def test_error_feedback_sign_trains_least_squares():
    """A seeded least-squares problem: 200 steps of error-feedback sign SGD take the loss below 10 % of its start."""
    g = torch.Generator().manual_seed(0)
    A = torch.randn(256, 64, generator=g) / 16.0
    b = A @ torch.randn(64, generator=g)
    x = torch.nn.Parameter(torch.zeros(64))
    opt = ps.SGD([("x", x)], [x], engine="host", use_mpi=False, lr=0.5, code=ps.Sign())
    losses = []
    for _ in range(200):
        opt.zero_grad(set_to_none=True)
        loss = 0.5 * ((A @ x - b) ** 2).sum()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    opt.close()
    assert losses[-1] < 0.1 * losses[0], (losses[0], losses[-1])


# ---------------------------------------------------------------------------------------------------------------------
# 8. the device engine on one GPU, two ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_engine_ranks_one_gpu():
    from pytorch_ps_mpi_b200.launch import spawn
    from tests.test_gpu_engine import ONE_GPU
    spawn(gpu_two_ranks, 2, env=ONE_GPU, timeout=240)


def gpu_two_ranks(rank, size):
    """One process of ``test_two_engine_ranks_one_gpu``: ``engine='device'`` on bf16 parameters (one with the stem placement)
    with ``Sign()``: 272-byte wire tiles equal to the oracle's, ranks bit-identical, padding exactly 0."""
    from pytorch_ps_mpi_b200 import runtime
    w = runtime.init()
    dev = w.device
    torch.manual_seed(0)
    shapes = [(3000,), (40, 70), STEM[0]]
    params = [torch.nn.Parameter(torch.randn(s).to(torch.bfloat16).to(dev)) for s in shapes]
    params[2].ps_arena_layout = STEM[1]
    opt = ps.SGD([(f"p{i}", p) for i, p in enumerate(params)], params, engine="device", mode="ps", lr=0.1, code=ps.Sign())
    eng = opt._engine
    assert eng is not None and eng.kind == KIND_SIGN and eng.wire_arena.numel() == BPT * eng.layout.ntiles
    slots = [eng.layout.by_id[id(p)] for p in params]
    oracle = ps.Sign()
    real = torch.from_numpy(ref_real_span(*STEM))
    for s in range(3):
        gs = [torch.randn(sh, generator=torch.Generator().manual_seed(100 * s + rank)).to(torch.bfloat16) for sh in shapes]
        opt.zero_grad(set_to_none=True)
        sum((p.float() * g.to(dev).float()).sum() for p, g in zip(params, gs)).backward()
        opt.step()
        torch.cuda.synchronize()
        for i, (sl, g) in enumerate(zip(slots, gs)):
            if i == 2:                                     # the span the engine encodes: the weight in its placement
                span = torch.zeros(sl.numel, dtype=g.dtype)
                torch.as_strided(span, g.shape, sl.strides).copy_(g)
                enc = oracle.encode(span, name=f"p{i}", real=torch.nn.functional.pad(real, (0, sl.ntiles * TILE - sl.numel)))
            else:
                enc = oracle.encode(g, name=f"p{i}")
            got = eng.wire_arena[sl.first_tile * BPT:(sl.first_tile + sl.ntiles) * BPT].view(sl.ntiles, BPT).cpu()
            assert torch.equal(got, enc["wire"]), (rank, s, i)
    eng.check()
    torch.cuda.synchronize()
    stem = eng.param_arena[slots[2].offset: slots[2].offset + slots[2].numel].cpu()
    assert (stem[~real] == 0).all()
    res = w.all_gather_object([p.detach().cpu().clone() for p in params])
    opt.close()
    if rank == 0:
        for a, b in zip(res[0], res[1]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    w.barrier()
