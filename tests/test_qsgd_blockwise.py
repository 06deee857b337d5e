"""Block-wise QSGD (``QSGD(blockwise=True)``), bit for bit: the Philox generator, the ``codings.py`` oracle, the encode and
update kernels, and the engines.

The reference here is numpy, written from the rules of ``DESIGN.md`` (wire numerics): a scalar Philox4x32-10 checked against
Random123's known answers, the tile norm scaled by the finite abs-max and summed in the kernel's documented order, stochastic
rounding, the NaN codes and the saturated scale.  Against it:

* ``QSGD(blockwise=True).encode`` (CPU);
* ``psb_encode_kernel<KIND_QSGD, WIRE_I8 | WIRE_I4>``: wire bytes and tile headers, levels 1 / 7 / 8 / 127, fp32 / bf16 / fp16
  gradients, random, partial and all-zero tiles, NaN / +-Inf / +-0 / subnormals / +-max, a tile whose norm overflows fp32, x on
  integer levels;
* unbiasedness of the kernel's codes over 4096 (GPU) or 512 (emulator) steps;
* ``psb_update_kernel<KIND_QSGD, ...>``: decode, rank-ordered sum, SGD / Adam, publication at 1, 2, 5 and 16 ranks;
* the engines: ps / allgather / async through the real bindings on the emulator, checkpoint and resume, two ranks on one GPU,
  and the host engine at two ranks.

Kernel cases run on the CPU emulator of the same source (default run) and on the GPU (``-m gpu``)."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200.codings import KIND_QSGD, TILE, WIRE_I4, WIRE_I8, philox4x32_10
from tests import _cuda_emu
from tests.test_multirank_engine_emulation import _attach, _data, _loss, _model, emu, run_ranks  # noqa: F401  (emu: fixture)

GDT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
FMAX = np.float32(np.finfo(np.float32).max)


# ---------------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------------
def philox_scalar(ctr, key):
    """Philox4x32-10 on Python integers, as in Random123's philox.h."""
    c, (k0, k1) = list(ctr), key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c[3] ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF]
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c


KNOWN = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
         ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
         ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
          (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]


def ref_uniforms(tile, step, rank, seed):
    """u of the 2048 elements of one arena tile: word e & 3 of Philox((e >> 2, tile, step, rank), seed), (w >> 8) * 2^-24."""
    words = [philox_scalar((i, tile, step, rank), (seed & 0xFFFFFFFF, seed >> 32)) for i in range(TILE // 4)]
    w = np.array(words, np.uint64).reshape(-1)
    return (w >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)


def ref_tile(g, levels, u):
    """(codes as ints, NaN mask, fp32 scale) of one tile ``g`` (float32, zero-padded to 2048)."""
    f32 = np.float32
    fin = np.isfinite(g)
    a = np.where(fin, np.abs(g), f32(0))
    m = a.max()
    anyv = m > 0
    m = m if anyv else f32(1)
    t = np.where(fin, a / m, f32(0)).astype(np.float32)
    per_thread = (t * t).reshape(256, 8)
    s = per_thread[:, 0]
    for j in range(1, 8):
        s = (s + per_thread[:, j]).astype(np.float32)
    s = s.reshape(8, 32)
    for off in (16, 8, 4, 2, 1):
        s = (s + s[:, np.arange(32) ^ off]).astype(np.float32)
    tot = s[0, 0]
    for w in range(1, 8):
        tot = f32(tot + s[w, 0])
    r = np.sqrt(tot, dtype=np.float32) if anyv else f32(1)
    lv = f32(levels)
    x = ((t / r).astype(np.float32) * lv).astype(np.float32)
    fl = np.floor(x)
    qi = np.minimum(fl.astype(np.int64) + (u < (x - fl)), levels)
    qi = np.where(np.isinf(g), levels, qi)
    q = np.where(np.signbit(g), -qi, qi)
    with np.errstate(over="ignore"):
        scale = f32(m * f32(r / lv))
    return q, np.isnan(g), (FMAX if np.isinf(scale) else scale)


def ref_wire(x, levels, seed, step, rank, first_tile):
    """Expected wire bytes [ntiles, bytes_per_tile] of one parameter (``x``: float64 values of the gradient dtype)."""
    g = np.zeros(max(1, -(-len(x) // TILE)) * TILE, np.float32)
    with np.errstate(over="ignore"):
        g[:len(x)] = x.astype(np.float32)
    rows = []
    for t in range(len(g) // TILE):
        q, nan, scale = ref_tile(g[t * TILE:(t + 1) * TILE], levels, ref_uniforms(first_tile + t, step, rank, seed))
        if levels <= 7:
            c = np.where(nan, 8, q & 0xF).astype(np.uint8)
            pay = c[0::2] | (c[1::2] << 4)
        else:
            pay = np.where(nan, 0x80, q & 0xFF).astype(np.uint8)
        head = np.zeros(4, np.float32)
        head[0] = scale
        rows.append(np.concatenate([pay, head.view(np.uint8)]))
    return np.stack(rows)


def ref_decode(wire_rows, n):
    """float64 values q * scale (fp32 product) of a parameter's wire rows; NaN codes → NaN."""
    pay = wire_rows.shape[1] - 16
    scale = wire_rows[:, pay:pay + 4].copy().view(np.float32)[:, 0]
    if pay == TILE // 2:
        b = wire_rows[:, :pay].astype(np.int64)
        q = np.stack([b & 0xF, b >> 4], axis=2).reshape(len(b), TILE)
        q = np.where(q >= 8, q - 16, q)
        nan = q == -8
    else:
        q = wire_rows[:, :pay].view(np.int8).astype(np.int64)
        nan = q == -128
    with np.errstate(over="ignore", invalid="ignore"):
        v = (q.astype(np.float32) * scale[:, None]).astype(np.float64)
    return np.where(nan, np.nan, v).reshape(-1)[:n]


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _as_dtype(x, gname):
    """float64 values rounded to the gradient dtype (NaN and -0 kept)."""
    with np.errstate(over="ignore"):
        return torch.from_numpy(x).to(GDT[gname]).double().numpy()


def edge_param(gname, rng):
    """Tiles: randn; specials among randn; all zero; +-max (norm overflows fp32 for fp32 / bf16); one non-zero element (x =
    levels exactly); four +-1 (x = levels / 2); only subnormals; then a partial tile."""
    dmax = float(torch.finfo(GDT[gname]).max)
    sub = float(torch.finfo(GDT[gname]).smallest_normal) / 4
    tiles = [rng.standard_normal(TILE) * 1e-3]
    t = rng.standard_normal(TILE)
    t[:14] = [np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, sub, -sub, 3 * sub, dmax, -dmax, 1e-30, -1e-30, 1e30]
    tiles.append(rng.permutation(t))
    tiles.append(np.zeros(TILE))
    tiles.append(np.where(rng.random(TILE) < 0.5, -dmax, dmax) * rng.choice([1.0, 0.5, 0.25], TILE))
    t = np.zeros(TILE)
    t[rng.integers(TILE)] = -3.0
    tiles.append(t)
    t = np.zeros(TILE)
    t[rng.choice(TILE, 4, replace=False)] = [1.0, -1.0, 1.0, -1.0]
    tiles.append(t)
    tiles.append(rng.integers(-5, 6, TILE) * sub / 8)
    tiles.append(rng.standard_normal(TILE - 613))
    return _as_dtype(np.concatenate(tiles), gname)


# ---------------------------------------------------------------------------------------------------------------------
# back-ends: the GPU harness and the CPU emulator, with the QSGD encode arguments
# ---------------------------------------------------------------------------------------------------------------------
DRIVER = r'''
extern "C" int emu_encode_qsgd(int wire, int n, const void** src, const int* first_tile, const int* ntiles, const int* param,
                               const void* tiles, void* wire_arena, int bpt, int grad_dt, uint64_t seed, uint32_t step,
                               uint32_t rank, int levels) {
  EncodeArgs a{};
  a.batch.n = n; a.batch.cum[0] = 0;
  for (int i = 0; i < n; ++i) { a.batch.src[i] = src[i]; a.batch.first_tile[i] = first_tile[i]; a.batch.param[i] = param[i]; a.batch.cum[i + 1] = a.batch.cum[i] + ntiles[i]; }
  a.tiles = reinterpret_cast<const TileInfo*>(tiles); a.wire = wire_arena; a.bytes_per_tile = bpt; a.grad_dt = grad_dt;
  a.seed = seed; a.step = step; a.rank = rank; a.levels = levels;
  psb_launch_encode(nullptr, KIND_QSGD, wire, a);
  return 0;
}
'''
_QLIB = []


def _qlib():
    if not _QLIB:
        import shutil
        if shutil.which("g++") is None:
            pytest.skip("no g++")
        _QLIB.append(_cuda_emu.compile_shared(_cuda_emu.kernel_source() + DRIVER, "psb_qsgd_emu_"))
    return _QLIB[0]


def _make(backend, shapes, dtype, code, nranks, optim="sgd"):
    if backend == "gpu":
        from tests.test_gpu_kernels import Virtual

        class QVirtual(Virtual):
            def encode(self, r, grads, step=0):
                L = self.L
                order = [(L.by_id[id(p)], g.cuda().contiguous()) for p, g in zip(self.params, grads)]
                self.m.encode(self.kind, self.wire, [g for _, g in order], [s.first_tile for s, _ in order],
                              [s.ntiles for s, _ in order], [s.index for s, _ in order], self.tiles.data_ptr(),
                              self.wires[r].data_ptr(), 0, 0, 0, self.bpt, 0, 1.0, seed=self.spec.seed, step=step, rank=r,
                              levels=self.spec.levels)
                torch.cuda.synchronize()

        return QVirtual(shapes, dtype, code, nranks, optim=optim)
    from tests.test_ps_kernels_cpu_emulation import VirtualCPU, _arr, _ptr

    class QVirtualCPU(VirtualCPU):
        def encode(self, r, grads, step=0):
            L = self.L
            order = [(L.by_id[id(p)], g.contiguous()) for p, g in zip(self.params, grads)]
            n = len(order)
            ia = lambda xs: (ctypes.c_int * n)(*xs)      # noqa: E731
            rc = self.lib.emu_encode_qsgd(self.wire, n, _arr([g.data_ptr() for _, g in order]), ia([s.first_tile for s, _ in order]),
                                          ia([s.ntiles for s, _ in order]), ia([s.index for s, _ in order]), _ptr(self.tiles),
                                          _ptr(self.wires[r]), self.bpt, DT[order[0][1].dtype], ctypes.c_uint64(self.spec.seed),
                                          ctypes.c_uint32(step), ctypes.c_uint32(r), self.spec.levels)
            assert rc == 0

    return QVirtualCPU(_qlib(), shapes, dtype, code, nranks, optim=optim)


def _wire_rows(V, r, slot):
    w = V.wires[r].cpu().numpy()
    return w[slot.first_tile * V.bpt:(slot.first_tile + slot.ntiles) * V.bpt].reshape(slot.ntiles, V.bpt)


def _to_torch(x, gname):
    return torch.from_numpy(x).to(GDT[gname])


BACKENDS = ["emu", pytest.param("gpu", marks=pytest.mark.gpu)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the oracle (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    for ctr, key, want in KNOWN:
        assert tuple(philox_scalar(ctr, key)) == want
        assert tuple(int(w) for w in philox4x32_10(*ctr, *key)) == want


@pytest.mark.parametrize("levels", [1, 7, 8, 127])
@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
def test_codings_oracle_matches_reference(levels, gname):
    rng = np.random.default_rng(levels * 7 + len(gname))
    x = edge_param(gname, rng)
    code = ps.QSGD(levels=levels, seed=0x1234_5678_9ABC_DEF0 + levels, blockwise=True)
    enc = code.encode(_to_torch(x, gname), step=3, rank=2, first_tile=5)
    want = ref_wire(x, levels, code.seed, 3, 2, 5)
    assert enc["wire"].dtype == torch.uint8 and tuple(enc["wire"].shape) == want.shape
    assert enc["wire"].shape[1] == code.device_spec().bytes_per_tile(GDT[gname]) == (1040 if levels <= 7 else 2064)
    assert np.array_equal(enc["wire"].numpy(), want)
    dec = code.decode(enc).double().numpy()
    assert np.array_equal(dec, ref_decode(want, len(x)), equal_nan=True)
    scales = want[:, -16:-12].copy().view(np.float32)[:, 0]
    assert np.isfinite(scales).all() and (want[:, -12:] == 0).all()


def test_interface_and_whole_tensor_qsgd_unchanged():
    assert ps.QSGD(levels=15, seed=1).device_spec() is None
    for bad in (0, 128, -3):
        with pytest.raises(ValueError):
            ps.QSGD(levels=bad, blockwise=True)
    spec = ps.QSGD(levels=7, seed=5, blockwise=True).device_spec()
    assert (spec.kind, spec.wire, spec.levels, spec.seed) == (KIND_QSGD, WIRE_I4, 7, 5)
    assert ps.QSGD(levels=8, blockwise=True).device_spec().wire == WIRE_I8
    assert "blockwise=True" in repr(ps.QSGD(levels=8, blockwise=True)) and "levels=8" in repr(ps.QSGD(levels=8, blockwise=True))
    # the whole-tensor coding: the same draws as before (torch.rand on the seeded generator), int8 codes, norm travels
    g = torch.randn(300, 7)
    enc = ps.QSGD(levels=15, seed=1).encode(g, name="w")
    norm = g.norm()
    x = g.abs() / norm * 15
    up = torch.rand(x.shape, generator=torch.Generator().manual_seed(1)) < (x - x.floor())
    assert set(enc) == {"q", "norm", "levels", "shape"} and enc["q"].dtype == torch.int8
    assert torch.equal(enc["q"], ((x.floor() + up.float()) * g.sign()).to(torch.int8))
    assert torch.equal(ps.QSGD(levels=15).decode(enc), enc["q"].float() * (enc["norm"] / 15.0))


def test_host_defaults_draw_per_name_and_step():
    """Without step / rank / first tile (the host engine passes only name=): a call counter per name and crc32(name)."""
    from pytorch_ps_mpi_b200 import runtime
    rank = runtime.rank() if runtime.is_initialized() else 0       # an earlier test in this process may have set up a world
    g = torch.randn(3000, generator=torch.Generator().manual_seed(34))
    code = ps.QSGD(levels=8, seed=9, blockwise=True)
    a0, b0, a1 = code.encode(g, name="a"), code.encode(g, name="b"), code.encode(g, name="a")
    assert np.array_equal(a0["wire"].numpy(), ref_wire(g.double().numpy(), 8, 9, 0, rank, zlib.crc32(b"a")))
    assert np.array_equal(a1["wire"].numpy(), ref_wire(g.double().numpy(), 8, 9, 1, rank, zlib.crc32(b"a")))
    assert np.array_equal(b0["wire"].numpy(), ref_wire(g.double().numpy(), 8, 9, 0, rank, zlib.crc32(b"b")))


# ---------------------------------------------------------------------------------------------------------------------
# 2. encode, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("levels", [1, 7, 8, 127])
@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
def test_encode_wire_bits(be, levels, gname):
    rng = np.random.default_rng(levels * 31 + len(gname))
    xs = [edge_param(gname, rng), _as_dtype(rng.standard_normal(TILE + 77) * 5, gname)]
    code = ps.QSGD(levels=levels, seed=(levels << 40) | 77, blockwise=True)
    V = _make(be, [(len(x),) for x in xs], GDT[gname], code, 2)
    for step, r in ((0, 0), (11, 1)):
        V.encode(r, [_to_torch(x, gname) for x in xs], step=step)
        for i, (p, x) in enumerate(zip(V.params, xs)):
            slot = V.L.by_id[id(p)]
            want = ref_wire(x, levels, code.seed, step, r, slot.first_tile)
            got = _wire_rows(V, r, slot)
            bad = np.flatnonzero((got != want).any(axis=1))
            assert not len(bad), (be, levels, gname, i, r, bad.tolist(), np.flatnonzero(got[bad[0]] != want[bad[0]])[:8].tolist())


@pytest.mark.parametrize("be", BACKENDS)
def test_unbiased_over_steps(be):
    """One fixed tile encoded at many step values: the mean decode is within 5 sigma of g per element."""
    steps = 4096 if be == "gpu" else 512
    rng = np.random.default_rng(5)
    x = _as_dtype(rng.standard_normal(TILE) * np.exp(rng.standard_normal(TILE)), "fp32")
    code = ps.QSGD(levels=7, seed=3, blockwise=True)
    V = _make(be, [(TILE,)], torch.float32, code, 1)
    slot = V.L.by_id[id(V.params[0])]
    g = _to_torch(x, "fp32")
    total = np.zeros(TILE)
    for s in range(steps):
        V.encode(0, [g], step=s)
        total += ref_decode(_wire_rows(V, 0, slot), TILE)
    mean = total / steps
    q, _, scale = ref_tile(x.astype(np.float32), 7, np.zeros(TILE, np.float32))
    xs = np.abs(x) / float(scale)
    f = xs - np.floor(xs)
    sigma = float(scale) * np.sqrt(f * (1 - f) / steps)
    assert (np.abs(mean - x) <= 5 * sigma + 1e-5 * float(scale)).all()


# ---------------------------------------------------------------------------------------------------------------------
# 3. decode + rank-ordered sum + optimizer + publication
# ---------------------------------------------------------------------------------------------------------------------
def _ulp32(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def _update_case(be, levels, pname, world, optim="sgd", n=3 * TILE + 99, extra=700):
    rng = np.random.default_rng(world * 17 + levels + len(pname))
    code = ps.QSGD(levels=levels, seed=world, blockwise=True)
    dtype = GDT[pname]
    shapes = [(n,), (extra,)]
    V = _make(be, shapes, dtype, code, world, optim=optim)
    for a in V.param_arenas:
        a.zero_()
    if V.master is not None:
        V.master.zero_()
    grads = []
    for r in range(world):
        gs = [rng.standard_normal(s[0]) * (1 + r) for s in shapes]
        if r == world - 1:
            gs[0][[5, 2 * TILE + 3]] = [np.nan, np.inf]
        gs = [_as_dtype(x, pname) for x in gs]
        grads.append(gs)
        V.encode(r, [_to_torch(x, pname) for x in gs], step=7)
    if optim == "sgd":
        V.update(1, [[1.0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1.0]])
    else:
        V.update(1, [[0.1, 0, 0, 0, 0.9, 0.999, 1e-8, 0.1 * math.sqrt(1 - 0.999) / (1 - 0.9), 0, 0, 1.0]])
    for i, p in enumerate(V.params):
        slot = V.L.by_id[id(p)]
        terms = [ref_decode(ref_wire(grads[r][i], levels, code.seed, 7, r, slot.first_tile), slot.numel) for r in range(world)]
        got = (V.master if V.master is not None else V.param_arenas[0])[slot.offset:slot.offset + slot.numel].cpu().numpy()
        with np.errstate(over="ignore", invalid="ignore"):
            part, bound = np.zeros(slot.numel), np.zeros(slot.numel)
            for t in terms:
                part = part + t
                bound += _ulp32(np.maximum(np.abs(part), np.abs(t)))
        nan = np.isnan(part)
        assert np.isnan(got[nan]).all() and np.isfinite(got[~nan]).all(), (be, "NaN code → NaN update")
        if optim == "sgd":
            err = np.abs(got[~nan].astype(np.float64) + part[~nan])      # master = -(sum), lr = 1, zero start
            assert (err <= bound[~nan]).all(), (be, levels, pname, world, i, float((err - bound[~nan]).max()))
        else:                                                         # the first Adam step from zero state
            g = part[~nan]
            want = -(0.1 * math.sqrt(1 - 0.999) / (1 - 0.9)) * (0.1 * g) / (np.sqrt(0.001 * g * g) + 1e-8)
            assert np.allclose(got[~nan], want, rtol=1e-5, atol=1e-7), float(np.abs(got[~nan] - want).max())
        if dtype != torch.float32:
            for r in range(world):
                pub = V.param_arenas[r][slot.offset:slot.offset + slot.numel].cpu().float().numpy()
                assert np.array_equal(pub, torch.from_numpy(got).to(dtype).float().numpy(), equal_nan=True)


_UPD = [(lv, p, n) for lv in (7, 127) for p in ("fp32", "bf16", "fp16") for n in (1, 2, 5, 16)]
_UPD_EMU = [(7, "fp32", 16), (127, "bf16", 5), (7, "fp16", 2), (127, "fp32", 1), (8, "bf16", 16)]


@pytest.mark.parametrize("levels,pname,world", _UPD_EMU)
def test_decode_sum_update_emulated(levels, pname, world):
    _update_case("emu", levels, pname, world)


@pytest.mark.gpu
@pytest.mark.parametrize("levels,pname,world", _UPD)
def test_decode_sum_update_gpu(levels, pname, world):
    _update_case("gpu", levels, pname, world)


@pytest.mark.parametrize("be", BACKENDS)
@pytest.mark.parametrize("levels", [7, 127])
def test_adam_update(be, levels):
    _update_case(be, levels, "bf16", 3, optim="adam")


@pytest.mark.gpu
@pytest.mark.parametrize("levels", [7, 127])
def test_grid_stride_arena_gpu(levels):
    """More than 3 x 132 tiles: the update kernel's grid-stride loop."""
    _update_case("gpu", levels, "bf16", 2, n=450 * TILE + 123)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the engines
# ---------------------------------------------------------------------------------------------------------------------
def _named_slots(eng, model):
    return [eng.layout.by_id[id(p)] for p in model.parameters()]


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
@pytest.mark.parametrize("n,mode,optim,levels", [(2, "ps", "sgd", 7), (3, "allgather", "adam", 127), (3, "ps", "adam", 8)])
def test_sync_modes_against_gathered_gradients(emu, n, mode, optim, levels):
    """Each step every rank's actual gradient is gathered and encoded by the oracle with that rank, step and arena tile; the
    decoded sum drives the reference optimizer on fp32 shadows.  The engine's masters match and all ranks are bit-identical."""
    hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-4) if optim == "sgd" else dict(lr=1e-2, eps=1e-8)
    dtype, steps = torch.bfloat16, 3

    def rank_main(rank, w):
        model = _model(dtype)
        shadow = [torch.nn.Parameter(p.detach().float().clone()) for p in model.parameters()]
        cls = ps.SGD if optim == "sgd" else ps.Adam
        oracle = cls([(f"p{i}", q) for i, q in enumerate(shadow)], shadow, engine="host", use_mpi=False, **hyper)
        for h in oracle._hooks:
            h.remove()
        groups = oracle._group_of()
        code = ps.QSGD(levels=levels, seed=42, blockwise=True)
        opt = cls(model.named_parameters(), model.parameters(), engine="host", mode=mode, code=code, **hyper)
        _attach(opt)
        eng = opt._engine
        assert eng.kind == KIND_QSGD and eng.reduce == 0 and eng.bpt == (1040 if levels <= 7 else 2064)
        slots = _named_slots(eng, model)
        for s in range(steps):
            opt.zero_grad(set_to_none=True)
            _loss(model, *_data(rank, s, dtype), skip_head=False).backward()
            mine = [p.grad.detach().clone() for p in model.parameters()]
            opt.step()
            allg = w.all_gather_object(mine)
            with torch.no_grad():
                for i, q in enumerate(shadow):
                    total = torch.zeros_like(q)
                    for r in range(n):
                        enc = code.encode(allg[r][i], step=s, rank=r, first_tile=slots[i].first_tile)
                        total += code.decode(enc).reshape(q.shape).float()
                    oracle.optim_step(q, total, **oracle._hyper(groups[id(q)]))
        eng.check()
        w.barrier()
        got = [(opt.state[p]["master_param"] if eng.master is not None else p).detach().float().clone() for p in model.parameters()]
        pub = [p.detach().clone() for p in model.parameters()]
        opt.close()
        oracle.close()
        return got, pub, [q.detach().clone() for q in shadow], eng.is_server

    res = run_ranks(emu, n, rank_main)
    for got, pub, shadow, is_server in res:
        for a, b in zip(pub, res[0][1]):
            assert torch.equal(a, b)
        if is_server:
            for g, q in zip(got, shadow):
                assert torch.allclose(g, q, rtol=2e-4, atol=2e-5), float((g - q).abs().max())


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_async_applies_each_coded_gradient_once(emu):
    """Async, one server and one worker: the server's parameters are w0 - lr * (sum of the decoded worker gradients)."""
    nsteps, n, lr = 3, 2, 0.05
    code_args = dict(levels=7, seed=11, blockwise=True)

    def rank_main(rank, w):
        model = _model()
        opt = ps.SGD(model.named_parameters(), model.parameters(), engine="host", mode="async", quota=1, lr=lr,
                     code=ps.QSGD(**code_args))
        _attach(opt)
        eng = opt._engine
        slots = [s.first_tile for s in _named_slots(eng, model)]
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
        return [p.detach().clone() for p in model.parameters()], grads, slots

    res = run_ranks(emu, n, rank_main)
    code = ps.QSGD(**code_args)
    want = [p.detach().clone() for p in _model().parameters()]
    for s, gs in enumerate(res[1][1]):
        for i, g in enumerate(gs):
            want[i] -= lr * code.decode(code.encode(g, step=s, rank=1, first_tile=res[1][2][i])).reshape(g.shape)
    for a, b in zip(res[0][0], want):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), float((a - b).abs().max())


@pytest.mark.parametrize("emu", ["bindings"], indirect=True)
def test_checkpoint_resume_bit_for_bit(emu):
    """2 steps + state_dict() + load into fresh objects + 2 steps == 4 straight steps, bit for bit, on both ranks."""
    import copy

    def rank_main(rank, w):
        def make():
            net = _model(torch.bfloat16)
            o = ps.SGD(net.named_parameters(), net.parameters(), engine="host", mode="ps", lr=0.05, momentum=0.9,
                       code=ps.QSGD(levels=7, seed=2, blockwise=True))
            _attach(o)
            return net, o

        def run(net, o, start, steps):
            for s in range(start, start + steps):
                o.zero_grad(set_to_none=True)
                _loss(net, *_data(rank, s, torch.bfloat16), skip_head=False).backward()
                o.step()

        m1, o1 = make()
        run(m1, o1, 0, 4)
        want = [p.detach().clone() for p in m1.parameters()]
        o1.close()
        m2, o2 = make()
        run(m2, o2, 0, 2)
        sd_model = {k: v.clone() for k, v in m2.state_dict().items()}
        sd_opt = copy.deepcopy(o2.state_dict())
        o2.close()
        assert all(st["qsgd_step"] == 2 for st in sd_opt["state"].values())
        m3, o3 = make()
        with torch.no_grad():
            for k, v in m3.state_dict().items():
                v.copy_(sd_model[k])
        o3.load_state_dict(sd_opt)
        assert o3._engine._qsgd_step == 2
        run(m3, o3, 2, 2)
        got = [p.detach().clone() for p in m3.parameters()]
        o3.close()
        return want, got

    for want, got in run_ranks(emu, 2, rank_main):
        for a, b in zip(want, got):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def host_two_ranks(rank, size):
    """One process of ``test_host_engine_two_ranks``."""
    from pytorch_ps_mpi_b200 import runtime
    w = runtime.init()
    assert (w.rank, w.size) == (rank, size)
    g = torch.from_numpy(np.random.default_rng(0).standard_normal(2 * TILE + 5).astype(np.float32))
    code = ps.QSGD(levels=7, seed=1, blockwise=True)
    wires = w.all_gather_object(code.encode(g, name="w")["wire"])
    assert not torch.equal(wires[0], wires[1])                         # each rank draws its own noise
    steps, total = 256, torch.zeros_like(g, dtype=torch.float64)
    for _ in range(steps):
        total += code.decode(code.encode(g, name="w")).double()
    scale = float(code.encode(g, name="w")["wire"][0, -16:-12].view(torch.float32))
    assert float((total / steps - g.double()).abs().max()) < 5 * scale * 0.5 / math.sqrt(steps)
    # one host-engine step, PS mode: the server applies both ranks' coded gradients (rank, call counter, crc32 of the name)
    torch.manual_seed(0)
    p = torch.nn.Parameter(torch.zeros(3000))
    opt = ps.SGD([("p", p)], [p], engine="host", mode="ps", lr=1.0, code=ps.QSGD(levels=8, seed=4, blockwise=True))
    gr = torch.randn(3000, generator=torch.Generator().manual_seed(10 + rank))
    (p * gr).sum().backward()
    opt.step()
    allg = w.all_gather_object(gr)
    want = -sum(ps.QSGD(levels=8, seed=4, blockwise=True).decode(
        ps.QSGD(levels=8, seed=4, blockwise=True).encode(allg[r], step=0, rank=r, first_tile=zlib.crc32(b"p"))) for r in range(2))
    assert torch.allclose(p.detach(), want, rtol=1e-6, atol=1e-6)
    opt.close()
    w.barrier()


def test_host_engine_two_ranks():
    from pytorch_ps_mpi_b200.launch import spawn
    spawn(host_two_ranks, 2, env={"PSB200_TRANSPORT": "shm"}, timeout=240)


# ---------------------------------------------------------------------------------------------------------------------
# 5. the device engine on one GPU, two ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_two_engine_ranks_one_gpu():
    from pytorch_ps_mpi_b200.launch import spawn
    from tests.test_gpu_engine import ONE_GPU
    spawn(gpu_two_ranks, 2, env=ONE_GPU, timeout=240)


def gpu_two_ranks(rank, size):
    """One process of ``test_two_engine_ranks_one_gpu``: ``engine='device'`` on bf16 parameters with QSGD(levels=7): 1040-byte
    wire tiles; three steps against the gathered-gradient oracle; ranks bit-identical."""
    from pytorch_ps_mpi_b200 import runtime
    w = runtime.init()
    dev = w.device
    torch.manual_seed(0)
    shapes = [(3000,), (40, 70)]
    params = [torch.nn.Parameter(torch.randn(s).to(torch.bfloat16).to(dev)) for s in shapes]
    w0 = [p.detach().float().cpu().clone() for p in params]
    code = ps.QSGD(levels=7, seed=8, blockwise=True)
    opt = ps.SGD([(f"p{i}", p) for i, p in enumerate(params)], params, engine="device", mode="ps", lr=0.1, code=code)
    eng = opt._engine
    assert eng is not None and eng.kind == KIND_QSGD and eng.wire_arena.numel() == 1040 * eng.layout.ntiles
    first = [eng.layout.by_id[id(p)].first_tile for p in params]
    want = [x.clone() for x in w0]
    for s in range(3):
        gs = [torch.randn(sh, generator=torch.Generator().manual_seed(100 * s + rank)).to(torch.bfloat16) for sh in shapes]
        opt.zero_grad(set_to_none=True)
        sum((p.float() * g.to(dev).float()).sum() for p, g in zip(params, gs)).backward()
        opt.step()
        allg = w.all_gather_object(gs)
        for i in range(len(params)):
            tot = sum(code.decode(code.encode(allg[r][i], step=s, rank=r, first_tile=first[i])).float() for r in range(size))
            want[i] -= 0.1 * tot.reshape(shapes[i])
    eng.check()
    torch.cuda.synchronize()
    master = [opt.state[p]["master_param"].detach().cpu().clone() for p in params] if eng.is_server else None
    res = w.all_gather_object((master, [p.detach().cpu().clone() for p in params]))
    opt.close()
    if rank == 0:
        for a, b in zip(res[0][1], res[1][1]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        for g, q in zip(res[0][0], want):
            assert torch.allclose(g, q, rtol=1e-5, atol=1e-5), float((g - q).abs().max())
    w.barrier()
