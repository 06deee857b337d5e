"""Gradient wires at their edges, bit for bit: rounding ties, subnormals, saturation, +-0, +-Inf and NaN.

Every wire format is decoded from its bit fields in numpy float64 (all 256 fp8 codes, all 65536 fp16 / bf16 codes), and the
rules of ``DESIGN.md`` (wire numerics) are applied by nearest-value search with ties to the even code.  Nothing in this
reference goes through a torch cast.  Against it:

* the encode kernels (``psb_absmax_kernel`` + ``psb_encode_kernel``): every dense and scaled coding x gradient dtype, wire bytes
  and per-parameter scales;
* the decode + rank-ordered sum + SGD + publication of ``psb_update_kernel`` at 1, 2, 5 and 16 ranks (16 = ``PSB_MAX_RANKS``),
  fp32 / bf16 / fp16 parameters;
* the block-wise top-k with NaN, +-Inf, -0, long runs of equal magnitudes, all-zero and partial tiles at 16 ranks;
* the ``codings.py`` oracle itself (CPU);
* two ranks of the real engine with a NaN and an Inf in one rank's gradient.

Each kernel test runs on the GPU (``-m gpu``, the ``Virtual`` harness of ``test_gpu_kernels.py``) and on the CPU emulator of
the same kernel source (``VirtualCPU``), which joins the default CPU run."""
import numpy as np
import pytest
import torch

import pytorch_ps_mpi_b200 as ps
from pytorch_ps_mpi_b200.codings import (KIND_SCALED, TILE, WIRE_BF16, WIRE_E4M3, WIRE_E5M2, WIRE_F16, WIRE_F32, WIRE_I8,
                                         tile_k)
from tests import _cuda_emu
from tests.test_multirank_engine_emulation import _attach, emu, run_ranks  # noqa: F401  (emu: fixture)

# ---------------------------------------------------------------------------------------------------------------------
# the reference: wire formats from their bit fields, rules 1-6 of DESIGN.md (wire numerics)
# ---------------------------------------------------------------------------------------------------------------------
_FORMATS = {WIRE_F16: (16, 5, 10, True), WIRE_BF16: (16, 8, 7, True), WIRE_E4M3: (8, 4, 3, False), WIRE_E5M2: (8, 5, 2, True)}
QMAX = {WIRE_I8: 127.0, WIRE_E4M3: 448.0, WIRE_E5M2: 57344.0, WIRE_F16: 65504.0}
NBITS = {WIRE_F32: 32, WIRE_BF16: 16, WIRE_F16: 16, WIRE_E4M3: 8, WIRE_E5M2: 8, WIRE_I8: 8}
GDT = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
GWIRE = {"fp32": WIRE_F32, "bf16": WIRE_BF16, "fp16": WIRE_F16}


def _float_table(nbits, ebits, mbits, ieee):
    """float64 value of every code of a binary float format (e4m3fn: no Inf, only S.1111.111 is NaN)."""
    c = np.arange(1 << nbits, dtype=np.int64)
    sign, exp, man = (c >> (nbits - 1)) & 1, (c >> mbits) & ((1 << ebits) - 1), c & ((1 << mbits) - 1)
    bias = (1 << (ebits - 1)) - 1
    mag = np.where(exp == 0, np.ldexp(man.astype(np.float64), 1 - bias - mbits),
                   np.ldexp((man + (1 << mbits)).astype(np.float64), exp - bias - mbits))
    top = exp == (1 << ebits) - 1
    if ieee:
        mag = np.where(top, np.where(man == 0, np.inf, np.nan), mag)
    else:
        mag = np.where(top & (man == (1 << mbits) - 1), np.nan, mag)
    return np.where(sign == 1, -mag, mag)


TABLE = {w: _float_table(*f) for w, f in _FORMATS.items()}


def ref_value(codes, wire):
    """float64 value of wire codes (int8: -128 is NaN)."""
    codes = np.asarray(codes, np.int64)
    if wire == WIRE_F32:
        return codes.astype(np.uint32).view(np.float32).astype(np.float64)
    if wire == WIRE_I8:
        v = ((codes + 128) % 256 - 128).astype(np.float64)
        return np.where(v == -128, np.nan, v)
    return TABLE[wire][codes]


def ref_cast(x, wire, saturate):
    """Codes of float64 values ``x`` cast to ``wire``: round to nearest, ties to the even code; ``saturate`` clamps finite
    values and +-Inf at +-max finite, otherwise values past max + 1/2 ulp become Inf.  NaN positions get code 0 and are
    returned as a mask (any NaN code is acceptable there)."""
    x = np.asarray(x, np.float64)
    nan = np.isnan(x)
    x0 = np.where(nan, 0.0, x)
    if wire == WIRE_I8:
        return np.where(nan, 0, np.clip(np.rint(x0), -127, 127).astype(np.int64) & 0xff), nan
    if wire == WIRE_F32:
        return x0.astype(np.float32).view(np.uint32).astype(np.int64), nan
    half = 1 << (NBITS[wire] - 1)
    pos = TABLE[wire][:half]                              # +0 ... +max finite (, +Inf), then the NaNs
    top = int(np.flatnonzero(np.isfinite(pos))[-1])
    vals = pos[:top + 1]
    a = np.abs(x0)
    if saturate:
        a = np.minimum(a, vals[top])
    else:
        assert np.isinf(pos[top + 1])                     # IEEE formats: Inf is the code after max finite, at max + 1 ulp
        vals = np.append(vals, 2 * vals[top] - vals[top - 1])
        a = np.minimum(a, vals[-1])
    hi = np.clip(np.searchsorted(vals, a), 0, len(vals) - 1)   # vals[hi - 1] < a <= vals[hi]
    lo = np.maximum(hi - 1, 0)
    mid = (vals[lo] + vals[hi]) / 2                       # exact: neighbouring codes of a <= 11-bit format
    code = np.where(a < mid, lo, np.where(a > mid, hi, np.where(hi % 2 == 0, hi, lo)))
    code = np.where(a == vals[hi], hi, code)
    return np.where(np.signbit(x0), code | half, code), nan


def narrows(gname, wire):
    """Does the cast of a ``gname`` gradient onto ``wire`` narrow it (then fp16 / fp8 wires saturate)?"""
    return wire in (WIRE_F16, WIRE_E4M3, WIRE_E5M2) and not (gname == "fp16" and wire == WIRE_F16)


def ref_encode(g, code, gname):
    """(codes, nan mask, fp32 scale or None) of one parameter's gradient ``g`` (float64 values of the gradient dtype)."""
    spec = code.device_spec()
    wire = spec.resolved_wire(GDT[gname])
    if spec.kind != KIND_SCALED:
        return (*ref_cast(g, wire, narrows(gname, wire)), None)
    g32 = g.astype(np.float32)
    fin = np.isfinite(g32)
    amax = np.float32(np.abs(g32[fin]).max()) if fin.any() else np.float32(0)
    amax = amax if amax > 0 else np.float32(1)
    inv = amax / np.float32(QMAX[wire])                   # IEEE fp32 division
    with np.errstate(over="ignore", invalid="ignore"):
        q = (g32 / inv).astype(np.float64)
    return (*ref_cast(q, wire, True), inv)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
NP_DT = {"fp32": np.float32, "fp16": np.float16}


def all_patterns(gname):
    """Every bit pattern of a 16-bit gradient dtype, as float64."""
    bits = np.arange(1 << 16, dtype=np.int64)
    return ref_value(bits, GWIRE[gname])


def _grid(wire):
    """Every finite value of ``wire`` (every int8 level) and the midpoint of each pair of neighbours."""
    v = np.arange(-127.0, 128.0) if wire == WIRE_I8 else np.unique(TABLE[wire][np.isfinite(TABLE[wire])])
    return v, (v[:-1] + v[1:]) / 2


def _with_ulps(x, gname):
    """``x`` in the gradient dtype and its neighbours one ulp either side."""
    t = NP_DT[gname]
    with np.errstate(over="ignore"):
        y = x.astype(t)
    return np.concatenate([y, np.nextafter(y, t(np.inf)), np.nextafter(y, t(-np.inf))]).astype(np.float64)


def _specials(gname):
    f = np.finfo(NP_DT[gname])
    sub = float(f.smallest_subnormal)
    return np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, float(f.max), -float(f.max), sub, -sub, 3 * sub, -2 * sub,
                     float(f.tiny), -float(f.tiny), float(f.tiny) - sub, -(float(f.tiny) - sub)])


def edge_grad(gname, wire, scaled):
    """The edge inputs of one (gradient dtype, wire) pair.  Scaled wires get amax = qmax (scale 1), so the scaled values are
    the inputs themselves: every level, every midpoint, +-1 ulp, the gradient dtype's subnormals, +-0, +-Inf and NaN."""
    if gname == "bf16" or (gname == "fp16" and wire in (WIRE_F16, WIRE_F32, WIRE_BF16)):
        return all_patterns(gname)
    if gname == "fp32" and wire == WIRE_F32:
        return np.concatenate([all_patterns("bf16"), _specials("fp32")])
    v, mids = _grid(wire)
    parts = [v, _with_ulps(mids, gname)]
    if not scaled:                                      # max finite + 1/2 ulp and its neighbours, values far past saturation
        top = v[-1] + (v[-1] - v[-2]) / 2
        parts += [_with_ulps(np.array([top, -top]), gname), np.array([v[-1] * 4, -v[-1] * 1024])]
    x = np.concatenate(parts + [_specials(gname)])
    if scaled:
        x = x[~(np.abs(x) > QMAX[wire]) | np.isinf(x)]          # keep amax = qmax
    with np.errstate(over="ignore"):
        return x.astype(NP_DT[gname]).astype(np.float64)


def wild_grad(gname, n, rng, big=True):
    """A second parameter: randn x 1e3 with the dtype's extremes, subnormals, +-Inf and NaN (its own amax and scale)."""
    x = rng.standard_normal(n) * 1e3
    s = _specials(gname if gname != "bf16" else "fp32")
    if not big:
        s = s[~(np.abs(s) > 1e30) | np.isinf(s)]
    x[rng.choice(n, len(s), replace=False)] = s
    with np.errstate(over="ignore"):
        return torch.tensor(x).to(GDT[gname]).double().numpy() if gname == "bf16" else x.astype(NP_DT[gname]).astype(np.float64)


def _layout(x, rng):
    """A fixed shuffle, padded so that the last tile is partial."""
    x = x[rng.permutation(len(x))]
    if len(x) % TILE == 0:
        x = np.append(x, [0.0] * 37)
    return x


def to_torch(x, gname):
    """float64 values of the gradient dtype → an exact torch tensor of that dtype (NaN and -0 kept)."""
    if gname == "bf16":
        bits = ref_cast(x, WIRE_BF16, False)[0]
        bits = np.where(np.isnan(x), 0x7fc0, bits)
        return torch.from_numpy(bits.astype(np.uint16).view(np.int16)).view(torch.bfloat16)
    return torch.from_numpy(x.astype(NP_DT[gname]))


# ---------------------------------------------------------------------------------------------------------------------
# back-ends: the GPU harness and the CPU emulator drive the same kernels through the same calls
# ---------------------------------------------------------------------------------------------------------------------
class Backend:
    def __init__(self, name):
        self.name = name
        if name == "emu":
            self.lib = _cuda_emu.build()
            if self.lib is None:
                pytest.skip("no g++")

    def make(self, shapes, dtype, code, nranks):
        if self.name == "gpu":
            from tests.test_gpu_kernels import Virtual
            return Virtual(shapes, dtype, code, nranks)
        from tests.test_ps_kernels_cpu_emulation import VirtualCPU
        return VirtualCPU(self.lib, shapes, dtype, code, nranks)

    def tensor(self, t):
        return t.cuda() if self.name == "gpu" else t

    def encode(self, V, r, grads):
        V.encode(r, [self.tensor(g) for g in grads])
        if self.name == "gpu":
            torch.cuda.synchronize()

    def update(self, V):
        V.update(1, [[1.0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1.0]])          # SGD, lr = 1, no momentum / weight decay

    @staticmethod
    def codes(V, r, slot, kind_bytes):
        """Wire codes of one parameter (int64), from its first tile on."""
        w = V.wires[r].cpu().numpy()
        esz = kind_bytes
        base = slot.first_tile * V.bpt
        raw = w[base: base + slot.ntiles * V.bpt].reshape(slot.ntiles, V.bpt)[:, :TILE * esz].reshape(-1)
        view = {1: np.uint8, 2: np.uint16, 4: np.uint32}[esz]
        return raw.view(view).astype(np.int64)


@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def be(request):
    return Backend(request.param)


@pytest.fixture(autouse=True)
def _single_threaded_torch():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


CODES = {
    "identity": lambda: ps.Identity(), "cast_fp32": lambda: ps.Cast("fp32"), "cast_bf16": lambda: ps.Cast("bf16"),
    "cast_fp16": lambda: ps.Cast("fp16"), "cast_e4m3": lambda: ps.Cast("fp8_e4m3"), "cast_e5m2": lambda: ps.Cast("fp8_e5m2"),
    "scale_i8": lambda: ps.Scale("int8"), "scale_e4m3": lambda: ps.Scale("fp8_e4m3"), "scale_e5m2": lambda: ps.Scale("fp8_e5m2"),
    "scale_f16": lambda: ps.Scale("fp16"),
}


def assert_codes(got, want, nan, wire, what):
    """Wire codes equal bit for bit; at NaN positions any NaN code."""
    got_nan = np.isnan(ref_value(got, wire))
    bad = np.flatnonzero(np.where(nan, ~got_nan, got != want))
    if len(bad):
        i = bad[:8]
        raise AssertionError(f"{what}: {len(bad)} codes differ, e.g. at {i.tolist()}: got {[hex(c) for c in got[i]]} "
                             f"want {[hex(c) for c in want[i]]} (nan expected {nan[i].tolist()})")


# ---------------------------------------------------------------------------------------------------------------------
# 0. the reference itself
# ---------------------------------------------------------------------------------------------------------------------
def test_reference_tables_decode_like_torch():
    """The bit-field tables agree with torch's decode of every code (decoding is not what is under test), and the reference
    cast reproduces each format's own codes (every finite / infinite value is its own nearest value)."""
    for wire, dt in ((WIRE_F16, torch.float16), (WIRE_BF16, torch.bfloat16), (WIRE_E4M3, torch.float8_e4m3fn),
                     (WIRE_E5M2, torch.float8_e5m2)):
        n = 1 << NBITS[wire]
        raw = torch.arange(n, dtype=torch.int32)
        t = (raw.to(torch.int16) if n > 256 else raw.to(torch.uint8)).view(dt).double().numpy()
        assert np.array_equal(t, TABLE[wire], equal_nan=True), wire
        codes = np.arange(n)
        ok = ~np.isnan(TABLE[wire])
        got, _ = ref_cast(TABLE[wire], wire, saturate=False if wire != WIRE_E4M3 else True)
        assert np.array_equal(got[ok], codes[ok]), wire
    # spot checks of rules 1-4 written out by hand
    assert ref_cast(np.array([2.5, 3.5, -2.5, np.inf, 200.0]), WIRE_I8, True)[0].tolist() == [2, 4, 0xfe, 127, 127]
    assert ref_cast(np.array([65520.0, 65519.99, np.inf]), WIRE_F16, False)[0].tolist() == [0x7c00, 0x7bff, 0x7c00]
    assert ref_cast(np.array([65520.0, np.inf, -np.inf]), WIRE_F16, True)[0].tolist() == [0x7bff, 0x7bff, 0xfbff]
    assert ref_cast(np.array([464.0, 480.0, 2.0 ** -10, 3 * 2.0 ** -10]), WIRE_E4M3, True)[0].tolist() == [0x7e, 0x7e, 0x00, 0x02]
    assert ref_cast(np.array([-0.0, 2.0 ** -150]), WIRE_F16, True)[0].tolist() == [0x8000, 0x0000]


# ---------------------------------------------------------------------------------------------------------------------
# 1. encode: wire bytes and scales
# ---------------------------------------------------------------------------------------------------------------------
def _encode_case(gname, cname):
    code = CODES[cname]()
    spec = code.device_spec()
    wire = spec.resolved_wire(GDT[gname])
    rng = np.random.default_rng(sum(map(ord, gname + cname)))
    a = _layout(edge_grad(gname, wire, spec.kind == KIND_SCALED), rng)
    b = wild_grad(gname, TILE + 301, rng)
    return code, wire, [a, b]


@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("cname", list(CODES))
def test_encode_wire_bits(be, gname, cname):
    code, wire, xs = _encode_case(gname, cname)
    V = be.make([(len(x),) for x in xs], GDT[gname], code, 1)
    be.encode(V, 0, [to_torch(x, gname) for x in xs])
    esz = NBITS[wire] // 8
    for i, (p, x) in enumerate(zip(V.params, xs)):
        slot = V.L.by_id[id(p)]
        got = Backend.codes(V, 0, slot, esz)
        want, nan, inv = ref_encode(x, code, gname)
        assert_codes(got[:len(x)], want, nan, wire, f"{be.name} {cname} {gname} param {i}")
        assert not got[len(x):].any(), "padding lanes of the last tile must encode 0"
        if inv is not None:
            s = np.float32(V.scales[0][slot.index].item())
            assert s.view(np.uint32) == inv.view(np.uint32), (float(s), float(inv))


@pytest.mark.parametrize("gname", ["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("cname", list(CODES))
def test_codings_oracle_matches_reference(gname, cname):
    """``codings.py`` (the host engine's encode / decode and every kernel test's oracle) follows the same table."""
    code, wire, xs = _encode_case(gname, cname)
    for x in xs:
        g = to_torch(x, gname)
        enc = code.encode(g)
        want, nan, inv = ref_encode(x, code, gname)
        payload = enc["grad"] if "grad" in enc else enc["v"] if "v" in enc else enc["q"]
        bits = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[NBITS[wire] // 8]
        got = payload.contiguous().view(bits).numpy().astype(np.int64) & ((1 << NBITS[wire]) - 1)
        assert_codes(got, want, nan, wire, f"codings {cname} {gname}")
        dec = code.decode(enc).double().numpy()
        val = ref_value(want, wire)
        if inv is not None:
            assert enc["inv"].numpy().view(np.uint32)[0] == inv.view(np.uint32)
            with np.errstate(over="ignore", invalid="ignore"):
                val = (val.astype(np.float32) * inv).astype(np.float64)
        assert np.array_equal(dec, np.where(nan, np.nan, val), equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------------
# 2. decode + rank-ordered sum + SGD + publication
# ---------------------------------------------------------------------------------------------------------------------
def _compact(gname, wire, scaled, rng, n=3 * TILE + 99):
    """``n`` edge inputs (a partial last tile): every special value of ``edge_grad`` and a random sample of the rest."""
    x = edge_grad(gname, wire, scaled)
    sp = np.flatnonzero(~np.isfinite(x) | (x == 0) | (np.abs(x) == np.abs(x[np.isfinite(x)]).max()))[:64]
    rest = rng.choice(len(x), n - len(sp), replace=len(x) < n - len(sp))
    return rng.permutation(np.concatenate([x[sp], x[rest]]))


def _ulp32(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


def check_update(be, V, grads, code, gname, what):
    """Master (zero before the step, SGD lr = 1) == -(fp32 sum of the decoded values in rank order); published parameter ==
    the master rounded to nearest even.  Scaled wires: the kernel may fuse each rank's ``f * scale`` into an FMA, so 1 ulp
    per rank against float64."""
    scaled = code.device_spec().kind == KIND_SCALED
    for i, p in enumerate(V.params):
        slot = V.L.by_id[id(p)]
        terms = []
        for r in range(V.n):
            c, nan, inv = ref_encode(grads[r][i], code, gname)
            wire = code.device_spec().resolved_wire(GDT[gname])
            d = np.where(nan, np.nan, ref_value(c, wire))
            terms.append(d * np.float64(inv) if scaled else d)
        if V.master is not None:
            got = V.master[slot.offset: slot.offset + slot.numel].cpu().numpy()
        else:
            got = V.param_arenas[0][slot.offset: slot.offset + slot.numel].cpu().numpy()
        if not scaled:
            acc = np.zeros(slot.numel, np.float32)
            with np.errstate(over="ignore", invalid="ignore"):
                for t in terms:
                    acc = acc + t.astype(np.float32)
            want = np.where(acc == 0, np.float32(0), -acc)
            same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
            bad = np.flatnonzero(~same)
            assert not len(bad), (what, i, bad[:5].tolist(), got[bad[:5]].tolist(), want[bad[:5]].tolist())
        else:
            with np.errstate(over="ignore", invalid="ignore"):
                part, bound, acc = np.zeros(slot.numel), np.zeros(slot.numel), np.zeros(slot.numel, np.float32)
                for t in terms:
                    part = part + t
                    bound += _ulp32(np.maximum(np.abs(part), np.abs(t)))
                    acc = acc + t.astype(np.float32)
            # NaN inputs, and sums past the fp32 range: the fp32 result (NaN, or Inf of the sign the fp32 sum reached)
            special = ~np.isfinite(part) | ~np.isfinite(acc)
            g, w = got[special], -acc[special]
            assert ((np.isnan(g) & np.isnan(w)) | (g == w)).all(), (what, i, "non-finite elements")
            err = np.abs(got[~special].astype(np.float64) + part[~special])
            assert (err <= bound[~special]).all(), (what, i, float((err - bound[~special]).max()))
        if V.dtype != torch.float32:
            pw = GWIRE["bf16" if V.dtype == torch.bfloat16 else "fp16"]
            want_pub, nan_pub = ref_cast(got.astype(np.float64), pw, saturate=False)
            for r in range(V.n):
                pub = V.param_arenas[r][slot.offset: slot.offset + slot.numel].cpu().view(torch.int16).numpy()
                assert_codes(pub.astype(np.int64) & 0xffff, want_pub, nan_pub, pw, f"{what} published, rank {r}")
        else:
            for r in range(1, V.n):
                assert torch.equal(V.param_arenas[r].view(torch.int32), V.param_arenas[0].view(torch.int32))


def _update_case(be, cname, gname, world, shapes_fn=None):
    code = CODES[cname]()
    spec = code.device_spec()
    wire = spec.resolved_wire(GDT[gname])
    rng = np.random.default_rng(world * 131 + sum(map(ord, gname + cname)))
    grads = []
    for r in range(world):
        if r % 3 == world % 2:                     # edge inputs on some ranks, moderate randn on the others
            a = _compact(gname, wire, spec.kind == KIND_SCALED, rng)
            b = wild_grad(gname, TILE + 5, rng, big=False)
        else:
            a = rng.standard_normal(3 * TILE + 99) * (1 + r)
            b = rng.standard_normal(TILE + 5)
        grads.append([to_torch(a, gname).double().numpy(), to_torch(b, gname).double().numpy()])
    V = be.make([(len(x),) for x in grads[0]], GDT[gname], code, world)
    for a in V.param_arenas:
        a.zero_()
    if V.master is not None:
        V.master.zero_()
    for r in range(world):
        be.encode(V, r, [to_torch(x, gname) for x in grads[r]])
    be.update(V)
    check_update(be, V, grads, code, gname, f"{be.name} {cname} {gname} x{world}")


_UPDATE_FULL = [(c, g, n) for c in CODES for g in ("fp32", "bf16", "fp16") for n in (1, 2, 5, 16)]
# the emulator runs one CTA after another: every coding and dtype once, each world size several times
_UPDATE_EMU = [(c, g, (1, 2, 5, 16)[(i + j) % 4]) for i, c in enumerate(CODES) for j, g in enumerate(("fp32", "bf16", "fp16"))]


@pytest.mark.parametrize("cname,gname,world", _UPDATE_EMU)
def test_decode_sum_publish_emulated(cname, gname, world):
    _update_case(Backend("emu"), cname, gname, world)


@pytest.mark.gpu
@pytest.mark.parametrize("cname,gname,world", _UPDATE_FULL)
def test_decode_sum_publish_gpu(cname, gname, world):
    _update_case(Backend("gpu"), cname, gname, world)


# ---------------------------------------------------------------------------------------------------------------------
# 3. block-wise top-k
# ---------------------------------------------------------------------------------------------------------------------
def topk_grad(rng, gname, n=3 * TILE + 700):
    """Tile 0: NaN, -NaN, +-Inf, -0 among randn; tile 1: long runs of equal magnitudes; tile 2: all zero; a partial tile 3."""
    x = rng.standard_normal(n)
    x[rng.choice(TILE, 12, replace=False)] = [np.nan, -np.nan, np.inf, -np.inf, np.inf, -0.0, -0.0, 0.0, 1e30, -1e30, 5e-45, -5e-45]
    run = rng.choice(TILE, 900, replace=False) + TILE
    x[run] = np.where(rng.random(900) < 0.5, -2.5, 2.5)
    x[run[:300]] = np.where(rng.random(300) < 0.5, -0.75, 0.75)
    x[2 * TILE: 3 * TILE] = 0.0
    x[3 * TILE + rng.choice(n - 3 * TILE, 40, replace=False)] = np.where(rng.random(40) < 0.5, -4.0, 4.0)
    x[3 * TILE + 5] = np.nan
    return to_torch(x if gname == "bf16" else x.astype(np.float32).astype(np.float64), gname).double().numpy()


def ref_topk(x, ratio):
    """(indices, fp32 values) per tile: magnitude keys = fp32 bits without the sign, descending, ties → lower index."""
    x32 = x.astype(np.float32)
    key = (x32.view(np.uint32) & 0x7fffffff).astype(np.int64)
    out = []
    for t in range((len(x) + TILE - 1) // TILE):
        lo, hi = t * TILE, min(len(x), (t + 1) * TILE)
        k = tile_k(ratio, hi - lo)
        order = np.argsort(-key[lo:hi], kind="stable")[:k]
        sel = np.sort(order)
        out.append((sel, x32[lo + sel]))
    return out


def _topk_case(be, values, gname, ratio, world=16):
    code = ps.TopK(ratio=ratio, values=values)
    rng = np.random.default_rng(int(ratio * 4096) + (values == "bf16") * 7 + (gname == "bf16") * 3)
    grads = [topk_grad(rng, gname) for _ in range(world)]
    V = be.make([(len(grads[0]),)], GDT[gname], code, world)
    for a in V.param_arenas:
        a.zero_()
    if V.master is not None:
        V.master.zero_()
    acc = np.zeros(len(grads[0]), np.float32)
    for r in range(world):
        be.encode(V, r, [to_torch(grads[r], gname)])
        w = V.wires[r].cpu().numpy()[: V.L.ntiles * V.bpt].reshape(V.L.ntiles, V.bpt)
        for t, (sel, val) in enumerate(ref_topk(grads[r], ratio)):
            if values == "bf16":
                e = w[t].view(np.uint32)[: V.cap].astype(np.int64)
                idx, bits = e >> 16, e & 0xffff
                want, nan = ref_cast(val.astype(np.float64), WIRE_BF16, False)
                dec = ref_value(want, WIRE_BF16)
            else:
                e = w[t].view(np.uint32)[: 2 * V.cap].reshape(-1, 2).astype(np.int64)
                idx, bits = e[:, 0], e[:, 1]
                want, nan = ref_cast(val.astype(np.float64), WIRE_F32, False)
                dec = val.astype(np.float64)
            k = len(sel)
            assert np.array_equal(idx[:k], sel), (be.name, ratio, r, t)
            assert (idx[k:] == TILE).all(), "unused entries must carry the no-entry index"
            assert_codes(bits[:k], want, nan, WIRE_BF16 if values == "bf16" else WIRE_F32, f"topk r{r} t{t}")
            with np.errstate(invalid="ignore"):
                acc[t * TILE + sel] += np.where(nan, np.nan, dec).astype(np.float32)
    be.update(V)
    got = (V.master if V.master is not None else V.param_arenas[0])[: len(acc)].cpu().numpy()
    want = np.where(acc == 0, np.float32(0), -acc)
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), (be.name, np.flatnonzero(~same)[:5].tolist())


_TOPK = [(v, g, r) for v in ("fp32", "bf16") for g in ("fp32", "bf16") for r in (1 / 2048, 0.05, 1.0)]
_TOPK_EMU = [("fp32", "fp32", 1 / 2048), ("bf16", "fp32", 0.05), ("fp32", "bf16", 1.0), ("bf16", "bf16", 1 / 2048)]


@pytest.mark.parametrize("values,gname,ratio", _TOPK_EMU)
def test_topk_edges_emulated(values, gname, ratio):
    _topk_case(Backend("emu"), values, gname, ratio, world=4 if ratio == 1.0 else 16)


@pytest.mark.gpu
@pytest.mark.parametrize("values,gname,ratio", _TOPK)
def test_topk_edges_gpu(values, gname, ratio):
    _topk_case(Backend("gpu"), values, gname, ratio)


# ---------------------------------------------------------------------------------------------------------------------
# 4. one arena of more than 3 x 132 tiles on the GPU: the update kernel's grid-stride loop against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cname,gname", [("identity", "bf16"), ("scale_i8", "fp32"), ("topk", "fp32")])
def test_grid_stride_arena_gpu(cname, gname):
    be = Backend("gpu")
    code = ps.TopK(ratio=0.05) if cname == "topk" else CODES[cname]()
    rng = np.random.default_rng(11)
    n = 450 * TILE + 123
    grads = []
    for r in range(2):
        x = rng.standard_normal(n) * (1 + r)
        x[rng.choice(n, 6, replace=False)] = [np.nan, np.inf, -np.inf, -0.0, 1e-42, 3e4]
        grads.append([to_torch(x, gname).double().numpy(), to_torch(rng.standard_normal(700), gname).double().numpy()])
    V = be.make([(n,), (700,)], GDT[gname], code, 2)
    assert V.L.ntiles > 3 * 132 and V.P.grid < V.L.ntiles
    for a in V.param_arenas:
        a.zero_()
    if V.master is not None:
        V.master.zero_()
    for r in range(2):
        be.encode(V, r, [to_torch(x, gname) for x in grads[r]])
    be.update(V)
    if cname != "topk":
        check_update(be, V, grads, code, gname, f"gpu grid-stride {cname}")
        return
    for i, p in enumerate(V.params):
        slot = V.L.by_id[id(p)]
        acc = np.zeros(slot.numel, np.float32)
        for r in range(2):
            for t, (sel, val) in enumerate(ref_topk(grads[r][i], 0.05)):
                acc[t * TILE + sel] += val
        got = V.param_arenas[0][slot.offset: slot.offset + slot.numel].cpu().numpy()
        want = np.where(acc == 0, np.float32(0), -acc)
        assert ((got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))).all()


# ---------------------------------------------------------------------------------------------------------------------
# 5. end to end: two ranks of the engine, a NaN and an Inf in rank 1's gradient, fp16 parameters
# ---------------------------------------------------------------------------------------------------------------------
E2E_CODES = {"cast_fp16": lambda: ps.Cast("fp16"), "scale_i8": lambda: ps.Scale("int8"), "identity": lambda: ps.Identity()}
NAN_AT, INF_AT = 3, 70


def e2e_grads(rank, shapes):
    """The gradient each rank's parameters receive (``loss = sum(p * c)``): fp16 randn; rank 1 holds a NaN and a +Inf."""
    g = torch.Generator().manual_seed(100 + rank)
    cs = [torch.randn(s, generator=g).to(torch.float16) for s in shapes]
    if rank == 1:
        cs[0].view(-1)[NAN_AT] = float("nan")
        cs[0].view(-1)[INF_AT] = float("inf")
    return cs


def e2e_check(coding, w0, got_master, pubs, lr):
    """Both ranks: NaN at the NaN element; at the Inf element -Inf (lossless fp16 wires) or the finite step of the saturated
    code (int8: Inf → +127 → +amax); everywhere else the host engine's result (``codings.py`` oracle + fp32 SGD), and the
    published parameters == the master rounded, identical on both ranks."""
    factory = E2E_CODES[coding]
    shapes = [w.shape for w in w0]
    total = [torch.zeros(s) for s in shapes]
    for r in range(2):
        for i, c in enumerate(e2e_grads(r, shapes)):
            code = factory()
            total[i] += code.decode(code.encode(c, name=f"p{i}")).reshape(shapes[i]).float()
    want = [w.float() - lr * t for w, t in zip(w0, total)]
    for pub in pubs:
        for a, b in zip(pub, pubs[0]):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        f = pub[0].float().view(-1)
        assert torch.isnan(f[NAN_AT])
        assert bool(torch.isfinite(f[INF_AT])) if coding == "scale_i8" else float(f[INF_AT]) == float("-inf")
    for i, (g, w) in enumerate(zip(got_master, want)):
        g, w = g.float().reshape(-1), w.reshape(-1)
        fin = torch.isfinite(w)
        assert torch.equal(torch.isnan(g), torch.isnan(w)) and torch.equal(torch.isinf(g), torch.isinf(w)), i
        assert torch.equal(g[torch.isinf(w)], w[torch.isinf(w)])
        assert torch.allclose(g[fin], w[fin], rtol=1e-5, atol=1e-6), (coding, i, float((g[fin] - w[fin]).abs().max()))
        pub, nan = pubs[0][i].reshape(-1), torch.isnan(g)
        assert torch.equal(torch.isnan(pub), nan)
        assert torch.equal(g.to(torch.float16)[~nan].view(torch.int16), pub[~nan].view(torch.int16))


def e2e_params():
    g = torch.Generator().manual_seed(0)
    return [torch.nn.Parameter(torch.randn(s, generator=g).to(torch.float16)) for s in E2E_SHAPES]


E2E_SHAPES = [(3000,), (40, 30)]


@pytest.mark.parametrize("emu", ["shim"], indirect=True)
@pytest.mark.parametrize("coding", list(E2E_CODES))
def test_nan_inf_two_ranks_emulated(emu, coding):
    lr = 0.5

    def rank_main(rank, w):
        params = e2e_params()
        w0 = [p.detach().clone() for p in params]
        opt = ps.SGD([(f"p{i}", p) for i, p in enumerate(params)], params, engine="host", mode="ps", code=E2E_CODES[coding](),
                     lr=lr)
        _attach(opt)
        eng = opt._engine
        opt.zero_grad(set_to_none=True)
        sum((p.float() * c.float()).sum() for p, c in zip(params, e2e_grads(rank, E2E_SHAPES))).backward()
        opt.step()
        eng.check()
        w.barrier()
        master = [opt.state[p]["master_param"].detach().clone() for p in params] if eng.is_server else None
        pub = [p.detach().clone() for p in params]
        opt.close()
        return w0, master, pub

    res = run_ranks(emu, 2, rank_main)
    masters = [m for _, m, _ in res if m is not None]
    assert len(masters) == 1
    e2e_check(coding, res[0][0], masters[0], [pub for _, _, pub in res], lr)


@pytest.mark.gpu
def test_nan_inf_two_ranks_one_gpu():
    """The same three codings on the device engine, two processes sharing one GPU (one spawn: process start-up dominates)."""
    from pytorch_ps_mpi_b200.launch import spawn
    from tests.test_gpu_engine import ONE_GPU
    spawn(gpu_wire_edges, 2, (tuple(E2E_CODES),), env=ONE_GPU, timeout=240)


def gpu_wire_edges(rank, size, codings):
    """One process of ``test_nan_inf_two_ranks_one_gpu``: the device engine on fp16 parameters, rank 1's gradient holding a
    NaN and an Inf, one engine per coding, checked by ``e2e_check`` on rank 0."""
    from pytorch_ps_mpi_b200 import runtime
    w = runtime.init()
    assert (w.rank, w.size) == (rank, size)
    dev = w.device
    lr = 0.5
    for coding in codings:
        params = [torch.nn.Parameter(p.detach().to(dev)) for p in e2e_params()]
        w0 = [p.detach().cpu().clone() for p in params]
        opt = ps.SGD([(f"p{i}", p) for i, p in enumerate(params)], params, engine="device", mode="ps", code=E2E_CODES[coding](),
                     lr=lr)
        eng = opt._engine
        assert eng is not None and (eng.master is not None or not eng.is_server)
        opt.zero_grad(set_to_none=True)
        sum((p.float() * c.to(dev).float()).sum() for p, c in zip(params, e2e_grads(rank, E2E_SHAPES))).backward()
        opt.step()
        eng.check()
        torch.cuda.synchronize()
        master = [opt.state[p]["master_param"].detach().cpu().clone() for p in params] if eng.is_server else None
        res = w.all_gather_object((master, [p.detach().cpu().clone() for p in params]))
        opt.close()
        if rank == 0:
            masters = [m for m, _ in res if m is not None]
            assert len(masters) == 1
            e2e_check(coding, w0, masters[0], [pub for _, pub in res], lr)
        w.barrier()
