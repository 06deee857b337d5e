"""Exact references and bit-level comparators for the tensor-core kernels: ``psb_bcast_gemm_kernel``,
``psb_stem_fwd_kernel`` (with its BatchNorm sums) and ``psb_stem_wgrad_kernel`` + its finalize.

Shared by the H100 tests (``test_gpu_gemm.py``, ``test_gpu_fused_ops.py``) and the CPU tests of the emulated stand-ins
(``test_wgmma_oracle.py``).  Every reference is computed in float64 from the operation's definition, never from a
repository kernel.

Exact data: entries in {-1, 0, +1} times a power of two per row of ``x`` and per output channel of ``w`` (of ``gy`` for
the weight gradient).  All products that meet in one output element then share one scale, so every partial sum is an
integer multiple of that power of two, bounded by the number of terms.  While that bound stays below 2^24 the fp32
accumulation is exact in any order, and below 2^13 it stays exact even for an adder that keeps only 13 bits of alignment.
The float64 reference is then the kernel's exact answer before its final roundings, which :func:`gemm_expected`
reproduces in the kernel's order: fp32 + fp32 bias (one IEEE add), ReLU, bf16 round-to-nearest-even.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

GEMM_MAX_K = 4096          # K terms of magnitude <= 1 (times the shared scale): every partial sum stays below 2^13
STEM_TAPS = 147            # 3 x 7 x 7 products per forward output


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _ternary(shape, g, dim=0):
    """Entries in {-1, 0, +1}; about half the slices along ``dim`` lean to +1, so that the sums where two such slices
    meet grow with the number of terms and need more than bf16's 8 bits: the output rounding is then exercised."""
    t = torch.randint(-1, 2, shape, generator=g)
    lean = torch.rand(shape[dim], generator=g) < 0.5
    lean = lean.view([-1 if d == dim else 1 for d in range(len(shape))])
    up = torch.rand(shape, generator=g) < 0.75
    return torch.where(lean & up, torch.ones_like(t), t).double()


def _pow2(n, g, lo=-3, hi=3):
    return torch.exp2(torch.randint(lo, hi + 1, (n,), generator=g).double())


def exact_gemm_operands(M, N, K, seed=0, device="cpu"):
    """bf16 ``x [M,K]``, ``w [N,K]`` whose fp32 products and sums are exact (see the module docstring)."""
    assert K <= GEMM_MAX_K, f"K={K}: partial sums could reach 2^13"
    g = _gen(seed)
    x = _ternary((M, K), g) * _pow2(M, g)[:, None]
    w = _ternary((N, K), g) * _pow2(N, g)[:, None]
    return x.bfloat16().to(device), w.bfloat16().to(device)


def exact_stem_input(n, h, w, seed=0, device="cpu"):
    """bf16 channels-last image ``[n,3,h,w]`` for the forward: ternary times a power of two per image, so the 147
    products of one output share one scale with an output channel of :func:`exact_stem_weight`."""
    g = _gen(seed)
    x = _ternary((n, 3, h, w), g) * _pow2(n, g)[:, None, None, None]
    return x.bfloat16().to(device).contiguous(memory_format=torch.channels_last)


def exact_stem_weight(seed=0, device="cpu"):
    """bf16 ``[64,3,7,7]``: ternary times a power of two per output channel."""
    g = _gen(seed)
    return (_ternary((64, 3, 7, 7), g) * _pow2(64, g)[:, None, None, None]).bfloat16().to(device)


def exact_wgrad_operands(n, h, w, seed=0, device="cpu"):
    """bf16 channels-last ``x [n,3,h,w]`` (ternary times a power of two per input channel) and ``gy [n,64,oh,ow]``
    (ternary times a power of two per output channel): each dW element is a sum of n*oh*ow products of one scale."""
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    assert n * oh * ow < 2 ** 24, "weight-gradient sums could leave the 24 bits of fp32"
    g = _gen(seed)
    x = _ternary((n, 3, h, w), g, 1) * _pow2(3, g)[None, :, None, None]
    gy = _ternary((n, 64, oh, ow), g, 1) * _pow2(64, g)[None, :, None, None]
    cl = torch.channels_last
    return x.bfloat16().to(device).contiguous(memory_format=cl), gy.bfloat16().to(device).contiguous(memory_format=cl)


# ------------------------------------------------------------------ references (float64, from the definitions)
def gemm_ref64(x, w, bias=None):
    ref = x.double() @ w.double().t()
    return ref if bias is None else ref + bias.double()


def gemm_expected(x, w, bias=None, relu=False):
    """The kernel's output on exact data: the exact product rounded as the epilogue rounds it."""
    acc = (x.double() @ w.double().t()).float()        # exact: the fp32 accumulator holds it
    if bias is not None:
        acc = acc + bias.float()                        # one IEEE fp32 add
    if relu:
        acc = torch.relu(acc)                           # F.relu: NaN stays NaN
    return acc.bfloat16()


def stem_fwd_ref64(x, weight):
    """``F.conv2d(x, weight, stride=2, padding=3)`` in float64, ``[n,64,oh,ow]``."""
    return F.conv2d(x.double(), weight.double(), stride=2, padding=3)


def stem_wgrad_ref64(x, gy):
    """The stem's weight gradient in float64, in the kernel's [64,176] layout (``ops.stem._w2d``)."""
    from pytorch_ps_mpi_b200.ops.stem import _w2d
    dw = torch.nn.grad.conv2d_weight(x.double(), (gy.shape[1], 3, 7, 7), gy.double(), stride=2, padding=3)
    return _w2d(dw)


def stem_sums_replay(y, sms, quarters=4):
    """Σy | Σy² (fp32, 128 values) of the bf16 stem output ``y [n,64,oh,ow]`` in ``psb_stem_fwd_kernel``'s order.

    The grid is min(tiles, sms) CTAs over the n*oh output rows ("tiles"); CTA b takes tiles b*per .. b*per+per-1 with
    per = ceil(tiles / grid).  Each (CTA, row quarter, channel) chain adds its rows in tile order (fmaf(v, v, s) is an
    fp32 add: v*v of a bf16 value is exact in fp32); the quarters are added as ((q0 + q1) + q2) + q3; then
    ``psb_stem_sums_kernel`` adds the CTAs in order.  ``sms=1, quarters=1`` is a plain sum over the pixels in order."""
    n, c, oh, ow = y.shape
    assert c == 64
    tiles = n * oh
    grid = min(tiles, sms)
    per = -(-tiles // grid)
    rq = -(-ow // quarters)
    rows = torch.zeros(grid * per, quarters * rq, 64, dtype=torch.float32, device=y.device)
    rows[:tiles, :ow] = y.permute(0, 2, 3, 1).reshape(tiles, ow, 64).float()   # zero rows: x + 0 == x in fp32
    chains = rows.view(grid, per, quarters, rq, 64).permute(0, 2, 4, 1, 3).reshape(grid, quarters, 64, per * rq)
    chains = chains.contiguous()
    sq = chains * chains
    s = torch.zeros(grid, quarters, 64, dtype=torch.float32, device=y.device)
    s2 = torch.zeros_like(s)
    for i in range(per * rq):
        s = s + chains[..., i]
        s2 = s2 + sq[..., i]
    part = torch.cat([s, s2], dim=2)                   # [grid, quarters, 128]
    q = part[:, 0]
    for k in range(1, quarters):
        q = q + part[:, k]
    out = torch.zeros(128, dtype=torch.float32, device=y.device)
    for b in range(grid):
        out = out + q[b]
    return out


# ------------------------------------------------------------------ comparators
def _canon_bits(t):
    """Integer bits with +0 == -0 and every NaN alike."""
    bits = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32,
            torch.float64: torch.int64}[t.dtype]
    b = t.contiguous().view(bits).long()
    b = torch.where(t.contiguous() == 0, torch.zeros_like(b), b)
    return torch.where(torch.isnan(t.contiguous()), torch.full_like(b, -1), b)


def assert_bits_equal(y, ref, tile=None, what=""):
    """The bits of ``y`` and ``ref`` (same dtype and shape) agree, except that +0 equals -0 and any NaN equals any NaN.
    ``tile``: the output tile shape over the last dims, named in the failure message with the first differing index."""
    assert y.dtype == ref.dtype and y.shape == ref.shape, (y.dtype, ref.dtype, y.shape, ref.shape)
    diff = _canon_bits(y) != _canon_bits(ref)
    if bool(diff.any()):
        flat = int(diff.reshape(-1).nonzero()[0])
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), y.shape))
        msg = (f"{what}: {int(diff.sum())} of {diff.numel()} elements differ; first at {idx}: "
               f"got {y[idx].item()!r}, want {ref[idx].item()!r}")
        if tile is not None:
            msg += f", in output tile {tuple(i // t for i, t in zip(idx[-len(tile):], tile))} of shape {tuple(tile)}"
        raise AssertionError(msg)


def bf16_ulp(v):
    """One bf16 ulp at |v| (8 significant bits; the smallest subnormal step below the normal range)."""
    a = v.double().abs()
    _, e = torch.frexp(a)
    return torch.where(a == 0, torch.full_like(a, 2.0 ** -133), torch.exp2((e - 8).clamp(min=-133).double()))


def assert_within_ulp(y, ref64, terms_abs, c, what=""):
    """Random data: every element of the bf16 ``y`` lies within one bf16 ulp of the float64 ``ref64``, plus
    ``c * 2^-24 * terms_abs``, where ``terms_abs`` is Σ|x_k w_k| (+ |bias|) of that element and ``c`` is the number of
    fp32 additions on the longest path from a product to the output.

    Derivation: each fp32 addition rounds its result, whose magnitude never exceeds Σ|x_k w_k|, by at most half an ulp of
    fp32, i.e. 2^-24 of that magnitude; ``c`` such roundings in a chain move the fp32 result at most
    c * 2^-24 * Σ|x_k w_k| from the exact sum (to first order).  The final bf16 round-to-nearest adds at most half a bf16
    ulp of the fp32 value, and one ulp at the exact value covers that even where the two straddle a power of two.
    For the GEMM c = K/16 (one add per wgmma k-step of 16) + 1 for the bias; for the stem forward c = 176/16; for the
    weight gradient c = (pixels per CTA)/16 + grid (the finalize adds the CTA partials in order).

    Returns the fraction of elements equal to bf16_rn(ref64)."""
    y64 = y.double()
    bound = bf16_ulp(ref64) + c * 2.0 ** -24 * terms_abs.double()
    err = (y64 - ref64).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        flat = int(bad.reshape(-1).nonzero()[0])
        idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), y.shape))
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at {idx}: "
                             f"got {y64[idx].item()!r}, want {ref64[idx].item()!r} +- {bound[idx].item()!r}")
    return float((_canon_bits(y) == _canon_bits(ref64.float().bfloat16())).double().mean())


def gemm_terms_abs(x, w, bias=None):
    t = x.double().abs() @ w.double().abs().t()
    return t if bias is None else t + bias.double().abs()


def gemm_ulp_c(K, bias):
    return math.ceil(K / 16) + (1 if bias is not None else 0)
