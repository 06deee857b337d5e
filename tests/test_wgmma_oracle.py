"""CPU checks of the tensor-core oracle (``_wgmma_oracle``) and of the emulator's stand-ins for the wgmma kernels.

- The exact data really is exact: float64 against fp32 sums in several orders and against an adder that keeps 13 bits.
- The sums replay reproduces a literal loop over the kernel's documented order.
- Torch models of each kernel's contract with one planted defect pass the loose check the oracle replaced and fail the
  oracle's check.
- The ATen stand-ins of ``_cuda_emu.GEMM_STANDINS`` meet the same contract through the emulated extension, which ties the
  emulated model tests to what the H100 kernels compute.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import _cuda_emu
from tests import _wgmma_oracle as wo

NAN = float("nan")


# ------------------------------------------------------------------ the exact data is exact
def _trunc13_sum(terms):
    """Sequential sum by an adder that aligns both operands to the larger exponent and keeps 13 bits (truncating)."""
    acc = torch.zeros(terms.shape[:-1], dtype=torch.float64)
    for k in range(terms.shape[-1]):
        b = terms[..., k]
        big = torch.maximum(acc.abs(), b.abs())
        _, e = torch.frexp(big)
        q = torch.exp2((e - 13).double())
        acc = torch.trunc(acc / q) * q + torch.trunc(b / q) * q
    return acc


def test_exact_gemm_data_sums_exactly_in_any_order():
    M, N, K = 6, 5, 4096
    x, w = wo.exact_gemm_operands(M, N, K, seed=11)
    ref = wo.gemm_ref64(x, w)
    prods = (x.float()[:, None, :] * w.float()[None, :, :])            # exact in fp32
    assert torch.equal(prods.double(), x.double()[:, None, :] * w.double()[None, :, :])
    fwd = torch.zeros(M, N)
    rev = torch.zeros(M, N)
    for k in range(K):
        fwd = fwd + prods[..., k]
        rev = rev + prods[..., K - 1 - k]
    blocked = torch.zeros(M, N)
    for k0 in range(0, K, 16):                                          # k16 blocks, then the fp32 accumulator
        blk = torch.zeros(M, N)
        for k in range(k0, k0 + 16):
            blk = blk + prods[..., k]
        blocked = blocked + blk
    for s in (fwd, rev, blocked):
        assert torch.equal(s.double(), ref)
    assert torch.equal(_trunc13_sum(prods.double()), ref)
    assert ref.abs().max() > 64                                         # the sums do grow
    # random data is not exact: the same checks notice
    xr, wr = torch.randn(M, K).bfloat16(), torch.randn(N, K).bfloat16()
    pr = xr.float()[:, None, :] * wr.float()[None, :, :]
    assert not torch.equal(_trunc13_sum(pr.double()), wo.gemm_ref64(xr, wr))


def test_builders_assert_their_preconditions():
    with pytest.raises(AssertionError):
        wo.exact_gemm_operands(8, 8, wo.GEMM_MAX_K + 8)
    with pytest.raises(AssertionError):
        wo.exact_wgrad_operands(22000, 56, 56)                          # 22000 * 28 * 28 > 2^24 products


def test_exact_stem_data_is_exact_in_fp32():
    x = wo.exact_stem_input(2, 20, 16, seed=1)
    wt = wo.exact_stem_weight(seed=2)
    ref = wo.stem_fwd_ref64(x, wt)
    assert torch.equal(F.conv2d(x.float(), wt.float(), stride=2, padding=3).double(), ref)
    xg, g = wo.exact_wgrad_operands(2, 20, 16, seed=3)
    dw = torch.nn.grad.conv2d_weight(xg.float(), (64, 3, 7, 7), g.float(), stride=2, padding=3)
    from pytorch_ps_mpi_b200.ops.stem import _w2d
    assert torch.equal(_w2d(dw).double(), wo.stem_wgrad_ref64(xg, g))


# ------------------------------------------------------------------ the sums replay
def _literal_stem_sums(y, sms):
    """psb_stem_fwd_kernel + psb_stem_sums_kernel, one fp32 scalar at a time."""
    n, _, oh, ow = y.shape
    v = y.permute(0, 2, 3, 1).reshape(n * oh, ow, 64).float().numpy()
    tiles = n * oh
    grid = min(tiles, sms)
    per = (tiles + grid - 1) // grid
    rq = (ow + 3) >> 2
    part = np.zeros((grid, 128), np.float32)
    for b in range(grid):
        t0, t1 = b * per, min(b * per + per, tiles)
        red = np.zeros((2, 4, 64), np.float32)
        for q in range(4):
            r0, r1 = q * rq, min(ow, q * rq + rq)
            for ch in range(64):
                s, s2 = np.float32(0), np.float32(0)
                for t in range(t0, t1):
                    for rr in range(r0, r1):
                        e = v[t, rr, ch]
                        s = np.float32(s + e)
                        s2 = np.float32(s2 + np.float32(e * e))
                red[0, q, ch], red[1, q, ch] = s, s2
        part[b] = np.concatenate([((red[0, 0] + red[0, 1]) + red[0, 2]) + red[0, 3],
                                  ((red[1, 0] + red[1, 1]) + red[1, 2]) + red[1, 3]])
    acc = np.zeros(128, np.float32)
    for b in range(grid):
        acc = acc + part[b]
    return torch.from_numpy(acc)


@pytest.mark.parametrize("n,h,w,sms", [(3, 9, 24, 4), (2, 7, 20, 5), (1, 3, 8, 132), (4, 5, 16, 3)])
def test_sums_replay_matches_a_literal_loop(n, h, w, sms):
    torch.manual_seed(n * 100 + sms)
    y = (torch.randn(n, 64, (h - 1) // 2 + 1, (w - 1) // 2 + 1) * 3).bfloat16()
    wo.assert_bits_equal(wo.stem_sums_replay(y, sms), _literal_stem_sums(y, sms), what="replay")


def test_comparators():
    a = torch.tensor([0.0, -0.0, NAN, 1.0]).bfloat16()
    wo.assert_bits_equal(a, torch.tensor([-0.0, 0.0, -NAN, 1.0]).bfloat16())
    with pytest.raises(AssertionError, match=r"first at \(1, 2\).*tile \(0, 1\)"):
        wo.assert_bits_equal(torch.zeros(2, 4).bfloat16(), torch.tensor([[0.0] * 4, [0, 0, 1e-3, 0]]).bfloat16(), (2, 2))
    ref = torch.tensor([1.0, 3.0, 0.0], dtype=torch.float64)
    assert wo.assert_within_ulp(ref.bfloat16(), ref, torch.zeros(3), 0) == 1.0
    wo.assert_within_ulp(torch.tensor([1.0078125, 3.0, 0.0]).bfloat16(), ref, torch.zeros(3), 0)     # one ulp at 1
    with pytest.raises(AssertionError):
        wo.assert_within_ulp(torch.tensor([1.015625, 3.0, 0.0]).bfloat16(), ref, torch.zeros(3), 0)  # two ulps


# ------------------------------------------------------------------ planted defects
def _rtz_bf16(v):
    return (v.float().view(torch.int32) & -65536).view(torch.float32).bfloat16()


def _gemm_model(x, w, b, relu, defect=None):
    """The GEMM's contract in torch (fp32 accumulator → + fp32 bias → ReLU → bf16), optionally with one defect."""
    acc = x.float() @ w.float().t()
    if defect == "bias_after_bf16":
        acc = acc.bfloat16().float()
    if b is not None:
        acc = acc + b.float()
    if relu:
        acc = torch.relu(acc)
        if defect == "relu_nan_to_zero":
            acc = torch.nan_to_num(acc, nan=0.0)
    return _rtz_bf16(acc) if defect == "round_toward_zero" else acc.bfloat16()


def _old_gemm_check(defect):
    """The replaced check: allclose(rtol=2e-2, atol=2e-2) against an fp32 reference, on random data."""
    for M, N, K in [(128, 128, 64), (256, 512, 784), (77, 10, 512), (8, 136, 72), (700, 128, 256)]:
        torch.manual_seed(0)
        x = (torch.randn(M, K) / K ** 0.5).bfloat16()
        w = torch.randn(N, K).bfloat16()
        b = torch.randn(N).bfloat16()
        for bias, relu in ((None, False), (b, True)):
            y = _gemm_model(x, w, bias, relu, defect)
            ref = x.float() @ w.float().t()
            if bias is not None:
                ref = ref + bias.float()
            if relu:
                ref = ref.relu()
            if not torch.allclose(y.float(), ref, rtol=2e-2, atol=2e-2):
                return False
    return True


def _new_gemm_checks(defect):
    """The oracle's GEMM checks; returns the names of those that fail."""
    failed = []
    x, w = wo.exact_gemm_operands(257, 136, 784, seed=1)
    b = torch.randn(136)
    try:
        wo.assert_bits_equal(_gemm_model(x, w, b, True, defect), wo.gemm_expected(x, w, b, True))
    except AssertionError:
        failed.append("exact")
    torch.manual_seed(0)
    xr, wr = (torch.randn(256, 512) / 512 ** 0.5).bfloat16(), torch.randn(384, 512).bfloat16()
    frac = wo.assert_within_ulp(_gemm_model(xr, wr, None, False, defect), wo.gemm_ref64(xr, wr), wo.gemm_terms_abs(xr, wr),
                                wo.gemm_ulp_c(512, None))
    if frac < 0.99:
        failed.append("random")
    xn = x.clone()
    xn[3, 7] = NAN
    try:
        wo.assert_bits_equal(_gemm_model(xn, w, b, True, defect), wo.gemm_expected(xn, w, b, True))
    except AssertionError:
        failed.append("nan")
    return failed


def test_gemm_model_without_defect_passes_both():
    assert _old_gemm_check(None)
    assert _new_gemm_checks(None) == []


@pytest.mark.parametrize("defect,caught_by", [("round_toward_zero", {"exact", "random"}),
                                              ("bias_after_bf16", {"exact"}),
                                              ("relu_nan_to_zero", {"nan"})])
def test_planted_gemm_defect_passes_the_old_check_and_fails_the_oracle(defect, caught_by):
    assert _old_gemm_check(defect)
    assert caught_by <= set(_new_gemm_checks(defect))


# ------------------------------------------------------------------ the emulator's stand-ins meet the same contract
@pytest.fixture(scope="module")
def emu():
    m = _cuda_emu.build_extension()
    if m is None:
        pytest.skip("no g++")
    return m


def _emu_gemm(m, x, w, b, relu):
    return m.bcast_gemm(x, w.data_ptr(), w.shape[0], w.shape[1], b, relu, 0, 0, 30.0, 0)


@pytest.mark.parametrize("M,N,K", [(1, 8, 8), (129, 65, 784), (257, 10, 176), (300, 136, 3072)])
@pytest.mark.parametrize("bias,relu", [(None, False), ("bf16", True), ("fp32", False), ("fp32", True)])
def test_standin_bcast_gemm_exact_data(emu, M, N, K, bias, relu):
    x, w = wo.exact_gemm_operands(M, N, K, seed=M + N + K)
    b = None if bias is None else torch.randn(N, generator=torch.Generator().manual_seed(1))
    if bias == "bf16":
        b = b.bfloat16()
    wo.assert_bits_equal(_emu_gemm(emu, x, w, b, relu), wo.gemm_expected(x, w, b, relu), what="stand-in bcast_gemm")


@pytest.mark.parametrize("relu", [False, True])
def test_standin_bcast_gemm_nan_and_inf(emu, relu):
    x, w = wo.exact_gemm_operands(130, 24, 72, seed=5)
    x[3, 11] = NAN
    x[128, 5] = float("inf")
    w[:, 5] = torch.tensor([1.0, -1.0, 0.0]).bfloat16().repeat(8)
    want = wo.gemm_expected(x, w, None, relu)
    assert bool(want[3].isnan().all()) and bool(want[128].isnan().any())
    wo.assert_bits_equal(_emu_gemm(emu, x, w, None, relu), want, what="stand-in bcast_gemm")


@pytest.mark.parametrize("shape", [(1, 1, 8), (5, 17, 8), (2, 30, 40)])
def test_standin_stem_fwd_exact_data_and_sums(emu, shape):
    from pytorch_ps_mpi_b200.ops.stem import _w2d
    n, h, w = shape
    x = wo.exact_stem_input(n, h, w, seed=4)
    wt = wo.exact_stem_weight(seed=5)
    y, _ = emu.stem_fwd(x, _w2d(wt), True, 0, 0, 30.0)
    wo.assert_bits_equal(y, wo.stem_fwd_ref64(x, wt).float().bfloat16(), what="stand-in stem_fwd")
    torch.manual_seed(0)
    xr = (torch.randn(n, 3, h, w) * 2).bfloat16().contiguous(memory_format=torch.channels_last)
    wr = (torch.randn(64, 3, 7, 7) * 0.05).bfloat16()
    y, sums = emu.stem_fwd(xr, _w2d(wr), True, 0, 0, 30.0)
    # one "CTA", one quarter: a plain sum over the bf16 y in pixel order
    wo.assert_bits_equal(sums, wo.stem_sums_replay(y, 1, quarters=1), what="stand-in sums")


def test_standin_stem_fwd_nan_pixel(emu):
    from pytorch_ps_mpi_b200.ops.stem import _w2d
    torch.manual_seed(3)
    wt = (torch.randn(64, 3, 7, 7) * 0.05).bfloat16()
    x = torch.randn(1, 3, 20, 24).bfloat16()
    x[0, 1, 9, 10] = NAN
    x = x.contiguous(memory_format=torch.channels_last)
    y, sums = emu.stem_fwd(x, _w2d(wt), True, 0, 0, 30.0)
    assert torch.equal(y.isnan(), wo.stem_fwd_ref64(x, wt).isnan()) and bool(y.isnan().any())
    assert bool(sums.isnan().all())


@pytest.mark.parametrize("shape", [(1, 1, 8), (3, 17, 8), (2, 30, 40)])
def test_standin_stem_wgrad_exact_data(emu, shape):
    n, h, w = shape
    x, g = wo.exact_wgrad_operands(n, h, w, seed=6)
    dw = emu.stem_wgrad_finalize(emu.stem_wgrad(x, g), None)
    wo.assert_bits_equal(dw, wo.stem_wgrad_ref64(x, g).float().bfloat16(), what="stand-in stem_wgrad")
