"""GPU tests of the fused ResNet stem (implicit-GEMM forward with BN statistics in the epilogue, implicit weight
gradient), and every epilogue of the GEMM.

Part of the default ``pytest -m gpu`` run.  The kernels are compared with exact float64 references
(``_wgmma_oracle``): bit for bit on exact data, within one bf16 ulp plus the fp32 accumulation bound on random data, and
the BatchNorm sums bit for bit against a replay of the kernel's summation order.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import _wgmma_oracle as wo

pytestmark = [pytest.mark.gpu]

NAN = float("nan")
# (N, H, W); a string N is resolved against the SM count so that N * OH tiles = SMs, SMs + 1 or 2 * SMs + 1 (one tile per
# CTA; CTAs with no tile; the A / patch / staging double buffers wrapping their parity)
SHAPES = [(1, 1, 8), (1, 2, 8), (1, 7, 16), (5, 17, 8), (1, 30, 40), (3, 64, 64), (2, 225, 256), (1, 224, 248),
          (256, 224, 224), ("sms", 1, 64), ("sms+1", 2, 64), ("2sms+1", 1, 64)]


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _shape(shape):
    n, h, w = shape
    if isinstance(n, str):
        n = {"sms": _sms(), "sms+1": _sms() + 1, "2sms+1": 2 * _sms() + 1}[n]
    return n, h, w


def _m():
    from pytorch_ps_mpi_b200.ops import ext
    return ext.cuda()


def _weight_in_gemm_layout(wt):
    """``wt`` stored as the zero-padded [64,176] GEMM matrix (``STEM_STRIDES``), the layout of the parameter arena."""
    from pytorch_ps_mpi_b200.ops.stem import STEM_K, STEM_STRIDES
    buf = torch.zeros(64 * STEM_K, dtype=wt.dtype, device=wt.device)
    w4 = torch.as_strided(buf, (64, 3, 7, 7), STEM_STRIDES)
    w4.copy_(wt)
    return w4


@pytest.mark.parametrize("shape", SHAPES)
def test_fused_stem_forward_exact_and_random(shape):
    from pytorch_ps_mpi_b200.ops.stem import _w2d, _w2d_of, in_gemm_layout
    n, h, w = _shape(shape)
    dev = torch.device("cuda", 0)
    m = _m()
    # exact data: bit-exact through both weight paths
    x = wo.exact_stem_input(n, h, w, seed=n + h + w, device=dev)
    wt = wo.exact_stem_weight(seed=1, device=dev)
    want = wo.stem_fwd_ref64(x, wt).float().bfloat16()
    y, _ = m.stem_fwd(x, _w2d(wt), True)
    assert y.shape == want.shape and y.is_contiguous(memory_format=torch.channels_last)
    wo.assert_bits_equal(y, want, (1, 64, 1, 128), "exact data, _w2d weight")
    w4 = _weight_in_gemm_layout(wt)
    assert in_gemm_layout(w4)
    wv = _w2d_of(w4)
    assert wv.data_ptr() == w4.data_ptr()                 # the zero-copy view
    wo.assert_bits_equal(m.stem_fwd(x, wv, False)[0], want, (1, 64, 1, 128), "exact data, STEM_STRIDES view")
    del y, want
    # random data: within one ulp, >= 99 % correctly rounded; the sums equal the replay of the kernel's order
    torch.manual_seed(0)
    wt = (torch.randn(64, 3, 7, 7, device=dev) * 0.05).bfloat16()
    x = _cl(torch.randn(n, 3, h, w, device=dev).bfloat16())
    y, sums = m.stem_fwd(x, _w2d(wt), True)
    ref = wo.stem_fwd_ref64(x, wt)
    terms = F.conv2d(x.double().abs(), wt.double().abs(), stride=2, padding=3)
    frac = wo.assert_within_ulp(y, ref, terms, 176 // 16, f"stem forward {n}x{h}x{w}")
    print(f"stem_fwd random {n}x{h}x{w}: equal fraction {frac:.6f}")
    assert frac >= 0.99, frac
    replay = wo.stem_sums_replay(y, _sms())
    wo.assert_bits_equal(sums, replay, what="stem sums")
    if n * ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1) >= 64:   # enough pixels for the unrounded sums to differ somewhere
        unrounded = wo.stem_sums_replay(ref.float(), _sms())
        assert not torch.equal(unrounded, replay), "sums of the unrounded accumulators should differ from the bf16 ones"


def test_fused_stem_nan_pixel():
    """One NaN input pixel: NaN in exactly the outputs whose 7x7 window covers it (all 64 channels), and NaN sums."""
    dev = torch.device("cuda", 0)
    from pytorch_ps_mpi_b200.ops.stem import _w2d
    torch.manual_seed(3)
    wt = (torch.randn(64, 3, 7, 7, device=dev) * 0.05).bfloat16()
    x = torch.randn(2, 3, 30, 40, device=dev).bfloat16()
    x[1, 2, 13, 21] = NAN
    x = _cl(x)
    y, sums = _m().stem_fwd(x, _w2d(wt), True)
    ref = wo.stem_fwd_ref64(x, wt)
    assert 0 < int(ref.isnan().sum()) < ref.numel() and bool(ref.isnan().any(1).eq(ref.isnan().all(1)).all())
    assert torch.equal(y.isnan(), ref.isnan())
    assert bool(sums.isnan().all())


@pytest.mark.parametrize("shape", SHAPES)
def test_implicit_stem_wgrad(shape):
    from pytorch_ps_mpi_b200.ops.stem import STEM_K, _w2d, stem_wgrad_implicit
    n, h, w = _shape(shape)
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    dev = torch.device("cuda", 0)
    m = _m()
    # exact data: bit-exact dW2d
    x, g = wo.exact_wgrad_operands(n, h, w, seed=n + h + w, device=dev)
    wo.assert_bits_equal(stem_wgrad_implicit(x, g), wo.stem_wgrad_ref64(x, g).float().bfloat16(), (64, 176), "exact data")
    # random data
    torch.manual_seed(0)
    x = _cl(torch.randn(n, 3, h, w, device=dev).bfloat16())
    g = _cl(torch.randn(n, 64, oh, ow, device=dev).bfloat16())
    partial = m.stem_wgrad(x, g)
    grid = partial.shape[0]
    dw = m.stem_wgrad_finalize(partial, None)
    per = -(-(n * oh) // grid)
    terms = _w2d(torch.nn.grad.conv2d_weight(x.double().abs(), (64, 3, 7, 7), g.double().abs(), stride=2, padding=3))
    frac = wo.assert_within_ulp(dw, wo.stem_wgrad_ref64(x, g), terms, per * -(-ow // 16) + grid, f"stem wgrad {n}x{h}x{w}")
    print(f"stem_wgrad random {n}x{h}x{w}: equal fraction {frac:.6f}")
    # CTAs with no tile write zero partials
    idle = torch.arange(grid, device=dev) * per >= n * oh
    assert bool(idle.any()) or shape[0] != "sms+1"
    assert bool((partial[idle] == 0).all())
    # two runs are bit-identical
    wo.assert_bits_equal(stem_wgrad_implicit(x, g), dw, (64, 176), "second run")
    # out=: a slot inside a NaN-filled buffer; the guard elements stay as they were
    buf = torch.full((64 * STEM_K + 2 * 64,), NAN, dtype=torch.bfloat16, device=dev)
    before = buf.clone()
    out = buf[64:64 + 64 * STEM_K]
    r = m.stem_wgrad_finalize(partial, out)
    assert r.data_ptr() == out.data_ptr()
    wo.assert_bits_equal(out.view(64, STEM_K), dw, (64, 176), "out=")
    assert torch.equal(buf[:64].view(torch.int16), before[:64].view(torch.int16))
    assert torch.equal(buf[-64:].view(torch.int16), before[-64:].view(torch.int16))


def test_fused_stem_gate_at_epoch_is_bit_identical():
    from pytorch_ps_mpi_b200.ops.stem import _w2d
    m = _m()
    dev = torch.device("cuda", 0)
    sig = torch.zeros(512, dtype=torch.int64, device=dev)
    m.signal([sig.data_ptr()], m.SIG_PARAMS_READY, 5)
    torch.manual_seed(4)
    wt = _w2d((torch.randn(64, 3, 7, 7, device=dev) * 0.05).bfloat16())
    x = _cl(torch.randn(3, 3, 64, 64, device=dev).bfloat16())
    y0, s0 = m.stem_fwd(x, wt, True)
    y1, s1 = m.stem_fwd(x, wt, True, sig.data_ptr() + 8 * m.SIG_PARAMS_READY, 5, 30.0)
    torch.cuda.synchronize()
    assert int(sig[m.SIG_ERROR]) == 0
    wo.assert_bits_equal(y1, y0, what="gated y")
    wo.assert_bits_equal(s1, s0, what="gated sums")


@pytest.mark.parametrize("shape", [(2, 224, 224), (5, 17, 8), (1, 30, 44)])
def test_stem_conv_fallback_exact_data(shape):
    """The fallback path (im2col + bcast_gemm) on exact data: bit-exact, like the fused kernel."""
    from pytorch_ps_mpi_b200.ops.stem import stem_conv
    n, h, w = shape
    dev = torch.device("cuda", 0)
    x = wo.exact_stem_input(n, h, w, seed=2, device=dev)
    wt = wo.exact_stem_weight(seed=3, device=dev)
    wo.assert_bits_equal(stem_conv(x, wt), wo.stem_fwd_ref64(x, wt).float().bfloat16(), what="stem_conv")


def test_fused_stem_autograd_matches_default_path():
    from pytorch_ps_mpi_b200.ops import stem as stem_mod
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    wt = (torch.randn(64, 3, 7, 7, device=dev) * 0.05).bfloat16()
    x = _cl(torch.randn(4, 3, 224, 224, device=dev).bfloat16())
    gy = _cl(torch.randn(4, 64, 112, 112, device=dev).bfloat16())
    grads = []
    for fused, implicit in ((False, False), (True, False), (True, True)):
        stem_mod._IMPLICIT_WGRAD = implicit
        wv = wt.clone().requires_grad_(True)
        y = stem_mod.stem_conv_fused(x, wv)[0] if fused else stem_mod.stem_conv(x, wv)
        y.backward(gy)
        grads.append(wv.grad.float())
    stem_mod._IMPLICIT_WGRAD = False
    rel = [(g - grads[0]).abs().max().item() / grads[0].abs().max().item() for g in grads[1:]]
    assert max(rel) < 1e-2, rel


@pytest.mark.parametrize("epi", [0, 1, 3, 4])   # 0 auto (TMA store / staged), 1 staged, 3 TMA store, 4 round-1 row-strided stores
@pytest.mark.parametrize("mnk", [(512, 256, 128), (1000, 328, 264), (4096, 3072, 768), (300, 64, 176), (515, 330, 72)])
def test_gemm_epilogue_variants(epi, mnk):
    from pytorch_ps_mpi_b200.ops.linear import bcast_linear
    M, N, K = mnk
    if epi == 3 and N % 8:
        pytest.skip("TMA-store epilogue needs N % 8 == 0")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    x = (torch.randn(M, K, device=dev) / K ** 0.5).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    b = torch.randn(N, device=dev)
    y = bcast_linear(x, w, b, relu=True, variant=2 | epi << 4)
    frac = wo.assert_within_ulp(y, wo.gemm_ref64(x, w, b).relu(), wo.gemm_terms_abs(x, w, b), wo.gemm_ulp_c(K, b))
    assert frac >= 0.99, frac
