"""wgmma / TMA GEMM (``bcast_gemm``) against exact float64 references (``_wgmma_oracle``).

Exact data must come out bit for bit; random data within one bf16 ulp plus the fp32 accumulation bound, and at least 99 %
of it equal to the correctly rounded product."""
import pytest
import torch

from pytorch_ps_mpi_b200.ops.linear import BcastLinear, bcast_linear

from tests import _wgmma_oracle as wo

pytestmark = pytest.mark.gpu

NAN = float("nan")
# bias kind, relu: rotated over the cases so every value meets each
EPILOGUE_OPS = [(None, False), ("bf16", True), ("fp32", False), ("fp32", True), ("bf16", False), (None, True)]


def _cover():
    """Each M, N and K value of the covering set, with the other two dims fixed, plus the multi-wave shapes."""
    ms = [1, 64, 127, 128, 129, 255, 256, 257, 1000, 4096]
    ns = [8, 10, 63, 64, 65, 127, 128, 129, 136, 768, 3072]
    ks = [8, 56, 64, 72, 176, 784, 3072]
    cases = [(m, 129, 784) for m in ms]          # K = 784: 13 k-blocks, the smem ring (5 / 7 stages) wraps inside a tile
    cases += [(257, n, 176) for n in ns]         # N = 10 with a pair: one CTA's half of B is out of bounds
    cases += [(129, 136, k) for k in ks]
    cases += [(4096, 3072, 768), (4096, 768, 3072)]   # more tiles than SMs (one CTA) and than clusters (pairs)
    return [(m, n, k) + EPILOGUE_OPS[i % len(EPILOGUE_OPS)] for i, (m, n, k) in enumerate(cases)]


def _epis(n):
    return [1, 3, 4] if n % 8 == 0 else [1, 4]


def _bias(kind, n, dev, seed=7):
    if kind is None:
        return None
    b = torch.randn(n, generator=torch.Generator().manual_seed(seed)).to(dev)
    return b.bfloat16() if kind == "bf16" else b


def _poison(M, N, dev):
    """Allocate, NaN-fill and free a block of y's size: the caching allocator then probably hands y that block, so an
    element the kernel leaves unwritten shows up as NaN."""
    t = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
    t.fill_(NAN)
    del t


def _gemm(x, w, b, relu, variant, epi, w_ptr=0, flag_ptr=0, epoch=0):
    from pytorch_ps_mpi_b200.ops import ext
    _poison(x.shape[0], w.shape[0], x.device)
    return ext.cuda().bcast_gemm(x, w_ptr or w.data_ptr(), w.shape[0], w.shape[1], b, relu, flag_ptr, epoch, 30.0,
                                 variant | epi << 4)


def _tile(variant, n):
    return (128 * variant, 64 if n <= 64 else 128)


@pytest.mark.parametrize("M,N,K,bias,relu", _cover())
@pytest.mark.parametrize("variant", [1, 2])
def test_bcast_gemm_exact_data_bit_exact(M, N, K, bias, relu, variant):
    dev = torch.device("cuda", 0)
    x, w = wo.exact_gemm_operands(M, N, K, seed=M * 7 + N * 3 + K, device=dev)
    b = _bias(bias, N, dev)
    want = wo.gemm_expected(x, w, b, relu)
    for epi in _epis(N):
        y = _gemm(x, w, b, relu, variant, epi)
        torch.cuda.synchronize()
        assert y.dtype == torch.bfloat16 and y.shape == (M, N)
        wo.assert_bits_equal(y, want, _tile(variant, N), f"variant {variant} epilogue {epi}")


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 784), (1000, 3072, 768), (77, 10, 512), (4096, 768, 3072),
                                   (8, 136, 72), (5000, 64, 176), (700, 128, 256)])
@pytest.mark.parametrize("bias,relu", [(None, False), ("fp32", True)])
@pytest.mark.parametrize("variant", [1, 2])
def test_bcast_gemm_random_data_within_one_ulp(M, N, K, bias, relu, variant):
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    x = (torch.randn(M, K, device=dev) / K ** 0.5).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    b = _bias(bias, N, dev)
    y = bcast_linear(x, w, b, relu, variant=variant)
    ref = wo.gemm_ref64(x, w, b)
    if relu:
        ref = ref.relu()
    frac = wo.assert_within_ulp(y, ref, wo.gemm_terms_abs(x, w, b), wo.gemm_ulp_c(K, b), f"{M}x{N}x{K}")
    print(f"bcast_gemm random {M}x{N}x{K} bias={bias} relu={relu} variant={variant}: equal fraction {frac:.6f}")
    assert frac >= 0.99, frac


@pytest.mark.parametrize("M,N,K", [(1000, 328, 264), (515, 136, 72), (300, 64, 176), (4096, 3072, 768)])
def test_bcast_gemm_variants_and_repeats_agree_bitwise(M, N, K):
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    x = (torch.randn(M, K, device=dev) / K ** 0.5).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    b = torch.randn(N, device=dev)
    first = _gemm(x, w, b, True, 1, 1)
    for variant in (1, 2):
        for epi in _epis(N):
            for _ in range(2):
                wo.assert_bits_equal(_gemm(x, w, b, True, variant, epi), first, _tile(variant, N),
                                     f"variant {variant} epilogue {epi}")


@pytest.mark.parametrize("M,N,K", [(129, 65, 72), (257, 10, 8), (300, 136, 200)])
@pytest.mark.parametrize("variant", [1, 2])
def test_bcast_gemm_operands_inside_nan_buffers(M, N, K, variant):
    """x and the weight sit inside larger NaN-filled buffers: TMA must zero-fill the out-of-bounds parts of its boxes."""
    dev = torch.device("cuda", 0)
    x0, w0 = wo.exact_gemm_operands(M, N, K, seed=3, device=dev)
    pad = 8 * 64                                          # 16-byte multiple, more than one box row / column on each side
    xb = torch.full((M * K + 2 * pad,), NAN, dtype=torch.bfloat16, device=dev)
    wb = torch.full((N * K + 2 * pad,), NAN, dtype=torch.bfloat16, device=dev)
    x = xb[pad:pad + M * K].view(M, K)
    x.copy_(x0)
    wb[pad:pad + N * K].view(N, K).copy_(w0)
    want = wo.gemm_expected(x0, w0, None, False)
    for epi in _epis(N):
        y = _gemm(x, w0, None, False, variant, epi, w_ptr=wb.data_ptr() + 2 * pad)
        wo.assert_bits_equal(y, want, _tile(variant, N), f"variant {variant} epilogue {epi}")


def test_bcast_gemm_gate_at_epoch_is_bit_identical():
    from pytorch_ps_mpi_b200.ops import ext
    m = ext.cuda()
    dev = torch.device("cuda", 0)
    sig = torch.zeros(512, dtype=torch.int64, device=dev)
    m.signal([sig.data_ptr()], m.SIG_PARAMS_READY, 7)
    torch.manual_seed(2)
    x = torch.randn(300, 264, device=dev).bfloat16()
    w = torch.randn(136, 264, device=dev).bfloat16()
    b = torch.randn(136, device=dev)
    flag = sig.data_ptr() + 8 * m.SIG_PARAMS_READY
    for variant in (1, 2):
        for epi in _epis(136):
            plain = _gemm(x, w, b, True, variant, epi)
            gated = _gemm(x, w, b, True, variant, epi, flag_ptr=flag, epoch=7)
            torch.cuda.synchronize()
            assert int(sig[m.SIG_ERROR]) == 0
            wo.assert_bits_equal(gated, plain, _tile(variant, 136), f"variant {variant} epilogue {epi}")


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("M,N,K", [(300, 136, 200), (129, 65, 72)])
def test_bcast_gemm_nan_and_inf(M, N, K, relu):
    """A NaN in a row of x makes that row NaN; +Inf against weights of both signs (and zeros) gives +-Inf / NaN where the
    float64 product has them; with relu=True NaN stays NaN (as F.relu) and -Inf becomes 0."""
    dev = torch.device("cuda", 0)
    x, w = wo.exact_gemm_operands(M, N, K, seed=5, device=dev)
    x[3, 11] = NAN
    x[M - 2, 5] = float("inf")
    w[:, 5] = torch.tensor([1.0, -1.0, 0.0], device=dev).bfloat16().repeat(N)[:N]
    want = wo.gemm_expected(x, w, None, relu)
    assert bool(want[3].isnan().all()) and bool(want[M - 2].isnan().any()) and bool((want[M - 2] == float("inf")).any())
    assert bool((want[M - 2] == -float("inf")).any()) != relu
    for variant in (1, 2):
        for epi in _epis(N):
            wo.assert_bits_equal(_gemm(x, w, None, relu, variant, epi), want, _tile(variant, N),
                                 f"variant {variant} epilogue {epi}")


def test_bcast_linear_module_grad():
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    lin = torch.nn.Linear(256, 384).to(dev).bfloat16()
    mine = BcastLinear.from_linear(lin, relu=True)
    x = torch.randn(4, 50, 256, device=dev).bfloat16().requires_grad_(True)
    y = mine(x)
    ref = torch.relu(lin(x))
    assert torch.allclose(y.float(), ref.float(), rtol=2e-2, atol=2e-2)
    g = torch.randn_like(y)
    gx, gw, gb = torch.autograd.grad(y, [x, mine.weight, mine.bias], g)
    rx, rw, rb = torch.autograd.grad(ref, [x, lin.weight, lin.bias], g)
    for a, b in ((gx, rx), (gw, rw), (gb, rb)):
        assert torch.allclose(a.float(), b.float(), rtol=5e-2, atol=5e-2)


def test_gate_flag_blocks_until_published():
    """The TMA producer must not read the weight before the epoch flag is raised."""
    from pytorch_ps_mpi_b200.ops import ext
    m = ext.cuda()
    dev = torch.device("cuda", 0)
    sig = torch.zeros(512, dtype=torch.int64, device=dev)
    x = torch.randn(128, 64, device=dev).bfloat16()
    w = torch.zeros(128, 64, device=dev).bfloat16()
    # Everything the "server" side needs must exist BEFORE the spinning kernel starts: a cudaMalloc or the
    # lazy loading of a not-yet-used kernel synchronises the context and would wait for the spinner.
    m.signal([sig.data_ptr()], m.SIG_PARAMS_READY + 1, 1)
    torch.empty(8, device=dev).copy_(torch.empty(8, device=dev))
    w_new = torch.randn(128, 64, device=dev).bfloat16()
    side = torch.cuda.Stream()                             # would device-sync against it
    torch.cuda.synchronize()
    flag_ptr = sig.data_ptr() + 8 * m.SIG_PARAMS_READY
    with torch.cuda.stream(side):
        y = m.bcast_gemm(x, w.data_ptr(), 128, 64, None, False, flag_ptr, 7, 20.0, 0)   # spins on the flag
    # "the server": write the real weight, then publish epoch 7
    w.copy_(w_new)
    m.signal([sig.data_ptr()], m.SIG_PARAMS_READY, 7)
    torch.cuda.synchronize()
    assert int(sig[m.SIG_ERROR]) == 0
    assert torch.allclose(y.float(), x.float() @ w_new.float().t(), rtol=2e-2, atol=2e-2)
