"""wgmma / TMA GEMM (``bcast_gemm``) vs a plain PyTorch fp32 reference of the same op."""
import pytest
import torch

from pytorch_ps_mpi_b200.ops.linear import BcastLinear, bcast_linear

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 784), (1000, 3072, 768), (77, 10, 512), (4096, 768, 3072),
                                   (8, 136, 72), (5000, 64, 176), (700, 128, 256)])
@pytest.mark.parametrize("bias,relu", [(False, False), (True, True)])
@pytest.mark.parametrize("variant", [1, 2])
def test_bcast_gemm_matches_fp32(M, N, K, bias, relu, variant):
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    x = (torch.randn(M, K, device=dev) / K ** 0.5).bfloat16()
    w = torch.randn(N, K, device=dev).bfloat16()
    b = torch.randn(N, device=dev).bfloat16() if bias else None
    y = bcast_linear(x, w, b, relu, variant=variant)
    ref = x.float() @ w.float().t()
    if bias:
        ref = ref + b.float()
    if relu:
        ref = ref.relu()
    torch.cuda.synchronize()
    assert y.dtype == torch.bfloat16 and y.shape == (M, N)
    err = (y.float() - ref).abs().max().item()
    assert torch.allclose(y.float(), ref, rtol=2e-2, atol=2e-2), err


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
