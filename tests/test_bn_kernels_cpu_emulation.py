"""The fused BatchNorm kernels AND their launchers (``csrc/kernels/bn_kernels.cu``: statistics with fat reduce grids, finalize,
apply with the 1-bit ReLU mask, backward reduce / finalize / apply reading the mask) compiled from the repository's text and run on
the CPU emulator, against ``F.batch_norm`` + autograd in fp32.  ``kernel<<<grid, block, smem, s>>>(args)`` is rewritten to the
emulator's CTA runner, so the real grid-size logic (``grid_for`` / ``REDUCE_MIN_ITERS``) is what runs."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests import _cuda_emu


@pytest.fixture(autouse=True)
def _single_threaded_torch():
    """The emulated kernels run on the calling thread; keeping torch single-threaded makes the timings of these tests repeatable."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)

DRIVER = r'''
#include <vector>
extern "C" void emu_bn_forward(const void* x, const void* res, const void* gamma, const void* beta, void* y, float* scratch /*6C*/,
                               float* rm, float* rv, long long pixels, int C, float eps, float mom, int relu, void* mask) {
  std::vector<float> part(psb_bn_partial_floats(pixels, C));
  psb_bn_forward(0, x, res, gamma, beta, y, part.data(), scratch + 2 * C, scratch + 3 * C, scratch + 4 * C, scratch + 5 * C, rm, rv, pixels, C,
                 eps, mom, relu, 1, mask);
}
extern "C" void emu_bn_forward_presummed(const void* x, const void* gamma, const void* beta, void* y, const float* sums,
                                         float* scratch /*4C*/, float* rm, float* rv, long long pixels, int C, float eps, float mom,
                                         int relu, void* mask) {
  psb_bn_forward_presummed(0, x, nullptr, gamma, beta, y, sums, scratch, scratch + C, scratch + 2 * C, scratch + 3 * C, rm, rv, pixels, C,
                           eps, mom, relu, mask);
}
extern "C" void emu_bn_backward(const void* dy, const void* x, const void* y, const void* gamma, const float* mean, const float* rstd,
                                float* scratch /*5C*/, void* dx, void* dres, void* dgamma, void* dbeta, long long pixels, int C, int relu,
                                const void* mask) {
  std::vector<float> part(psb_bn_partial_floats(pixels, C));
  psb_bn_backward(0, dy, x, y, gamma, mean, rstd, part.data(), scratch + 2 * C, dx, dres, dgamma, dbeta, pixels, C, relu, mask);
}
'''


@pytest.fixture(scope="module")
def lib():
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return _cuda_emu.compile_shared(_cuda_emu.bn_source() + DRIVER, "psb_emu_bn_")


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


@pytest.mark.parametrize("shape,relu,has_res", [((2, 16, 6, 5), True, True), ((3, 64, 9, 9), True, False), ((2, 8, 4, 4), False, True),
                                                ((1, 512, 5, 5), True, False), ((12, 16, 12, 12), False, False)])
def test_bn_forward_backward_emulated(lib, shape, relu, has_res):
    _bn_case(lib, shape, relu, has_res)


def test_bn_with_capped_grids(lib):
    """One "SM": every launcher's grid cap (8 CTAs per SM) binds, so the apply / reduce kernels run their grid-stride loops several
    times per CTA — the normal case on hardware (ResNet-18 layer1: 25 088 pixel batches on 1 184 CTAs)."""
    lib.emu_set_sm_count(1)
    try:
        _bn_case(lib, (4, 64, 12, 12), True, True)
        _bn_case(lib, (3, 16, 9, 7), False, False)
    finally:
        lib.emu_set_sm_count(148)


def _bn_case(lib, shape, relu, has_res):
    torch.manual_seed(0)
    N, C, H, W = shape
    pixels = N * H * W
    x = (torch.randn(N, H, W, C) * 1.5 + 0.3).bfloat16()                       # NHWC storage
    res = torch.randn(N, H, W, C).bfloat16() if has_res else None
    gamma, beta = (torch.rand(C) + 0.5).bfloat16(), (torch.randn(C) * 0.3).bfloat16()
    rm, rv = torch.zeros(C), torch.ones(C)
    y = torch.empty_like(x)
    scratch = torch.zeros(6 * C)
    mask = torch.zeros(pixels * (C // 8), dtype=torch.uint8) if relu else None
    lib.emu_bn_forward(_p(x), _p(res), _p(gamma), _p(beta), _p(y), _p(scratch), _p(rm), _p(rv), ctypes.c_longlong(pixels), C,
                       ctypes.c_float(1e-5), ctypes.c_float(0.1), int(relu), _p(mask))
    mean, rstd = scratch[2 * C:3 * C].clone(), scratch[3 * C:4 * C].clone()
    # fp32 oracle on the same bf16 inputs
    xf = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    rf = res.float().permute(0, 3, 1, 2).requires_grad_(True) if has_res else None
    gf, bf = gamma.float().requires_grad_(True), beta.float().requires_grad_(True)
    orm, orv = torch.zeros(C), torch.ones(C)
    out = F.batch_norm(xf, orm, orv, gf, bf, True, 0.1, 1e-5)
    if has_res:
        out = out + rf
    if relu:
        out = F.relu(out)
    want = out.detach().permute(0, 2, 3, 1)
    assert torch.allclose(y.float(), want, rtol=2e-2, atol=2e-2)
    assert torch.allclose(rm, orm, rtol=1e-4, atol=1e-5) and torch.allclose(rv, orv, rtol=1e-4, atol=1e-5)
    if relu:                                                                   # one bit per element: y > 0
        bits = ((mask.view(pixels, C // 8, 1) >> torch.arange(8, dtype=torch.uint8)) & 1).view(N, H, W, C)
        assert torch.equal(bits.bool(), y.float() > 0)
    # backward through the mask (never re-reading y)
    dy = torch.randn(N, H, W, C).bfloat16()
    dx, dres = torch.empty_like(x), (torch.empty_like(x) if has_res else None)
    dgamma, dbeta = torch.empty(C, dtype=torch.bfloat16), torch.empty(C, dtype=torch.bfloat16)
    s2 = torch.zeros(5 * C)
    lib.emu_bn_backward(_p(dy), _p(x), None, _p(gamma), _p(mean), _p(rstd), _p(s2), _p(dx), _p(dres), _p(dgamma), _p(dbeta),
                        ctypes.c_longlong(pixels), C, int(relu), _p(mask))
    out.backward(dy.float().permute(0, 3, 1, 2))
    tol = dict(rtol=3e-2, atol=3e-2)
    assert torch.allclose(dx.float(), xf.grad.permute(0, 2, 3, 1), **tol)
    if has_res:
        assert torch.allclose(dres.float(), rf.grad.permute(0, 2, 3, 1), **tol)
    scale = max(1.0, float(gf.grad.abs().max()))
    assert torch.allclose(dgamma.float() / scale, gf.grad / scale, rtol=2e-2, atol=2e-2)
    assert torch.allclose(dbeta.float() / scale, bf.grad / scale, rtol=2e-2, atol=2e-2)


def test_bn_forward_with_sums_from_the_producer(lib):
    """``psb_bn_forward_presummed`` (the default ResNet stem: Σy / Σy² come out of the stem kernel's epilogue, so BatchNorm
    skips its statistics pass): same output, mask and running statistics as the full forward."""
    torch.manual_seed(1)
    N, H, W, C = 3, 6, 10, 64
    pixels = N * H * W
    x = (torch.randn(N, H, W, C) * 2.0 - 0.5).bfloat16()
    gamma, beta = (torch.rand(C) + 0.5).bfloat16(), (torch.randn(C) * 0.3).bfloat16()
    xf = x.float().reshape(-1, C)
    sums = torch.cat([xf.sum(0), (xf * xf).sum(0)]).contiguous()               # what the producer's epilogue accumulates (fp32)
    rm, rv, y = torch.zeros(C), torch.ones(C), torch.empty_like(x)
    scratch = torch.zeros(4 * C)
    mask = torch.zeros(pixels * (C // 8), dtype=torch.uint8)
    lib.emu_bn_forward_presummed(_p(x), _p(gamma), _p(beta), _p(y), _p(sums), _p(scratch), _p(rm), _p(rv), ctypes.c_longlong(pixels), C,
                                 ctypes.c_float(1e-5), ctypes.c_float(0.1), 1, _p(mask))
    orm, orv = torch.zeros(C), torch.ones(C)
    want = F.relu(F.batch_norm(x.float().permute(0, 3, 1, 2), orm, orv, gamma.float(), beta.float(), True, 0.1, 1e-5)).permute(0, 2, 3, 1)
    assert torch.allclose(y.float(), want, rtol=2e-2, atol=2e-2)
    assert torch.allclose(rm, orm, rtol=1e-4, atol=1e-5) and torch.allclose(rv, orv, rtol=1e-4, atol=1e-5)
    assert torch.allclose(scratch[:C], xf.mean(0), rtol=1e-5, atol=1e-6)         # mean
    bits = ((mask.view(pixels, C // 8, 1) >> torch.arange(8, dtype=torch.uint8)) & 1).view(N, H, W, C)
    assert torch.equal(bits.bool(), y.float() > 0)
