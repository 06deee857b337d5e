"""The BatchNorm finalize kernels (``csrc/kernels/bn_kernels.cu``) add the per-CTA partial rows in one documented order: slice
``i`` of 8 adds rows ``i, i + 8, i + 16, ...`` one after another in fp32, then the 8 slice sums are added in slice order.  A
run therefore gives the same bits on every launch and every build that keeps that order.  This checks the order bit for bit
on the CPU emulator against a float32 numpy reference, for row counts below, at and across the kernels' load batches (the
launchers use up to 8 x 132 rows on an H100)."""
import ctypes

import numpy as np
import pytest
import torch

from tests import _cuda_emu

DRIVER = r'''
extern "C" void emu_bn_bwd_finalize(const float* part, int nparts, const float* mean, const float* rstd, float* coef /*3C*/,
                                    void* dgamma, void* dbeta, int C) {
  emu_launch((C + FIN_CH - 1) / FIN_CH, FIN_THREADS, [&] {
    psb_bn_bwd_finalize(part, nparts, nullptr, mean, rstd, coef, coef + C, coef + 2 * C,
                        reinterpret_cast<__nv_bfloat16*>(dgamma), reinterpret_cast<__nv_bfloat16*>(dbeta), C, 1LL);
  });
}
'''


@pytest.fixture(scope="module")
def lib():
    import shutil
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    return _cuda_emu.compile_shared(_cuda_emu.bn_source() + DRIVER, "psb_emu_bn_fin_")


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _ordered_sum(col: np.ndarray) -> np.float32:
    slices = []
    for i in range(8):
        s = np.float32(0)
        for v in col[i::8]:
            s = np.float32(s + v)
        slices.append(s)
    t = np.float32(0)
    for s in slices:
        t = np.float32(t + s)
    return t


@pytest.mark.parametrize("nparts", [1, 5, 8, 127, 128, 129, 300, 1056])
@pytest.mark.parametrize("C", [64, 48])
def test_finalize_adds_partials_in_slice_order(lib, nparts, C):
    rng = np.random.default_rng(nparts * 7 + C)
    # magnitudes over 12 binades: a different association of the same numbers gives different bits
    part = (rng.standard_normal((nparts, 2 * C)) * np.exp2(rng.integers(-6, 6, (nparts, 2 * C)))).astype(np.float32)
    mean, rstd = torch.zeros(C), torch.ones(C)          # pixels = 1, rstd = 1, mean = 0: the coefficients are -Σdy·x̂ and -Σdy
    coef = torch.full((3 * C,), float("nan"))
    dgamma = torch.zeros(C, dtype=torch.bfloat16)
    dbeta = torch.zeros(C, dtype=torch.bfloat16)
    lib.emu_bn_bwd_finalize(_p(torch.from_numpy(part)), nparts, _p(mean), _p(rstd), _p(coef), _p(dgamma), _p(dbeta), C)
    want_dy = np.array([_ordered_sum(part[:, c]) for c in range(C)], dtype=np.float32)
    want_dyx = np.array([_ordered_sum(part[:, C + c]) for c in range(C)], dtype=np.float32)
    got = coef.numpy()
    assert np.array_equal(got[:C], np.ones(C, dtype=np.float32))
    assert np.array_equal((-got[C:2 * C]).view(np.uint32), want_dyx.view(np.uint32))
    assert np.array_equal((-got[2 * C:]).view(np.uint32), want_dy.view(np.uint32))
    assert torch.equal(dbeta, torch.from_numpy(want_dy).bfloat16())
    assert torch.equal(dgamma, torch.from_numpy(want_dyx).bfloat16())
