"""ResNet stem (7x7 / stride 2 / pad 3, 3 → 64 channels) on OUR wgmma kernels.

Default path (round 2): ``stem_conv_fused`` — ONE implicit-GEMM kernel (``psb_stem_fwd_kernel``, ``csrc/kernels/stem_kernels.cu``:
smem patch → swizzled A tile → ``wgmma`` → TMA-store epilogue that also produces the BatchNorm Σy / Σy²) and the implicit
weight gradient ``psb_stem_wgrad_kernel`` (the same A tile as an MN-major operand, accumulators resident in registers); no 1.13 GB patch matrix.

The convolution weight is kept **in the parameter arena in the [64,176] GEMM layout** the kernel TMA-loads (``STEM_STRIDES``: a
``[64,3,7,7]`` view with strides ``(176,1,24,3)``; the device engine honours ``param.ps_arena_layout``), so the parameter
server's broadcast lands it ready to use and, with ``ResNet.attach(optimizer)``, the kernel's weight load acquires the
``PARAMS_READY`` epoch itself — the first forward GEMM *is* the ``req.Wait()`` of the broadcast
(``/root/reference/mpi_comms.py:120-124``).

Fallback (``PSB200_STEM=im2col``, or widths the fused kernel does not cover): ``stem_conv`` — ``psb_im2col_stem`` builds the
``[N*OH*OW, 176]`` patch matrix, the product runs on ``psb_bcast_gemm``, the weight gradient is one library GEMM.
cuDNN is slow on this layer (C=3 defeats its tensor-core kernels).
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F

from . import ext
from .linear import bcast_linear

STEM_K = 176          # 7 kernel rows x 24 (21 real + 3 zero) + 8 zero columns (csrc/kernels/pool_kernels.cu)
#: strides of a [cout,3,7,7] weight stored as the zero-padded [cout,176] GEMM matrix: element (o,c,kh,kw) at o*176 + kh*24 + kw*3 + c
STEM_STRIDES = (STEM_K, 1, 24, 3)
# weight gradient of the fused stem through psb_stem_wgrad_kernel (default) or im2col + library GEMM (PSB200_STEM_WGRAD=im2col)
_IMPLICIT_WGRAD = os.environ.get("PSB200_STEM_WGRAD", "implicit").lower() != "im2col"


class _StemGemm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, w2d):
        y = bcast_linear(a, w2d)                       # [M,176] x [64,176]^T on wgmma
        ctx.save_for_backward(a)
        return y

    @staticmethod
    def backward(ctx, gy):
        (a,) = ctx.saved_tensors
        gw = gy.t() @ a if ctx.needs_input_grad[1] else None     # [64,M] x [M,176]; no transpose copy (4.1 ms → 0.28 ms)
        return None, gw


def stem_supported(x: torch.Tensor, conv: torch.nn.Conv2d) -> bool:
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] == 3
            and x.is_contiguous(memory_format=torch.channels_last) and not x.requires_grad
            and conv.weight.dtype == torch.bfloat16 and conv.bias is None and conv.kernel_size == (7, 7)
            and conv.stride == (2, 2) and conv.padding == (3, 3) and conv.dilation == (1, 1) and conv.groups == 1)


def _w2d(weight: torch.Tensor) -> torch.Tensor:
    """[cout,3,7,7] → [cout,176]: (kh | kw,c) rows padded 21→24, then 8 zero columns (the layout psb_im2col_stem writes)."""
    cout = weight.shape[0]
    w2d = F.pad(weight.permute(0, 2, 3, 1).reshape(cout, 7, 21), (0, 3)).reshape(cout, 168)
    return F.pad(w2d, (0, STEM_K - 168)).contiguous()


def in_gemm_layout(weight: torch.Tensor) -> bool:
    return tuple(weight.stride()) == STEM_STRIDES and weight.shape[1:] == (3, 7, 7)


def _w2d_of(weight: torch.Tensor) -> torch.Tensor:
    """The [cout,176] GEMM matrix of ``weight``: a zero-copy view when the weight already lives in that layout."""
    w = weight.detach()
    if in_gemm_layout(w) and w.data_ptr() % 16 == 0:
        return torch.as_strided(w, (w.shape[0], STEM_K), (STEM_K, 1))
    return _w2d(w)


class _StemFused(torch.autograd.Function):
    """One implicit-GEMM kernel (``csrc/kernels/stem_kernels.cu``) instead of im2col + GEMM; also returns the BatchNorm
    sums of its output.  Backward: the implicit weight-gradient kernel (no patch matrix), returned in the GEMM layout."""

    @staticmethod
    def forward(ctx, x, weight, flag_ptr, epoch):
        y, sums = ext.cuda().stem_fwd(x, _w2d_of(weight), True, flag_ptr, epoch, 900.0)
        ctx.save_for_backward(x)
        ctx.cout = weight.shape[0]
        ctx.gout = getattr(weight, "ps_grad_out", None) if in_gemm_layout(weight) else None
        ctx.mark_non_differentiable(sums)
        return y, sums

    @staticmethod
    def backward(ctx, gy, _gsums):
        (x,) = ctx.saved_tensors
        gw = None
        if ctx.needs_input_grad[1]:
            if not gy.is_contiguous(memory_format=torch.channels_last):
                gy = gy.contiguous(memory_format=torch.channels_last)
            if _IMPLICIT_WGRAD:
                out = ctx.gout() if ctx.gout is not None else None     # the stem weight's wire-arena slot (GEMM layout) or None
                if out is not None:
                    out = torch.as_strided(out, (ctx.cout * STEM_K,), (1,))
                gw2d = stem_wgrad_implicit(x, gy, out)
            else:
                a = ext.cuda().im2col_stem(x)
                g2 = gy.permute(0, 2, 3, 1).reshape(-1, gy.shape[1])      # NHWC view of the channels-last gradient
                gw2d = g2.t() @ a
            # [cout,176] → the logical [cout,3,7,7] gradient, still in the GEMM layout (zero-copy into the wire arena's order)
            gw = torch.as_strided(gw2d, (ctx.cout, 3, 7, 7), STEM_STRIDES)
        return None, gw, None, None


def stem_wgrad_implicit(x: torch.Tensor, gy: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """``dW2d [64,176]`` (bf16) of the stem from ``psb_stem_wgrad_kernel`` — no patch matrix.  ``out``: a contiguous
    bf16 buffer of 64*176 elements to write into (the PS wire arena slot of the weight)."""
    m = ext.cuda()
    partial = m.stem_wgrad(x, gy)                                         # [grid,176,64] fp32
    return m.stem_wgrad_finalize(partial, out)                            # Σ partials, transpose, cast: one kernel


def stem_fused_supported(x: torch.Tensor, conv: torch.nn.Conv2d) -> bool:
    return stem_supported(x, conv) and conv.out_channels == 64 and x.shape[3] % 8 == 0 and x.shape[3] <= 256


def stem_conv_fused(x: torch.Tensor, weight: torch.Tensor, flag_ptr: int = 0, epoch: int = 0):
    """``(F.conv2d(x, weight, stride=2, padding=3), sums)`` where ``sums`` = per-channel Σy | Σy² (fp32, 128 values)
    for the BatchNorm that follows (``FusedBatchNormAct2d.forward(y, sums=sums)``).  ``flag_ptr`` / ``epoch``: the
    ``PARAMS_READY`` slot the kernel acquires before its weight load (``DeviceEngine.gate()``)."""
    return _StemFused.apply(x, weight, flag_ptr, epoch)


def stem_conv(x: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """``F.conv2d(x, weight, stride=2, padding=3)`` for a 3-channel channels-last bf16 ``x`` (no input grad)."""
    n, _, h, w = x.shape
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    cout = weight.shape[0]
    a = ext.cuda().im2col_stem(x)                                             # [n*oh*ow, 176]
    w2d = F.pad(weight.permute(0, 2, 3, 1).reshape(cout, 7, 21), (0, 3)).reshape(cout, 168)   # (kh | kw,c) rows padded 21→24
    w2d = F.pad(w2d, (0, STEM_K - 168))
    y = _StemGemm.apply(a, w2d.contiguous())                                  # [n*oh*ow, cout] == NHWC
    return y.view(n, oh, ow, cout).permute(0, 3, 1, 2)                        # logical NCHW, channels_last memory
