"""``FusedBatchNormAct2d``: BatchNorm2d (+ residual add) (+ ReLU) in hand-written channels-last bf16
kernels (``csrc/kernels/bn_kernels.cu``), forward and backward.

ATen's channels-last BatchNorm plus the separate add / ReLU kernels are a large share of a ResNet-18
step; fusing them turns 5-6 HBM passes per
BN-add-ReLU into 3 (forward) and the backward's 4 kernels into 2 passes over ``dy``/``x``.

Same parameters / buffers / ``state_dict`` as ``nn.BatchNorm2d``; running statistics stay fp32 even
after ``model.bfloat16()``.  Any input the kernels do not cover (CPU, fp32, NCHW, C % 8 != 0) takes
the stock ``F.batch_norm`` path with identical semantics.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ext


class _FusedBN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, res, gamma, beta, running_mean, running_var, eps, momentum, relu, training, sums=None):
        m = ext.cuda()
        if sums is not None and training:    # Σx / Σx² came out of the producer's epilogue (fused stem)
            y, mean, rstd, mask = m.bn_forward_presummed(x, res, gamma, beta, running_mean, running_var, eps, momentum, relu, sums)
        else:
            y, mean, rstd, mask = m.bn_forward(x, res, gamma, beta, running_mean, running_var, eps, momentum, relu, training)
        # ReLU: the backward needs only the sign of y — a 1-bit mask (1/16 of y's bytes) written by the forward kernel
        ctx.save_for_backward(x, (mask if mask is not None else y) if relu else None, gamma, mean, rstd)
        ctx.relu, ctx.has_res = relu, res is not None
        # PS device engine attached (Identity wire): dgamma / dbeta are written straight into the wire arena (no encode pass)
        ctx.gout = (getattr(gamma, "ps_grad_out", None), getattr(beta, "ps_grad_out", None))
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, gamma, mean, rstd = ctx.saved_tensors
        m = ext.cuda()
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        og = ctx.gout[0]() if ctx.gout[0] is not None else None
        ob = ctx.gout[1]() if ctx.gout[1] is not None else None
        dx, dres, dgamma, dbeta = m.bn_backward(dy, x, y if ctx.relu else x, gamma, mean, rstd, ctx.relu, ctx.has_res, og, ob)
        return dx, (dres if ctx.has_res else None), dgamma, dbeta, None, None, None, None, None, None, None


class _FusedBNMaxPool(torch.autograd.Function):
    """Training BN (sums from the producer) + ReLU + 3x3/s2/p1 max-pool: the ResNet stem tail without its full-resolution
    output or gradient.  Saves x and the pooled taps, no ReLU mask."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, eps, momentum, sums):
        y, mean, rstd, arg = ext.cuda().bn_forward_presummed(x, None, gamma, beta, running_mean, running_var, eps, momentum, True,
                                                             sums, pool=True)
        ctx.save_for_backward(x, arg, gamma, mean, rstd)
        ctx.gout = (getattr(gamma, "ps_grad_out", None), getattr(beta, "ps_grad_out", None))
        return y

    @staticmethod
    def backward(ctx, dy):
        x, arg, gamma, mean, rstd = ctx.saved_tensors
        if not dy.is_contiguous(memory_format=torch.channels_last):
            dy = dy.contiguous(memory_format=torch.channels_last)
        og = ctx.gout[0]() if ctx.gout[0] is not None else None
        ob = ctx.gout[1]() if ctx.gout[1] is not None else None
        dx, _, dgamma, dbeta = ext.cuda().bn_backward(dy, x, x, gamma, mean, rstd, True, False, og, ob, pool_arg=arg)
        return dx, dgamma, dbeta, None, None, None, None, None


def _kernel_ok(x: torch.Tensor, res: Optional[torch.Tensor], weight) -> bool:
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and weight is not None
            and weight.dtype == torch.bfloat16 and x.shape[1] % 8 == 0 and x.shape[1] <= 2048
            and x.is_contiguous(memory_format=torch.channels_last)
            and (res is None or (res.dtype == torch.bfloat16 and res.shape == x.shape
                                 and res.is_contiguous(memory_format=torch.channels_last))))


class FusedBatchNormAct2d(nn.BatchNorm2d):
    """``y = relu?(BN(x) [+ residual])`` — drop-in for ``nn.BatchNorm2d`` with optional fused epilogue."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, relu: bool = False, **kw):
        super().__init__(num_features, eps=eps, momentum=momentum, affine=True, track_running_stats=True, **kw)
        self.relu = relu
        # num_batches_tracked is only an input of the computation when momentum is None (cumulative average); with a fixed
        # momentum it is bookkeeping, so the kernel path counts on the host and writes the buffer when somebody looks
        # (state_dict / eval fallback) instead of launching one tiny add kernel per layer per step (20 per ResNet-18 step)
        self._nbt_pending = 0

    def _flush_batches_tracked(self):
        if self._nbt_pending and self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(self._nbt_pending)
        self._nbt_pending = 0

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        self._flush_batches_tracked()
        super()._save_to_state_dict(destination, prefix, keep_vars)

    def _load_from_state_dict(self, *args, **kwargs):
        self._nbt_pending = 0
        super()._load_from_state_dict(*args, **kwargs)

    def _apply(self, fn, *a, **k):
        super()._apply(fn, *a, **k)
        # statistics stay fp32 whatever the parameter dtype becomes (model.bfloat16())
        for name in ("running_mean", "running_var"):
            b = getattr(self, name)
            if b is not None and b.dtype != torch.float32:
                setattr(self, name, b.float())
        return self

    def _count_batch(self):
        if self.training and self.num_batches_tracked is not None:
            if self.momentum is None:
                self.num_batches_tracked.add_(1)
            else:
                self._nbt_pending += 1

    def maxpool_ok(self, x: torch.Tensor) -> bool:
        """Whether :meth:`forward_maxpool` covers ``x``: training, ReLU, the kernels' layout and even H and W."""
        return (self.training and self.relu and self.running_mean is not None and _kernel_ok(x, None, self.weight)
                and x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0)

    def forward_maxpool(self, x: torch.Tensor, sums: torch.Tensor) -> torch.Tensor:
        """``max_pool2d(self(x, sums=sums), 3, 2, 1)`` in one pass forward and two backward, bit for bit (needs
        :meth:`maxpool_ok`)."""
        self._count_batch()
        return _FusedBNMaxPool.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps,
                                     self.momentum if self.momentum is not None else 0.1, sums)

    def forward(self, x: torch.Tensor, residual: Optional[torch.Tensor] = None,
                sums: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``sums``: fp32 ``[2C]`` = Σx | Σx² over N·H·W already computed by the producer of ``x``."""
        if _kernel_ok(x, residual, self.weight) and (self.training or self.running_mean is not None):
            self._count_batch()
            return _FusedBN.apply(x, residual, self.weight, self.bias, self.running_mean, self.running_var,
                                  self.eps, self.momentum if self.momentum is not None else 0.1, self.relu, self.training,
                                  sums)
        self._flush_batches_tracked()
        rm, rv = self.running_mean, self.running_var
        w, b = self.weight, self.bias
        if rm is not None and rm.dtype != x.dtype and not x.is_cuda:
            w, b = w.to(rm.dtype), b.to(rm.dtype)
            y = F.batch_norm(x.to(rm.dtype), rm, rv, w, b, self.training, self.momentum or 0.1, self.eps).to(x.dtype)
        else:
            y = F.batch_norm(x, rm, rv, w, b, self.training, self.momentum or 0.1, self.eps)
        if residual is not None:
            y = y + residual
        return F.relu(y) if self.relu else y
