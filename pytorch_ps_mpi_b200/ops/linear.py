"""``BcastLinear``: a linear layer whose forward GEMM is the hand-written wgmma kernel
(``csrc/kernels/bcast_gemm.cu``) and whose weight operand is consumed straight out of the
symmetric parameter arena the parameter server broadcasts into.

With a device-engine optimizer attached (:meth:`BcastLinear.attach`), the kernel's TMA producer
acquires the ``PARAMS_READY`` epoch flag itself, so ``opt.step()`` on a worker no longer queues a
separate wait kernel: the first forward GEMM *is* the ``req.Wait()`` of the broadcast
(``/root/reference/mpi_comms.py:120-124``) and everything stream-ordered after it sees the fresh
weights.  ``pull=True`` makes the weight tensor map point at the SERVER's arena (mapped over
NVLink), i.e. the worker's TMA engine pulls the tiles across the switch directly into shared
memory.

Backward is plain library GEMMs (cuBLAS via ``torch.matmul``) — only the forward is on the named
hot path.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ext


class _BcastLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x2d, weight, bias, relu, w_ptr, flag_ptr, epoch, variant):
        m = ext.cuda()
        N, K = weight.shape
        y = m.bcast_gemm(x2d, w_ptr or weight.data_ptr(), N, K, bias, relu, flag_ptr, epoch, 30.0, variant)
        ctx.save_for_backward(x2d, weight, y if relu else None)
        ctx.relu, ctx.has_bias = relu, bias is not None
        ctx.gout = getattr(weight, "ps_grad_out", None) if weight.is_contiguous() else None
        return y

    @staticmethod
    def backward(ctx, gy):
        x2d, weight, y = ctx.saved_tensors
        if ctx.relu:
            gy = gy * (y > 0).to(gy.dtype)
        gx = gy @ weight if ctx.needs_input_grad[0] else None
        gw = None
        if ctx.needs_input_grad[1]:
            out = ctx.gout() if ctx.gout is not None else None
            # PS device engine attached (Identity wire): the dW GEMM writes straight into the wire arena (no encode pass)
            gw = torch.mm(gy.t(), x2d, out=out) if out is not None else gy.t() @ x2d
        gb = gy.sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb, None, None, None, None, None


def bcast_linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, relu: bool = False,
                 w_ptr: int = 0, flag_ptr: int = 0, epoch: int = 0, variant: int = 0) -> torch.Tensor:
    """``act(x @ weight.T + bias)`` on wgmma (bf16 in, fp32 accumulate, bf16 out).

    ``variant``: 0 = auto (CTA pairs sharing the weight tile when M >= 256), 1 = one CTA per tile, 2 = CTA pairs.  Bits 4-7
    select the epilogue (``csrc/kernels/bcast_gemm.cu``: 0 = auto → TMA store, 1 = staged full-line stores, 3 = TMA store,
    4 = direct stores from the accumulator fragment, kept for A/B; ``bench/gemm_variants.py``)."""
    if not (x.is_cuda and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and weight.is_contiguous()
            and weight.shape[1] % 8 == 0):
        y = F.linear(x, weight, bias)          # shapes/dtypes the kernel does not cover
        return F.relu(y) if relu else y
    shp = x.shape
    x2d = x.reshape(-1, shp[-1])
    if not x2d.is_contiguous() or x2d.data_ptr() % 16:
        x2d = x2d.contiguous()
    y = _BcastLinearFn.apply(x2d, weight, bias, relu, w_ptr, flag_ptr, epoch, variant)
    return y.view(*shp[:-1], weight.shape[0])


class BcastLinear(nn.Linear):
    """Drop-in ``nn.Linear`` (same parameters / state_dict) running on the wgmma GEMM."""

    def __init__(self, in_features, out_features, bias=True, relu=False, **kw):
        super().__init__(in_features, out_features, bias=bias, **kw)
        self.relu = relu
        self._engine = None
        self._pull = False
        self._gate = True

    def attach(self, optimizer, pull: bool = False, gate: bool = True) -> "BcastLinear":
        """Bind this layer to ``optimizer``'s device engine.

        ``gate=True``: the kernel's TMA producer acquires the broadcast epoch itself and workers stop queueing
        the separate wait kernel — only valid when this layer is the FIRST consumer of parameters in the
        forward pass (an MLP's first layer; NOT BERT's first linear, whose embeddings are read earlier).
        ``gate=False``: the engine keeps its wait kernel; the layer just runs on the wgmma GEMM.
        ``pull=True``: weight tiles are TMA-loaded from the server's arena over NVLink."""
        eng = getattr(optimizer, "_engine", None)
        if eng is None:
            raise ValueError("attach() needs an optimizer running the device engine")
        self._engine, self._pull, self._gate = eng, pull, gate
        if gate:
            eng.register_gate(self)
        return self

    def forward(self, x):
        eng = self._engine
        if eng is None or not self.weight.is_cuda:
            return bcast_linear(x, self.weight, self.bias, self.relu)
        flag_ptr, epoch = eng.gate() if self._gate else (0, 0)
        w_ptr = eng.peer_param_ptr(self.weight, 0) if (self._pull and eng.size > 1) else 0
        return bcast_linear(x, self.weight, self.bias, self.relu, w_ptr, flag_ptr, epoch)

    @classmethod
    def from_linear(cls, lin: nn.Linear, relu: bool = False) -> "BcastLinear":
        new = cls(lin.in_features, lin.out_features, bias=lin.bias is not None, relu=relu,
                  device=lin.weight.device, dtype=lin.weight.dtype)
        new.weight, new.bias = lin.weight, lin.bias
        return new


def convert_first_linear(model: nn.Module, optimizer=None, relu: bool = False, pull: bool = False,
                         gate: bool = True) -> Optional[BcastLinear]:
    """Swap the FIRST ``nn.Linear`` of ``model`` (the first forward GEMM) for a :class:`BcastLinear`
    sharing the same parameters, and — given a device-engine optimizer — gate it on the broadcast."""
    for parent in model.modules():
        for name, child in list(parent.named_children()):
            if isinstance(child, nn.Linear) and not isinstance(child, BcastLinear):
                new = BcastLinear.from_linear(child, relu=relu)
                setattr(parent, name, new)
                if optimizer is not None and getattr(optimizer, "_engine", None) is not None:
                    new.attach(optimizer, pull=pull, gate=gate)
                return new
    return None
