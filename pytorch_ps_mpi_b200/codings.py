"""L3 gradient codings: the ``encode`` / ``decode`` / ``codes`` plug-in contract and built-ins.

The reference imports an *external* ``codings`` module (``/root/reference/ps.py:16-18``) and
uses exactly three members of the object passed as ``code=``:

* ``code.encode(grad.data, **kw)`` in the backward hook (``ps.py:65-66,94``),
* ``code.decode(code_obj, cuda=bool)`` per rank's message (``ps.py:166``),
* ``code.codes = [...]`` — every rank's code for the current parameter, assigned before
  decoding (``ps.py:165``).

This module ships that contract as :class:`Coding` plus the built-ins the framework fuses into
its sm_90a kernels: :class:`Identity`, :class:`Cast`, :class:`Scale`, :class:`TopK`.  Each
built-in has

* a pure-PyTorch ``encode``/``decode`` (host slow path **and** the numerical oracle every CUDA
  kernel is tested against), and
* a :meth:`Coding.device_spec` describing the fixed binary wire layout the device path uses
  (no pickle, no size exchange — ``/root/reference/mpi_comms.py:150-158`` is eliminated).

Arbitrary user codings (any object with ``encode``/``decode``) keep working on the host path.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, List, Optional

import torch

__all__ = [
    "Coding", "Identity", "Cast", "Scale", "TopK", "QSGD", "SVD", "DeviceCodeSpec", "TILE",
    "WIRE_F32", "WIRE_BF16", "WIRE_F16", "WIRE_E4M3", "WIRE_E5M2", "WIRE_I8",
    "KIND_DENSE", "KIND_SCALED", "KIND_TOPK", "wire_dtype_of", "wire_code_of", "tile_k",
]

#: elements per tile of the flat arena; every parameter starts on a tile boundary and the
#: block-wise top-k selects inside one tile.  Must match ``PSB_TILE`` in csrc/kernels/common.cuh.
TILE = 2048

# wire element types (must match csrc/kernels/common.cuh)
WIRE_F32, WIRE_BF16, WIRE_F16, WIRE_E4M3, WIRE_E5M2, WIRE_I8 = 0, 1, 2, 3, 4, 5
# coding kinds
KIND_DENSE, KIND_SCALED, KIND_TOPK = 0, 1, 2

_WIRE_TORCH = {
    WIRE_F32: torch.float32, WIRE_BF16: torch.bfloat16, WIRE_F16: torch.float16,
    WIRE_E4M3: torch.float8_e4m3fn, WIRE_E5M2: torch.float8_e5m2, WIRE_I8: torch.int8,
}
_WIRE_NAMES = {
    "fp32": WIRE_F32, "float32": WIRE_F32, "f32": WIRE_F32,
    "bf16": WIRE_BF16, "bfloat16": WIRE_BF16,
    "fp16": WIRE_F16, "float16": WIRE_F16, "half": WIRE_F16,
    "fp8": WIRE_E4M3, "fp8_e4m3": WIRE_E4M3, "e4m3": WIRE_E4M3, "float8_e4m3fn": WIRE_E4M3,
    "fp8_e5m2": WIRE_E5M2, "e5m2": WIRE_E5M2, "float8_e5m2": WIRE_E5M2,
    "int8": WIRE_I8, "i8": WIRE_I8,
}
_WIRE_MAX = {WIRE_E4M3: 448.0, WIRE_E5M2: 57344.0, WIRE_I8: 127.0, WIRE_F16: 65504.0}


def wire_code_of(dtype) -> int:
    """Map a torch dtype / string to a wire element code."""
    if isinstance(dtype, int):
        return dtype
    if isinstance(dtype, str):
        return _WIRE_NAMES[dtype.lower()]
    for k, v in _WIRE_TORCH.items():
        if v == dtype:
            return k
    raise ValueError(f"unsupported wire dtype {dtype!r}")


def wire_dtype_of(code: int) -> torch.dtype:
    return _WIRE_TORCH[code]


def tile_k(ratio: float, valid: int) -> int:
    """Entries kept in a tile that holds ``valid`` real elements (block-wise top-k)."""
    return max(1, min(valid, int(math.ceil(ratio * valid - 1e-9))))


@dataclass(frozen=True)
class DeviceCodeSpec:
    """Fixed binary wire layout of a built-in coding (consumed by the CUDA kernels)."""

    kind: int                 # KIND_DENSE | KIND_SCALED | KIND_TOPK
    wire: int                 # WIRE_* element type of the payload values (-1 = same as grad)
    ratio: float = 1.0        # top-k keep ratio (KIND_TOPK)
    error_feedback: bool = False

    def resolved_wire(self, grad_dtype: torch.dtype) -> int:
        return wire_code_of(grad_dtype) if self.wire < 0 else self.wire

    def tile_capacity(self) -> int:
        """Entries reserved per tile on the wire (KIND_TOPK)."""
        return tile_k(self.ratio, TILE) if self.kind == KIND_TOPK else TILE

    def bytes_per_tile(self, grad_dtype: torch.dtype) -> int:
        w = self.resolved_wire(grad_dtype)
        esz = torch.empty((), dtype=_WIRE_TORCH[w]).element_size()
        if self.kind == KIND_TOPK:
            # entry = value + index packed to 2x the value width (bf16+u16 / f32+u32)
            esz = 4 if esz <= 2 else 8
            n = self.tile_capacity() * esz
        else:
            n = TILE * esz
        return (n + 15) // 16 * 16


class Coding:
    """Base class of the coding plug-in interface (``ps.py:57,60,65-66,94,165-166``)."""

    #: every rank's code for the parameter being decoded, set by the optimizer (``ps.py:165``)
    codes: Optional[List[Any]] = None
    #: encode is a view / one elementwise pass: the host engine encodes small gradients inside the hook instead of on its pool
    cheap: bool = False

    def encode(self, grad: torch.Tensor, **kwargs) -> Any:   # pragma: no cover - interface
        raise NotImplementedError

    def decode(self, code: Any, cuda: bool = False) -> torch.Tensor:   # pragma: no cover
        raise NotImplementedError

    def device_spec(self) -> Optional[DeviceCodeSpec]:
        """Binary layout for the fused kernels, or ``None`` → host (pickle) slow path."""
        return None

    # helpers shared by built-ins ----------------------------------------------------
    @staticmethod
    def _place(t: torch.Tensor, cuda: bool) -> torch.Tensor:
        if cuda and torch.cuda.is_available() and not t.is_cuda:
            return t.cuda(non_blocking=True)
        return t

    def __repr__(self) -> str:
        return f"{type(self).__name__}()"


def _as_tensor(x) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x
    return torch.as_tensor(x)


class Identity(Coding):
    """Send the gradient as it is (dtype preserved)."""

    cheap = True

    def encode(self, grad, **kwargs):
        return {"grad": grad.detach()}

    def decode(self, code, cuda=False):
        g = _as_tensor(code["grad"])
        return self._place(g, cuda)

    def device_spec(self):
        return DeviceCodeSpec(KIND_DENSE, -1)


def _sat_cast(x: torch.Tensor, wire: int) -> torch.Tensor:
    """Cast to the wire type by the rules of ``DESIGN.md`` (wire numerics): round to nearest even; narrowing to fp16 / fp8 /
    int8 saturates finite values and +-Inf at +-max finite; a wire of the tensor's own dtype is an exact copy; NaN stays NaN
    (int8: the code -128)."""
    dt = _WIRE_TORCH[wire]
    if x.dtype == dt:
        return x
    if wire in (WIRE_E4M3, WIRE_E5M2, WIRE_F16):
        m = _WIRE_MAX[wire]
        return x.float().clamp(-m, m).to(dt)         # clamp keeps NaN
    if wire == WIRE_I8:
        r = x.float().round().clamp(-127, 127)       # torch.round: ties to even
        return torch.where(torch.isnan(r), torch.full_like(r, -128.0), r).to(torch.int8)   # no NaN -> int conversion
    return x.to(dt)


class Cast(Coding):
    """Down-cast the gradient to a narrower float on the wire (bf16 / fp16 / fp8).

    Round to nearest even.  fp16 and fp8 wires saturate finite values and +-Inf at +-max finite (e4m3 448, e5m2 57344,
    fp16 65504) when they narrow the gradient; bf16 and fp32 wires do not saturate (an fp32 value past the bf16 range
    becomes Inf).  A wire of the gradient's own dtype is an exact copy, Inf and NaN included.  NaN stays NaN.
    """

    cheap = True

    def __init__(self, dtype="bf16"):
        self.wire = wire_code_of(dtype)
        if self.wire == WIRE_I8:
            raise ValueError("Cast to int8 needs a scale: use Scale('int8')")

    def encode(self, grad, **kwargs):
        return {"v": _sat_cast(grad.detach(), self.wire), "dtype": str(grad.dtype)}

    def decode(self, code, cuda=False):
        v = _as_tensor(code["v"])
        return self._place(v, cuda).float()

    def device_spec(self):
        return DeviceCodeSpec(KIND_DENSE, self.wire)

    def __repr__(self):
        return f"Cast({_WIRE_TORCH[self.wire]})"


class Scale(Coding):
    """Per-tensor abs-max scaling into a narrow type (int8 / fp8 / fp16).

    ``wire = cast(grad / inv)`` with the fp32 ``inv = absmax / qmax``, which travels with the message;
    ``decode = wire * inv``.  ``absmax`` is the largest ``|g|`` over the FINITE elements (1 if none is non-zero), so
    an Inf element saturates to +-qmax, decodes to +-absmax and leaves the rest of the tensor its resolution.  The
    cast rounds to nearest even and saturates at +-qmax; NaN stays NaN (int8: the code -128, which decodes to NaN).
    """

    def __init__(self, dtype="int8"):
        self.wire = wire_code_of(dtype)
        if self.wire not in _WIRE_MAX:
            raise ValueError("Scale supports int8 / fp8_e4m3 / fp8_e5m2 / fp16")

    def encode(self, grad, **kwargs):
        g = grad.detach().float()
        qmax = _WIRE_MAX[self.wire]
        amax = torch.where(torch.isfinite(g), g.abs(), g.new_zeros(())).max() if g.numel() else g.new_zeros(())
        amax = torch.where(amax > 0, amax, torch.ones_like(amax))
        inv = amax / torch.full_like(amax, qmax)   # IEEE fp32 division (a Python-scalar divisor is a
        #                                            reciprocal-multiply on CUDA and differs by 1 ulp)
        q = _sat_cast(g / inv, self.wire)       # == g * (qmax/amax) up to fp32 rounding
        return {"q": q, "inv": inv.reshape(1)}

    def decode(self, code, cuda=False):
        q = self._place(_as_tensor(code["q"]), cuda)
        inv = self._place(_as_tensor(code["inv"]), cuda).float()
        f = q.float()
        if q.dtype == torch.int8:
            f = torch.where(q == -128, torch.full_like(f, float("nan")), f)
        return f * inv

    def device_spec(self):
        return DeviceCodeSpec(KIND_SCALED, self.wire)

    def __repr__(self):
        return f"Scale({_WIRE_TORCH[self.wire]})"


class TopK(Coding):
    """Magnitude top-k sparsification.

    Two flavours:

    * ``exact=False`` (default, fused on device): **block-wise** top-k — the flattened tensor is
      cut into ``TILE``-element blocks and each block keeps its ``ceil(ratio * valid)`` largest
      magnitudes (ties → lower index).  Fixed per-block capacity means a fixed-size wire slot —
      no size exchange round (``mpi_comms.py:150-158``) — and the PS decodes a block entirely in
      shared memory.
    * ``exact=True``: classic per-tensor ``k`` / ``ratio`` (host path only).

    ``values`` picks the payload float type (``bf16`` → 4-byte ``(u16 idx, bf16 val)`` entries,
    ``fp32`` → 8-byte ``(u32 idx, f32 val)`` entries).
    """

    def __init__(self, ratio: Optional[float] = None, k: Optional[int] = None,
                 values="fp32", exact: bool = False, error_feedback: bool = False):
        if (ratio is None) == (k is None):
            raise ValueError("give exactly one of ratio= or k=")
        if k is not None and not exact:
            raise ValueError("k= needs exact=True (block-wise top-k is ratio based)")
        if ratio is not None and not (0.0 < ratio <= 1.0):
            raise ValueError("ratio must be in (0, 1]")
        self.ratio, self.k, self.exact = ratio, k, exact
        self.wire = wire_code_of(values)
        if self.wire not in (WIRE_F32, WIRE_BF16):
            raise ValueError("TopK values must be fp32 or bf16")
        self.error_feedback = bool(error_feedback)
        self._residual = {}

    # -- oracle / host path -------------------------------------------------------------
    def _select_blockwise(self, flat: torch.Tensor):
        n = flat.numel()
        nt = (n + TILE - 1) // TILE
        pad = nt * TILE - n
        x = torch.cat([flat, flat.new_zeros(pad)]) if pad else flat
        x = x.view(nt, TILE)
        mag = x.abs().float()
        if pad:  # padded lanes must never win
            mag = mag.clone()
            mag.view(-1)[n:] = -1.0
        order = torch.sort(mag, dim=1, descending=True, stable=True).indices
        idx_parts, val_parts = [], []
        for t in range(nt):
            valid = min(TILE, n - t * TILE)
            kt = tile_k(self.ratio, valid)
            sel = torch.sort(order[t, :kt]).values
            idx_parts.append(sel + t * TILE)
            val_parts.append(x[t, sel])
        return torch.cat(idx_parts), torch.cat(val_parts)

    def encode(self, grad, name=None, **kwargs):
        g = grad.detach()
        flat = g.reshape(-1)
        if self.error_feedback:
            if name is None:
                # id(grad) of a temporary is recycled across parameters and steps: it would mix residuals
                raise ValueError("TopK(error_feedback=True).encode needs name= (the parameter the residual belongs to)")
            key = name
            res = self._residual.get(key)
            work = flat.float() if res is None else flat.float() + res
        else:
            work = flat
        if self.exact:
            k = self.k if self.k is not None else max(1, int(math.ceil(self.ratio * flat.numel())))
            k = min(k, flat.numel())
            idx = torch.sort(torch.topk(work.abs().float(), k, sorted=False).indices).values
            val = work[idx]
        else:
            idx, val = self._select_blockwise(work)
        val = val.to(_WIRE_TORCH[self.wire])
        if self.error_feedback:
            res = work.float().clone()
            res[idx] -= val.float()
            self._residual[key] = res
        return {"idx": idx.to(torch.int32), "val": val, "shape": tuple(g.shape)}

    def decode(self, code, cuda=False):
        idx = self._place(_as_tensor(code["idx"]), cuda).long()
        val = self._place(_as_tensor(code["val"]), cuda).float()
        shape = tuple(int(s) for s in code["shape"])
        out = torch.zeros(int(math.prod(shape)) if shape else 1, dtype=torch.float32, device=val.device)
        out.index_add_(0, idx, val)
        return out.view(shape)

    def device_spec(self):
        if self.exact:
            return None
        return DeviceCodeSpec(KIND_TOPK, self.wire, float(self.ratio), self.error_feedback)

    def __repr__(self):
        what = f"k={self.k}" if self.k is not None else f"ratio={self.ratio}"
        return f"TopK({what}, values={_WIRE_TORCH[self.wire]}, exact={self.exact})"


class QSGD(Coding):
    """QSGD-style stochastic quantisation (Alistarh et al. 2017): ``sign · ‖g‖₂ · ξ/levels`` with ``ξ`` drawn so
    the code is an unbiased estimate of the gradient.  Host (generic-object) path — the kind of user coding the
    reference's external ``codings`` module carried (SURVEY §2.2); the fused device codings are
    :class:`Cast` / :class:`Scale` / :class:`TopK`.
    """

    def __init__(self, levels: int = 255, seed: Optional[int] = None):
        if not 1 <= levels <= 32767:
            raise ValueError("levels must be in [1, 32767]")
        self.levels = int(levels)
        self._gen = torch.Generator().manual_seed(seed) if seed is not None else None

    def encode(self, grad, **kwargs):
        g = grad.detach().float().cpu()
        norm = g.norm()
        if float(norm) == 0.0 or not torch.isfinite(norm):
            q = torch.zeros(g.shape, dtype=torch.int16)
            return {"q": q, "norm": torch.zeros(1), "levels": self.levels, "shape": tuple(g.shape)}
        x = g.abs() / norm * self.levels                      # in [0, levels]
        low = x.floor()
        up = torch.rand(x.shape, generator=self._gen) < (x - low)      # stochastic rounding → unbiased
        q = (low + up.float()) * g.sign()
        dt = torch.int8 if self.levels <= 127 else torch.int16
        return {"q": q.to(dt), "norm": norm.reshape(1), "levels": self.levels, "shape": tuple(g.shape)}

    def decode(self, code, cuda=False):
        q = self._place(_as_tensor(code["q"]), cuda).float()
        norm = self._place(_as_tensor(code["norm"]), cuda).float()
        return (q * (norm / float(code["levels"]))).reshape(tuple(int(d) for d in code["shape"]))

    def __repr__(self):
        return f"QSGD(levels={self.levels})"


class SVD(Coding):
    """Rank-``r`` truncated SVD of every ≥2-D gradient (sent as ``U·S`` and ``Vᵀ``); 1-D gradients travel as is.
    Host path (ATOMO / PowerSGD family of the reference author's coding experiments, SURVEY §2.2)."""

    def __init__(self, rank: int = 4):
        if rank < 1:
            raise ValueError("rank must be >= 1")
        self.rank = int(rank)

    def encode(self, grad, **kwargs):
        g = grad.detach().float().cpu()
        if g.dim() < 2 or min(g.shape[0], g[0].numel()) <= self.rank:
            return {"dense": g, "shape": tuple(g.shape)}
        m = g.reshape(g.shape[0], -1)
        u, s, vh = torch.linalg.svd(m, full_matrices=False)
        r = self.rank
        return {"us": (u[:, :r] * s[:r]).contiguous(), "vh": vh[:r].contiguous(), "shape": tuple(g.shape)}

    def decode(self, code, cuda=False):
        shape = tuple(int(d) for d in code["shape"])
        if "dense" in code:
            return self._place(_as_tensor(code["dense"]), cuda).float().reshape(shape)
        us = self._place(_as_tensor(code["us"]), cuda).float()
        vh = self._place(_as_tensor(code["vh"]), cuda).float()
        return (us @ vh).reshape(shape)

    def __repr__(self):
        return f"SVD(rank={self.rank})"
