"""L3 gradient codings: the ``encode`` / ``decode`` / ``codes`` plug-in contract and built-ins.

The reference imports an *external* ``codings`` module (``/root/reference/ps.py:16-18``) and
uses exactly three members of the object passed as ``code=``:

* ``code.encode(grad.data, **kw)`` in the backward hook (``ps.py:65-66,94``),
* ``code.decode(code_obj, cuda=bool)`` per rank's message (``ps.py:166``),
* ``code.codes = [...]`` — every rank's code for the current parameter, assigned before
  decoding (``ps.py:165``).

This module ships that contract as :class:`Coding` plus the built-ins the framework fuses into
its sm_90a kernels: :class:`Identity`, :class:`Cast`, :class:`Scale`, :class:`TopK`, block-wise :class:`QSGD` and
:class:`Sign`.  Each
built-in has

* a pure-PyTorch ``encode``/``decode`` (host slow path **and** the numerical oracle every CUDA
  kernel is tested against), and
* a :meth:`Coding.device_spec` describing the fixed binary wire layout the device path uses
  (no pickle, no size exchange — ``/root/reference/mpi_comms.py:150-158`` is eliminated).

Arbitrary user codings (any object with ``encode``/``decode``) keep working on the host path.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import Any, List, Optional

import numpy as np
import torch

__all__ = [
    "Coding", "Identity", "Cast", "Scale", "TopK", "QSGD", "Sign", "SVD", "DeviceCodeSpec", "TILE",
    "WIRE_F32", "WIRE_BF16", "WIRE_F16", "WIRE_E4M3", "WIRE_E5M2", "WIRE_I8", "WIRE_I4", "WIRE_B1",
    "KIND_DENSE", "KIND_SCALED", "KIND_TOPK", "KIND_QSGD", "KIND_SIGN", "wire_dtype_of", "wire_code_of", "tile_k", "philox4x32_10",
]

#: elements per tile of the flat arena; every parameter starts on a tile boundary and the
#: block-wise top-k selects inside one tile.  Must match ``PSB_TILE`` in csrc/kernels/common.cuh.
TILE = 2048

# wire element types (must match csrc/kernels/common.cuh); WIRE_I4 = two 4-bit codes per byte (block-wise QSGD only), WIRE_B1 =
# eight sign bits per byte (Sign only)
WIRE_F32, WIRE_BF16, WIRE_F16, WIRE_E4M3, WIRE_E5M2, WIRE_I8, WIRE_I4, WIRE_B1 = 0, 1, 2, 3, 4, 5, 6, 7
# coding kinds
KIND_DENSE, KIND_SCALED, KIND_TOPK, KIND_QSGD, KIND_SIGN = 0, 1, 2, 3, 4

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

    kind: int                 # KIND_DENSE | KIND_SCALED | KIND_TOPK | KIND_QSGD | KIND_SIGN
    wire: int                 # WIRE_* element type of the payload values (-1 = same as grad)
    ratio: float = 1.0        # top-k keep ratio (KIND_TOPK)
    error_feedback: bool = False
    levels: int = 0           # largest code magnitude (KIND_QSGD)
    seed: int = 0             # Philox key (KIND_QSGD)

    def resolved_wire(self, grad_dtype: torch.dtype) -> int:
        return wire_code_of(grad_dtype) if self.wire < 0 else self.wire

    def tile_capacity(self) -> int:
        """Entries reserved per tile on the wire (KIND_TOPK)."""
        return tile_k(self.ratio, TILE) if self.kind == KIND_TOPK else TILE

    def bytes_per_tile(self, grad_dtype: torch.dtype) -> int:
        if self.kind == KIND_QSGD:
            # 2048 codes (int8, or int4 two per byte) + a 16-byte header: fp32 scale, 12 zero bytes
            return (TILE if self.wire == WIRE_I8 else TILE // 2) + 16
        if self.kind == KIND_SIGN:
            return TILE // 8 + 16           # 2048 sign bits + a 16-byte header: fp32 scale, 12 zero bytes
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


_PHILOX_M0, _PHILOX_M1, _PHILOX_W0, _PHILOX_W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_U32 = 0xFFFFFFFF


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 (Random123): counter words ``c0..c3`` and key words ``k0, k1`` (integers or numpy arrays) → the four
    output words as uint64 numpy arrays holding 32-bit values.  Same rounds as ``psb::philox4x32_10`` in common.cuh."""
    c = [np.asarray(x, np.uint64) & np.uint64(_U32) for x in (c0, c1, c2, c3)]
    k0, k1 = (np.asarray(x, np.uint64) & np.uint64(_U32) for x in (k0, k1))
    m, sh = np.uint64(_U32), np.uint64(32)
    for _ in range(10):
        p0, p1 = np.uint64(_PHILOX_M0) * c[0], np.uint64(_PHILOX_M1) * c[2]
        c = [(p1 >> sh) ^ c[1] ^ k0, p1 & m, (p0 >> sh) ^ c[3] ^ k1, p0 & m]
        k0, k1 = (k0 + np.uint64(_PHILOX_W0)) & m, (k1 + np.uint64(_PHILOX_W1)) & m
    return c


class QSGD(Coding):
    """QSGD-style stochastic quantisation (Alistarh et al. 2017): ``sign · ‖g‖₂ · ξ/levels`` with ``ξ`` drawn so
    the code is an unbiased estimate of the gradient.

    ``blockwise=False`` (default): whole-tensor norm, int8 / int16 codes, host (generic-object) path only — the kind of user
    coding the reference's external ``codings`` module carried (SURVEY §2.2).

    ``blockwise=True``: every ``TILE``-element block of the flattened tensor is quantised against its own L2 norm, fused into the
    device engine's encode and update kernels.  ``levels`` in [1, 127]; ``levels <= 7`` travels as 4-bit two's-complement codes,
    two per byte (element ``2i`` in the low nibble, -8 = NaN), otherwise as int8 codes (-128 = NaN).  A wire tile is the 2048
    codes followed by a 16-byte header: the fp32 ``scale = norm / levels`` and 12 zero bytes (1040 or 2064 bytes per tile).
    The rules (DESIGN.md, wire numerics): ``norm`` is the L2 norm of the tile's finite elements (1 if none is non-zero),
    ``x = |g| / norm · levels``, ``q = sign(g) · (floor(x) + [u < x − floor(x)])``, ±Inf saturates to ±levels, NaN gets the NaN
    code, and ``u`` is word ``e & 3`` of Philox4x32-10 with counter ``(e >> 2, arena tile, step, rank)`` and key ``seed``
    (``None`` = 0), ``e`` the element's index in its tile.  ``decode`` returns ``q · scale``, so ``E[decode] == g``.

    :meth:`encode` is the kernels' oracle and the host engine's path; it returns ``{"wire": uint8 [ntiles, bytes_per_tile],
    "shape": ...}``, the exact bytes the device writes.  The device engine passes the arena tile, its step counter and the
    rank.  The host engine passes only ``name=``; then ``step`` is the number of earlier ``encode`` calls for that name in
    this object, ``rank`` the process rank of the initialised runtime (0 without one), and the first tile
    ``zlib.crc32(name)``, so that ranks, steps and parameters draw independent numbers.
    """

    def __init__(self, levels: int = 255, seed: Optional[int] = None, blockwise: bool = False):
        self.blockwise = bool(blockwise)
        if self.blockwise:
            if not 1 <= levels <= 127:
                raise ValueError("QSGD(blockwise=True) needs levels in [1, 127]")
            self.levels = int(levels)
            self.seed = 0 if seed is None else int(seed) & ((1 << 64) - 1)
            self.wire = WIRE_I4 if self.levels <= 7 else WIRE_I8
            self._calls = {}
            return
        if not 1 <= levels <= 32767:
            raise ValueError("levels must be in [1, 32767]")
        self.levels = int(levels)
        self._gen = torch.Generator().manual_seed(seed) if seed is not None else None

    def device_spec(self):
        if not self.blockwise:
            return None
        return DeviceCodeSpec(KIND_QSGD, self.wire, levels=self.levels, seed=self.seed)

    def _encode_blockwise(self, grad, name, step, rank, first_tile):
        if step is None:
            step = self._calls.get(name, 0)
            self._calls[name] = step + 1
        if rank is None:
            from . import runtime
            rank = runtime.rank() if runtime.is_initialized() else 0
        if first_tile is None:
            first_tile = zlib.crc32(name.encode()) if name is not None else 0
        flat = grad.detach().reshape(-1).float().cpu()
        n = flat.numel()
        nt = max(1, (n + TILE - 1) // TILE)
        g = torch.zeros(nt * TILE, dtype=torch.float32)
        g[:n] = flat
        g = g.view(nt, TILE)
        fin = torch.isfinite(g)
        a = torch.where(fin, g.abs(), torch.zeros_like(g))
        m = a.max(dim=1).values
        any_ = m > 0
        m = torch.where(any_, m, torch.ones_like(m))
        t = torch.where(fin, a / m[:, None], torch.zeros_like(g))
        # fp32 sum of t² in the kernel's order: 8 elements per thread in index order, xor butterfly over 32 lanes, 8 warps in order
        sq = (t * t).view(nt, 256, 8)
        s = sq[:, :, 0].clone()
        for j in range(1, 8):
            s = s + sq[:, :, j]
        s = s.view(nt, 8, 32)
        lane = torch.arange(32)
        for off in (16, 8, 4, 2, 1):
            s = s + s[:, :, lane ^ off]
        tot = s[:, 0, 0].clone()
        for w in range(1, 8):
            tot = tot + s[:, w, 0]
        # correctly rounded fp32 sqrt (= __fsqrt_rn): via float64, since torch's vectorised fp32 sqrt may be 1 ulp off
        r = torch.where(any_, torch.sqrt(tot.double()).float(), torch.ones_like(tot))
        lv = torch.tensor(float(self.levels), dtype=torch.float32)
        x = (t / r[:, None]) * lv
        fl = torch.floor(x)
        e = np.arange(TILE)
        tiles = (np.arange(nt, dtype=np.uint64) + np.uint64(first_tile))[:, None]
        words = philox4x32_10(e[None, :] >> 2, tiles, step, rank, self.seed & _U32, self.seed >> 32)
        w = np.choose(e & 3, words).astype(np.int64)                      # word e & 3 of the element's draw
        u = torch.from_numpy(w >> 8).float() * 2.0 ** -24
        qi = torch.clamp(fl.long() + (u < x - fl).long(), max=self.levels)
        qi = torch.where(torch.isinf(g), torch.full_like(qi, self.levels), qi)
        q = torch.where(torch.signbit(g), -qi, qi)
        nan_code, mask = (-8, 0xF) if self.wire == WIRE_I4 else (-128, 0xFF)
        q = torch.where(torch.isnan(g), torch.full_like(q, nan_code), q) & mask
        if self.wire == WIRE_I4:
            payload = (q[:, 0::2] | (q[:, 1::2] << 4)).to(torch.uint8)
        else:
            payload = q.to(torch.uint8)
        scale = m * (r / lv)
        fmax = torch.finfo(torch.float32).max
        scale = torch.where(scale > fmax, torch.full_like(scale, fmax), scale)
        header = torch.zeros(nt, 4, dtype=torch.float32)
        header[:, 0] = scale
        wire = torch.cat([payload, header.view(torch.uint8)], dim=1)
        return {"wire": wire, "shape": tuple(grad.shape), "levels": self.levels}

    def _decode_blockwise(self, code, cuda):
        wire = _as_tensor(code["wire"]).cpu()
        shape = tuple(int(d) for d in code["shape"])
        pay = wire.shape[1] - 16
        scale = wire[:, pay: pay + 4].contiguous().view(torch.float32)
        if pay == TILE // 2:
            b = wire[:, :pay].to(torch.int32)
            q = torch.stack([b & 0xF, b >> 4], dim=2).reshape(wire.shape[0], TILE)
            q = q - ((q & 0x8) << 1)                                          # sign-extend the nibbles
            nan = q == -8
        else:
            q = wire[:, :pay].contiguous().view(torch.int8).to(torch.int32)
            nan = q == -128
        f = torch.where(nan, torch.full(q.shape, float("nan")), q.float()) * scale
        n = math.prod(shape)
        return self._place(f.reshape(-1)[:n].reshape(shape), cuda)

    def encode(self, grad, name=None, step=None, rank=None, first_tile=None, **kwargs):
        if self.blockwise:
            return self._encode_blockwise(grad, name, step, rank, first_tile)
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
        if "wire" in code:
            return self._decode_blockwise(code, cuda)
        q = self._place(_as_tensor(code["q"]), cuda).float()
        norm = self._place(_as_tensor(code["norm"]), cuda).float()
        return (q * (norm / float(code["levels"]))).reshape(tuple(int(d) for d in code["shape"]))

    def __repr__(self):
        if self.blockwise:
            return f"QSGD(levels={self.levels}, blockwise=True)"
        return f"QSGD(levels={self.levels})"


class Sign(Coding):
    """Block-wise scaled sign with error feedback (1-bit SGD, Seide et al. 2014; EF-SignSGD, Karimireddy et al. 2019): one bit per
    element and one fp32 scale per ``TILE``-element block of the flattened tensor, fused into the device engine's kernels.

    A wire tile is 256 payload bytes, bit ``e & 7`` of byte ``e >> 3`` the sign bit of element ``e`` (so -0 sends 1, a NaN 0), then a
    16-byte header: the fp32 ``scale`` and 12 zero bytes (272 bytes per tile, 1/15 of a bf16 wire).  The rules (DESIGN.md, wire
    numerics): ``p = g + residual`` over the tile's real elements ``R``; ``scale`` is the mean of ``|p|`` over ``R``, computed as
    ``m * (sum of |p| / m) / |R|`` with ``m`` the abs-max, in the kernel's fixed order (0 when ``m == 0``, NaN when a NaN or ±Inf
    is in ``R``, at most FLT_MAX).  ``decode`` is ``bit ? -scale : +scale`` on ``R`` and +0 elsewhere.  With ``error_feedback=True``
    the coding keeps ``p - decode`` per parameter name and adds it to the next gradient of that name, so the compression error is
    sent later instead of lost.

    :meth:`encode` is the kernels' oracle and the host engine's path; it returns ``{"wire": uint8 [ntiles, 272], "shape": ...}``,
    the exact bytes the device writes.  ``real`` (a boolean mask over the tile-padded span) describes a custom arena placement;
    it defaults to ``index < numel``.
    """

    def __init__(self, error_feedback: bool = True):
        self.error_feedback = bool(error_feedback)
        self._residual = {}

    def device_spec(self):
        return DeviceCodeSpec(KIND_SIGN, WIRE_B1, error_feedback=self.error_feedback)

    def encode(self, grad, name=None, real=None, **kwargs):
        if self.error_feedback and name is None:
            raise ValueError("Sign(error_feedback=True).encode needs name= (the parameter the residual belongs to)")
        flat = grad.detach().reshape(-1).float().cpu().numpy()
        n = flat.size
        nt = max(1, -(-n // TILE))
        p = np.zeros(nt * TILE, np.float32)
        p[:n] = flat
        if self.error_feedback and name in self._residual:
            p = p + self._residual[name]
        real = np.arange(nt * TILE) < n if real is None else np.asarray(real, bool).reshape(-1)
        if real.size != nt * TILE:
            raise ValueError(f"real must cover the {nt * TILE} tile-padded elements")
        p, real = p.reshape(nt, TILE), real.reshape(nt, TILE)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            bad = (real & ~np.isfinite(p)).any(axis=1)
            m = np.where(real & np.isfinite(p), np.abs(p), np.float32(0)).max(axis=1)
            t = np.where(real, np.abs(p) / np.where(m > 0, m, np.float32(1))[:, None], np.float32(0)).astype(np.float32)
            # fp32 sum in the kernel's order: 8 elements per thread in index order, xor butterfly over 32 lanes, 8 warps in order
            t = t.reshape(nt, 256, 8)
            s = np.zeros((nt, 256), np.float32)
            for j in range(8):
                s = s + t[:, :, j]
            s = s.reshape(nt, 8, 32)
            lane = np.arange(32)
            for off in (16, 8, 4, 2, 1):
                s = s + s[:, :, lane ^ off]
            tot = s[:, 0, 0]
            for w in range(1, 8):
                tot = tot + s[:, w, 0]
            cnt = np.maximum(real.sum(axis=1), 1).astype(np.float32)
            scale = (m * (tot / cnt)).astype(np.float32)
        fmax = np.finfo(np.float32).max
        scale = np.where(m > 0, np.minimum(scale, fmax), np.float32(0)).astype(np.float32)
        scale = np.where(bad, np.uint32(0x7FFFFFFF).view(np.float32), scale)
        bits = np.signbit(p) & ~np.isnan(p) & real
        payload = np.packbits(bits.reshape(nt, TILE // 8, 8), axis=2, bitorder="little").reshape(nt, TILE // 8)
        header = np.zeros((nt, 4), np.float32)
        header[:, 0] = scale
        if self.error_feedback:
            with np.errstate(invalid="ignore"):
                dec = np.where(bits, -scale[:, None], scale[:, None])
                self._residual[name] = np.where(real, p - dec, np.float32(0)).astype(np.float32).reshape(-1)
        wire = np.concatenate([payload, header.view(np.uint8)], axis=1)
        return {"wire": torch.from_numpy(wire), "shape": tuple(grad.shape)}

    def decode(self, code, cuda=False, real=None):
        """The fp32 tensor ``bit ? -scale : +scale``; lanes outside ``real`` (default: past the tensor's end) are +0."""
        wire = _as_tensor(code["wire"]).cpu().numpy()
        shape = tuple(int(d) for d in code["shape"])
        nt = wire.shape[0]
        scale = wire[:, TILE // 8: TILE // 8 + 4].copy().view(np.float32)
        bits = np.unpackbits(wire[:, :TILE // 8], axis=1, bitorder="little").astype(bool)
        f = np.where(bits, -scale, scale).reshape(-1)
        n = math.prod(shape)
        real = np.arange(nt * TILE) < n if real is None else np.asarray(real, bool).reshape(-1)
        f = np.where(real, f, np.float32(0)).astype(np.float32)
        return self._place(torch.from_numpy(f[:n].copy()).reshape(shape), cuda)

    def __repr__(self):
        return f"Sign(error_feedback={self.error_feedback})"


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
