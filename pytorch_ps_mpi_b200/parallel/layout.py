"""Flat arena layout: every parameter packed, tile-aligned, into one contiguous index space.

The reference walks parameters one by one in reverse registration (= backward) order
(``/root/reference/ps.py:121-123``) and pays one message + several eager kernels per parameter.
Here all parameters live in ONE flat arena so a single kernel launch covers the whole model:

* parameters are laid out in **reverse registration order** (gradients that are ready first sit
  at the front of the arena);
* every parameter starts on a :data:`~pytorch_ps_mpi_b200.codings.TILE`-element boundary and owns
  an integral number of tiles, so a tile never straddles two parameters (per-tensor scales and
  block-wise top-k stay tile-local);
* a small ``[ntiles, 4]`` int32 table (parameter, valid elements, param-group, first tile)
  drives the kernels.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import torch

from ..codings import TILE


@dataclass
class ParamSlot:
    index: int            # position in arena order
    name: str
    param: torch.nn.Parameter
    group: int
    first_tile: int
    ntiles: int
    numel: int            # elements the parameter occupies in the arena (its storage span if it has a custom placement)
    strides: Optional[tuple] = None   # custom placement: the parameter is as_strided(shape, strides) over `numel` elements

    @property
    def offset(self) -> int:      # element offset in the arena
        return self.first_tile * TILE

    def view(self, flat: torch.Tensor) -> torch.Tensor:
        """The parameter-shaped view of ``flat``, this slot's ``numel`` elements of an arena (parameters, gradients or optimizer
        state), in the parameter's physical layout: the custom placement if the module asked for one, else the parameter's own
        strides when they are a dense permutation (e.g. channels_last conv weights, as cuDNN wants them), else contiguous."""
        p = self.param
        if self.strides is not None:
            return torch.as_strided(flat, p.shape, self.strides)
        if p.is_contiguous() or not _dense(p):
            return flat.view(p.shape)
        return torch.as_strided(flat, p.shape, p.stride())


def _dense(t: torch.Tensor) -> bool:
    """True if ``t``'s strides describe a dense, non-overlapping permutation of its shape."""
    if t.is_contiguous():
        return True
    dims = sorted(((st, sz) for st, sz in zip(t.stride(), t.shape) if sz > 1), key=lambda x: x[0])
    expect = 1
    for st, sz in dims:
        if st != expect:
            return False
        expect *= sz
    return True


class FlatLayout:
    def __init__(self, param_groups, names: Dict[int, str]):
        ordered = []
        for gi, g in enumerate(param_groups):
            for p in g["params"]:
                ordered.append((gi, p))
        ordered.reverse()                                    # backward order (ps.py:121-123)
        self.slots: List[ParamSlot] = []
        self.by_id: Dict[int, ParamSlot] = {}
        t = 0
        for i, (gi, p) in enumerate(ordered):
            n, strides = p.numel(), None
            # A module may ask for a custom physical placement of its parameter inside the arena
            # (``param.ps_arena_layout = (strides, span_numel)``): e.g. the ResNet stem keeps its [64,3,7,7] weight in the
            # zero-padded [64,176] GEMM layout its wgmma kernel TMA-loads, so the PS broadcast lands the weight directly in
            # the form the first forward GEMM consumes (no per-step re-layout).  Elements of the span the view does not
            # cover are padding: zero, zero gradient, untouched by SGD/Adam (0 stays 0).
            hint = getattr(p, "ps_arena_layout", None)
            if hint is not None:
                strides, n = tuple(int(x) for x in hint[0]), int(hint[1])
                reach = 1 + sum((sz - 1) * st for sz, st in zip(p.shape, strides))
                if len(strides) != p.dim() or reach > n:
                    raise ValueError(f"ps_arena_layout of {names.get(id(p))!r} does not fit its span")
            nt = max(1, (n + TILE - 1) // TILE)
            s = ParamSlot(i, names.get(id(p), f"param{i}"), p, gi, t, nt, n, strides)
            self.slots.append(s)
            self.by_id[id(p)] = s
            t += nt
        self.ntiles = t
        self.numel_padded = t * TILE
        self.nparams = len(self.slots)
        self.ngroups = len(param_groups)

    def plan_chunks(self, elem_bytes: int, chunk_bytes: int, single: bool = False, max_chunks: int = 48) -> List[List[ParamSlot]]:
        """Static chunks of the update pipeline: contiguous runs of WHOLE parameters in arena (= backward) order, each holding at
        least ``chunk_bytes`` of (tile-padded) parameter bytes — the last one takes the remainder — and at most ``max_chunks`` of
        them.  They depend on the layout only, so every rank computes the same plan.  ``single``: one chunk (no pipeline)."""
        total = self.numel_padded * elem_bytes
        target = max(int(chunk_bytes), TILE * elem_bytes, -(-total // max_chunks))
        if single:
            target = max(target, total)
        chunks: List[List[ParamSlot]] = []
        cur: List[ParamSlot] = []
        nbytes = 0
        for sl in self.slots:
            cur.append(sl)
            nbytes += sl.ntiles * TILE * elem_bytes
            if nbytes >= target:
                chunks.append(cur)
                cur, nbytes = [], 0
        if cur:
            chunks.append(cur)
        return chunks

    def tile_table(self) -> torch.Tensor:
        """``[ntiles, 4]`` int32: (param, valid, group, first_tile) — ``TileInfo`` in common.cuh."""
        tab = torch.empty(self.ntiles, 4, dtype=torch.int32)
        for s in self.slots:
            for k in range(s.ntiles):
                valid = min(TILE, s.numel - k * TILE)
                tab[s.first_tile + k] = torch.tensor([s.index, max(valid, 0), s.group, s.first_tile], dtype=torch.int32)
        return tab

    def tile_table_fast(self) -> torch.Tensor:
        """Vectorised construction of :meth:`tile_table` (BERT-size models have ~54k tiles)."""
        import numpy as np
        tab = np.empty((self.ntiles, 4), dtype=np.int32)
        for s in self.slots:
            k = np.arange(s.ntiles, dtype=np.int64)
            sl = slice(s.first_tile, s.first_tile + s.ntiles)
            tab[sl, 0] = s.index
            tab[sl, 1] = np.clip(s.numel - k * TILE, 0, TILE)
            tab[sl, 2] = s.group
            tab[sl, 3] = s.first_tile
        return torch.from_numpy(tab)
