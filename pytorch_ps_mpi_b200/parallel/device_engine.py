"""Device engine: the GPU hot path behind ``MPI_PS.step()``.

Per step, per rank (nothing on this path touches the host after the launches are queued, and
nothing goes through NCCL/MPI):

1. **backward hooks** (``ps.py:65-66,98-101`` in the reference: encode on a thread pool) collect
   gradients into buckets; each full bucket is encoded by ONE ``psb_encode_kernel`` launch on a
   side stream straight into this rank's *symmetric wire arena* (cast / abs-max scale /
   block-wise top-k), overlapping with the rest of backward;
2. ``step()`` raises this rank's ``GRAD_READY`` epoch flag (``st.release.sys`` into the server's
   signal pad — the ``Igatherv`` post of ``mpi_comms.py:88``);
3. every rank that serves the chunk in the static serve plan (``_make_plan``: rank 0 in ``mode='ps'``, every rank in
   ``mode='allgather'``, every rank for its own share in ``mode='sharded'``) launches ``psb_update_kernel`` once over its
   tiles: wait flags → pull every rank's wire tiles over NVLink (or one ``multimem.ld_reduce`` through the switch) → decode +
   rank-ordered fp32 sum → SGD/Adam on fp32 master state → publish the new parameter tiles into every rank's *symmetric
   parameter arena* (``multimem.st`` or peer stores; ``allgather``: its own) → the plan's completion signal on the last
   chunk (``PARAMS_READY``; ``CONSUMED`` in ``allgather``; a counted ``PARAMS_READY`` add in ``sharded``);
4. workers queue a one-thread wait kernel on their compute stream (the ``req.Wait()`` of
   ``mpi_comms.py:121``); the model's parameters ARE views of the parameter arena, so the next
   forward reads the fresh weights with no copy.

``mode='async'`` (AsySG-InCon, ``README.md:56-81``): rank 0 is a dedicated server; a device-side
``select`` kernel waits until ``quota`` workers (ANY source) have posted a gradient, the update
kernel sums exactly those, publishes parameters + version and acknowledges the contributors;
workers never wait for parameters (inconsistent reads) — only for the ack of their previous
gradient before overwriting their wire arena.
"""
from __future__ import annotations

import contextlib
import math
import os
import time
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple

import torch

from .. import runtime
from ..codings import KIND_DENSE, KIND_QSGD, KIND_SCALED, KIND_SIGN, TILE, WIRE_BF16, WIRE_F16, WIRE_F32, wire_code_of
from ..ops import ext
from ..utils.misc import CudaStepTimer, MicroBatchCounter, raise_collectively
from .layout import FlatLayout
from .symmetric import SymmetricArena

_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
_DONE_EPOCH = 1 << 62
# launch modes of psb_update_kernel (must match csrc/kernels/common.cuh; the extension exports the same names)
OPT_SGD, OPT_ADAM = 0, 1
BCAST_LOCAL, BCAST_UNICAST, BCAST_MULTICAST = 0, 1, 2
REDUCE_P2P, REDUCE_NVLS = 0, 1
SIGNAL_NONE, SIGNAL_PARAMS_READY, SIGNAL_CONSUMED = 0, 1, 2


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


# ---- what the engine needs to know about each optimizer (``MPI_PS.optim``) ----
def _sgd_group(g, t):
    return [float(g["lr"]), float(g["weight_decay"]), float(g["momentum"]), float(g["dampening"]),
            0.0, 0.0, 0.0, 0.0, float(bool(g["nesterov"])), 0.0, float(t == 1)]


def _adam_step_size(g, t):
    b1, b2 = g["betas"]
    return float(g["lr"]) * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)     # ps.py:257-259


def _adam_group(g, t):
    b1, b2 = g["betas"]
    return [float(g["lr"]), float(g["weight_decay"]), 0.0, 0.0, float(b1), float(b2),
            float(g["eps"]), _adam_step_size(g, t), 0.0, float(bool(g.get("amsgrad", False))), float(t == 1)]


def _adamw_bias(g, t):
    """``(s, c2)`` of step ``t``: ``lr / (1 - β1^t)`` and ``sqrt(1 - β2^t)``, in double as ``torch.optim.AdamW`` forms them."""
    b1, b2 = g["betas"]
    return float(g["lr"]) / (1 - b1 ** t), (1 - b2 ** t) ** 0.5


def _adamw_group(g, t):
    """The AdamW slot layout of ``GroupHyper`` (csrc/kernels/common.cuh); the binding rounds each entry to fp32 once."""
    b1, b2 = g["betas"]
    lr, wd = float(g["lr"]), float(g["weight_decay"])
    s, c2 = _adamw_bias(g, t)
    return [lr, 1 - lr * wd, 1 - b1, 1 - b2, c2, float(b2), float(g["eps"]), s, 0.0,
            float(bool(g.get("amsgrad", False))), 0.0]


def _any(key):
    return lambda groups: any(g.get(key, 0) for g in groups)


class _OptimSpec(NamedTuple):
    code: int                                       # psb_update_kernel's optimizer id (OPT_* of common.cuh)
    buffers: Tuple[Tuple[str, str, Callable], ...]  # (opt.state key, engine buffer, needed(param_groups)) of the fp32 state
    step_key: bool                                  # opt.state[p] carries "step" next to the buffers
    group: Callable[[dict, int], List[float]]       # the group's 11-entry kernel tuple at step t
    per_param: Callable[[dict, int], Tuple[float, float]]   # a parameter's param_hyper pair at its own step t
    cache_key: Optional[Callable[[dict], tuple]]    # group fields the tuple depends on after step 1 (None: it changes every step)


_ADAM_BUFFERS = (("exp_avg", "buf0", lambda groups: True), ("exp_avg_sq", "buf1", lambda groups: True),
                 ("max_exp_avg_sq", "buf2", _any("amsgrad")))
_OPTIMS = {
    "sgd": _OptimSpec(OPT_SGD, (("momentum_buffer", "buf0", _any("momentum")),), False, _sgd_group,
                      lambda g, t: (0.0, 1.0 if t == 1 else 0.0),
                      lambda g: (g["lr"], g["weight_decay"], g["momentum"], g["dampening"], g["nesterov"])),
    "adam": _OptimSpec(OPT_ADAM, _ADAM_BUFFERS, True, _adam_group,
                       lambda g, t: (_adam_step_size(g, t), 1.0 if t == 1 else 0.0), None),
    "adamw": _OptimSpec(2,                         # OPT_ADAMW (the extension exports it; tests/test_adamw.py checks)
                        _ADAM_BUFFERS, True, _adamw_group, _adamw_bias, None),
}


class DeviceEngine:
    def __init__(self, opt, master_fp32: bool = True, reduce: str = "auto"):
        self.opt = opt
        self.m = ext.cuda()
        self.world = runtime.world()
        self.rank, self.size = opt.rank, opt.size
        if self.size > self.m.MAX_RANKS:
            raise ValueError(f"device engine supports up to {self.m.MAX_RANKS} ranks per server")
        if len(opt.param_groups) > self.m.MAX_GROUPS:
            raise ValueError(f"device engine supports up to {self.m.MAX_GROUPS} param groups")
        self.mode = opt.mode
        # mode='sharded': every rank serves one contiguous share of every chunk (N = 1 is mode='ps')
        self.sharded = self.mode == "sharded" and opt.size > 1
        names = {id(p): n for n, p in opt._named.items()}
        self.layout = FlatLayout(opt.param_groups, names)
        p0 = self.layout.slots[0].param
        self.device, self.dtype = p0.device, p0.dtype
        self.dt = _DT[self.dtype]
        self.psz = p0.element_size()
        self.spec = opt.code.device_spec()
        self.kind = self.spec.kind
        self.wire = self.spec.resolved_wire(self.dtype)
        self.bpt = self.spec.bytes_per_tile(self.dtype)
        self.cap = self.spec.tile_capacity()
        # bounded device spins: a dead peer must never hang the GPU, but an honest stall (rank-0 validation, a
        # checkpoint, a slow data loader) must not poison the flags either — hence a long default, surfaced by
        # _poll_error() every few steps instead of silently disabling synchronisation
        self.timeout_s = float(os.environ.get("PSB200_DEVICE_TIMEOUT", "900"))
        self.chunk_bytes = int(os.environ.get("PSB200_CHUNK_BYTES", os.environ.get("PSB200_BUCKET_BYTES", 4 << 20)))
        self.pipeline = bool(getattr(opt, "pipeline", True)) and os.environ.get("PSB200_PIPELINE", "1") != "0" \
            and self.mode in ("ps", "allgather", "sharded")
        L = self.layout
        nt, n_pad = L.ntiles, L.numel_padded
        self._check_same_layout_everywhere()

        # ---- symmetric block: [signal pad | scales | wire arena | parameter arena] ----
        self.off_signal = 0
        self.off_scales = _align(self.m.SIGNAL_SLOTS * 8)
        self.off_wire = self.off_scales + _align(max(L.nparams, 1) * 4)
        self.off_param = self.off_wire + _align(nt * self.bpt)
        total = self.off_param + _align(n_pad * self.psz)
        # consistent reads (README.md:79-81 "a buffered broadcast"): the server publishes into a STAGING copy of
        # the parameter arena; workers adopt whole snapshots from it under a sequence lock (see _snapshot)
        self.consistent = bool(getattr(opt, "consistent", False)) and self.mode == "async" and self.size > 1
        self.off_stage = total
        if self.consistent:
            total += _align(n_pad * self.psz)
        self.arena = SymmetricArena(total, self.device, self.world)
        A = self.arena
        self.signal = A.tensor(self.off_signal, self.m.SIGNAL_SLOTS * 8, torch.int64)
        self.scales = A.tensor(self.off_scales, max(L.nparams, 1) * 4, torch.float32)
        self.wire_arena = A.tensor(self.off_wire, nt * self.bpt, torch.uint8)
        self.param_arena = A.tensor(self.off_param, n_pad * self.psz, self.dtype)
        self.stage_arena = A.tensor(self.off_stage, n_pad * self.psz, self.dtype) if self.consistent else None
        self._sig_base = [p + self.off_signal for p in A.ptrs]

        # ---- move the model's parameters into the parameter arena (zero-copy from now on) ----
        with torch.no_grad():
            self.wire_arena.zero_()          # tile padding must be (and then stays) zero: see grad_out()
            self.param_arena.zero_()
            for s in L.slots:   # a custom placement's padding stays zero
                view = s.view(self.param_arena[s.offset: s.offset + s.numel])
                view.copy_(s.param.data)
                s.param.data = view
        torch.cuda.synchronize(self.device)
        self.world.barrier()
        # identical start on every rank: adopt rank 0's weights (the reference silently relies on
        # equal seeds — there is no initial synchronisation anywhere in ps.py)
        if self.size > 1 and self.rank != 0 and os.environ.get("PSB200_SYNC_INIT", "1") == "1":
            src = A.tensor(self.off_param, n_pad * self.psz, self.dtype, rank=0)
            self.param_arena.copy_(src)
            torch.cuda.synchronize(self.device)
        self.world.barrier()

        if self.consistent:
            self.stage_arena.copy_(self.param_arena)
            torch.cuda.synchronize(self.device)
            self.world.barrier()

        # ---- the pipeline chunks: contiguous runs of whole parameters in arena (= backward) order ----
        self._make_chunks()
        self._make_plan()

        # ---- server-side state: only the tiles this rank serves (compact in mode='sharded') ----
        self.tiles = L.tile_table_fast().to(self.device)
        self.amax = torch.zeros(max(L.nparams, 1), dtype=torch.int32, device=self.device)
        self.active_dev = torch.ones(max(L.nparams, 1), dtype=torch.uint8, device=self.device)
        self.active_host = torch.ones(max(L.nparams, 1), dtype=torch.uint8).pin_memory()
        self._active_all = True
        self._last_fired = None
        self.counters = torch.zeros(8, dtype=torch.int32, device=self.device)   # [0] done, [1] stats
        self.residual = None
        if self.spec.error_feedback:
            self.residual = torch.zeros(n_pad, dtype=torch.float32, device=self.device)
        # the sign wire has no zero code: its kernels take part only over each tile's real elements (the lanes a parameter's arena
        # view covers), so tile padding and a custom placement's interior padding stay exactly 0
        self.real_mask = self._real_mask() if self.kind == KIND_SIGN else None
        # gradient accumulation (MPI_PS.no_sync): micro-batch gradients are summed in fp32 into `carry` (arena-shaped, allocated on
        # first use; an error-feedback coding sums into its residual) by accumulate launches on the compute stream; the step's encode
        # adds the carry to the last gradient (or to `_zeros` for a parameter that fired only inside no_sync) and zeroes it
        self.carry = None
        self._carry_ptr = 0
        self._zeros = None
        self._no_sync = False
        self._mb = MicroBatchCounter()
        self.master = self.buf0 = self.buf1 = self.buf2 = None
        if opt.optim not in _OPTIMS:
            raise ValueError(f"the device engine has no optimizer {opt.optim!r} (one of {sorted(_OPTIMS)})")
        self.optim = _OPTIMS[opt.optim]
        if self.is_server:
            n_state = self.state_tiles * TILE
            if self.dtype != torch.float32 and master_fp32:
                self.master = torch.empty(n_state, dtype=torch.float32, device=self.device)
                self._to_state(self.param_arena, self.master)
            for _key, buf, needed in self.optim.buffers:
                if needed(opt.param_groups):
                    setattr(self, buf, torch.zeros(n_state, dtype=torch.float32, device=self.device))
        # weight average (ema_decay, DESIGN.md rule E1): fp32, compact like the state; psb_ema_kernel runs behind every update
        # launch over the same tiles.  `_ema_n`: averages taken (the first one copies); async counts them on the device.
        self.ema = None
        self._ema_on = getattr(opt, "ema_decay", None) is not None
        self._ema_n = 0
        self._ema_count = None
        self._ema_weight = None
        self._num_sms = 0
        self._in_ema_weights = False
        self._published = None
        if self._ema_on and self.is_server:
            self.ema = torch.zeros(self.state_tiles * TILE, dtype=torch.float32, device=self.device)
            self._ema_weight = 1.0 - float(opt.ema_decay)        # in double; the binding rounds it to fp32 once
            self._num_sms = self.m.num_sms()                       # the EMA / publication grids, queried once
            if self.mode == "async":
                self._ema_count = torch.zeros(2, dtype=torch.int64, device=self.device)
        if self.is_server and not self.sharded:
            self._expose_state()
        self._group_steps = [0] * len(opt.param_groups)
        self._hyper_cache = None
        # per-parameter step counts (the reference keeps optimizer state per parameter and skips p.grad is None,
        # ps.py:178-179,203-205,226-241).  While every parameter has fired on every step they all equal the group's count and
        # the kernel uses the group tuple; after the first step that skipped a parameter a per-parameter table is uploaded.
        self._param_steps = [0] * max(L.nparams, 1)
        self._uniform_steps = True
        # (a ring: the async H2D copy of step e may still be queued when the host fills the table of step e+1)
        self._phyper_host = [torch.zeros(max(L.nparams, 1), 2, dtype=torch.float32).pin_memory() for _ in range(4)]
        self._phyper_dev = [torch.zeros(max(L.nparams, 1), 2, dtype=torch.float32, device=self.device) for _ in range(4)]

        # ---- publication / reduction strategy ----
        mc = A.has_multicast
        if self.mode == "allgather" or self.size == 1:
            self.bcast = BCAST_LOCAL
        else:
            self.bcast = BCAST_MULTICAST if (mc and os.environ.get("PSB200_BCAST", "auto") != "unicast") else BCAST_UNICAST
        nvls_ok = mc and self.kind == KIND_DENSE and self.wire in (WIRE_F32, WIRE_BF16, WIRE_F16) and self.size > 1
        if reduce == "nvls" and not nvls_ok:
            raise ValueError("reduce='nvls' needs multicast memory and a dense fp32/bf16/fp16 wire")
        if reduce == "nvls" and self.mode == "async":
            # multimem.ld_reduce sums EVERY bound rank's wire tile; async sums only the device-selected contributors
            # (quota < N-1), so the switch reduction would re-apply stale / torn gradients of the others
            raise ValueError("reduce='nvls' cannot be combined with mode='async' (the contributor set is a subset)")
        # 'auto': the switch reduces (multimem.ld_reduce: server ingress 1x instead of (N-1)x, 1.9-2x faster than
        # the P2P pull at 16-64 MB on 8 GPUs) for dense fp32 / bf16 / fp16 wires when there is ONE reducer whose
        # contributor set is always every rank (mode='ps') and N >= 4.  bf16/fp16 wires: the switch accumulates in
        # fp32 and returns the sum rounded once to the wire type (|rel err| <= 2^-9 for bf16) before the fp32 master
        # update.  allgather keeps the rank-ordered P2P sum (every rank must produce bit-identical sums), async keeps
        # it because only the selected contributors may be summed.  'nvls' / 'p2p' force either.
        auto_nvls = (nvls_ok and self.mode in ("ps", "sharded") and self.size >= 4
                     and os.environ.get("PSB200_REDUCE", "") != "p2p")
        if reduce == "p2p":
            self.reduce = REDUCE_P2P
        else:
            self.reduce = REDUCE_NVLS if (reduce == "nvls" or (reduce == "auto" and (auto_nvls or (
                nvls_ok and os.environ.get("PSB200_REDUCE", "") == "nvls")))) else REDUCE_P2P

        # ---- the launch plan ----
        self.plan = None
        if self.is_server:
            P = self.m.UpdatePlan()
            P.kind, P.wire, P.opt = self.kind, self.wire, self.optim.code
            P.grid = min(nt, self.m.update_max_grid(self.kind, self.wire, P.opt))
            pub = self.off_stage if self.consistent else self.off_param      # where fresh parameters are published
            for r in range(self.size):
                base = A.ptrs[r]
                P.set_rank_ptrs(r, base + self.off_wire, base + self.off_scales, base + pub,
                                base + self.off_signal)
            P.configure(self.size, self.rank, nt, self.bpt, self.cap, self.dt, self.bcast, self.reduce,
                        (A.mc_ptr + pub) if mc else 0, (A.mc_ptr + self.off_wire) if mc else 0,
                        A.local_ptr + pub,
                        self.master.data_ptr() if self.master is not None else 0,
                        self.buf0.data_ptr() if self.buf0 is not None else 0,
                        self.buf1.data_ptr() if self.buf1 is not None else 0,
                        self.buf2.data_ptr() if self.buf2 is not None else 0,
                        self.tiles.data_ptr(), A.local_ptr + self.off_signal,
                        self.counters.data_ptr(), self.counters.data_ptr() + 4)
            if self.kind == KIND_SIGN:
                P.set_real_mask(self.real_mask.data_ptr())
            self.plan = P
        self.comm_stream = torch.cuda.Stream(device=self.device)
        self._cs = self.comm_stream.cuda_stream            # raw handle for explicit-stream launches
        self._ev_pool = [torch.cuda.Event() for _ in range(64)]
        self._ev_i = 0
        self._ema_src = (self.master.data_ptr() if self.master is not None else 0,
                         0 if self.master is not None else A.local_ptr + (self.off_stage if self.consistent else self.off_param))
        self._tiles_ptr = self.tiles.data_ptr()
        self._wire_ptr = self.arena.local_ptr + self.off_wire
        self._scales_ptr = self.arena.local_ptr + self.off_scales
        self._amax_ptr = self.amax.data_ptr()
        self._residual_ptr = self.residual.data_ptr() if self.residual is not None else 0
        self._sigctr_ptr = self.counters.data_ptr() + 8
        self._ratio = float(self.spec.ratio)
        # block-wise QSGD: the Philox counter holds (element, arena tile, step, rank).  `_qsgd_step` counts the steps this rank
        # has encoded; it is saved with the optimizer state ("qsgd_step") on every rank, so a resumed run draws what a straight
        # run draws.
        self._qsgd_step = 0
        self._start_step()
        self._keep_prev: List[torch.Tensor] = []   # last step's gradients: freed one step late (see _flush)
        self._prev_done = None                      # comm-stream completion of the last step
        self.launches = 0                     # kernels of OURS launched (bench 'gpu_launches')
        self._closed = False
        self._gates: list = []
        self._gate_epoch = -1                 # the last epoch whose PARAMS_READY a forward has acquired (gate / ensure_params)
        self._prof = CudaStepTimer(bool(getattr(opt, "profile", False)))
        self._epoch = 0                       # completed engine steps (the epoch-flag clock)
        # async bookkeeping
        self.version = 0
        self._consumed = torch.zeros(64, dtype=torch.int64, device=self.device)
        self._select_out = torch.zeros(64, dtype=torch.int64, device=self.device)
        self._select_host = torch.zeros(64, dtype=torch.int64).pin_memory()
        self._async_done_workers: set = set()
        self._async_depth = max(1, int(os.environ.get("PSB200_ASYNC_DEPTH", "4")))
        self._async_ring = [{"host": torch.zeros(64, dtype=torch.int64).pin_memory(), "event": torch.cuda.Event(), "version": 0}
                            for _ in range(self._async_depth + 1)]
        self._async_pending: list = []
        self._async_i = 0
        self._async_applied = 0
        self._async_last = {"contributors": [], "param_version": 0, "staleness": {}, "updates_applied": 0}
        # K10 "no separate serialization pass": producers we own (our BN / stem / linear backward kernels) write their
        # gradient straight into this rank's wire arena when the wire layout IS the gradient layout
        self._direct_ok = (self.kind == KIND_DENSE and self.wire == wire_code_of(self.dtype) and self.mode in ("ps", "sharded")
                           and os.environ.get("PSB200_DIRECT_GRAD", "1") != "0")
        self.direct_grads = 0
        self.direct_names: set = set()
        if self._direct_ok:
            import functools
            for sl in self.layout.slots:
                sl.param.ps_grad_out = functools.partial(self.grad_out, sl.param)
        self._snap_version = 0
        self._snap_shadow = None
        self._phyper_ptr = 0
        self._update_spans: list = []
        # device-timeout surfacing: an async copy of SIG_ERROR into pinned memory every few steps, read one poll late
        self._err_host = torch.zeros(1, dtype=torch.int64).pin_memory()
        self._err_event = None
        self._err_every = max(1, int(os.environ.get("PSB200_ERROR_POLL", "16")))
        self.world.barrier()

    def _check_same_layout_everywhere(self):
        """Every rank must describe the SAME flat arena (the kernels address peers' arenas by tile number): compare a fingerprint
        of mode / optimizer / dtype / wire format / parameter names and shapes across ranks and fail on all of them with the first
        difference.  The reference silently assumes identical models on every rank; a mismatch there hangs or corrupts."""
        if self.size == 1 or os.environ.get("PSB200_CHECK_LAYOUT", "1") == "0":
            return
        L = self.layout
        mine = (self.mode, self.opt.optim, str(self.dtype), int(self.kind), int(self.wire), int(self.bpt), L.nparams, L.ntiles,
                tuple((s.name, tuple(s.param.shape)) for s in L.slots))
        every = self.world.all_gather_object(mine)
        for r, other in enumerate(every):
            if other != every[0]:
                what = ["mode", "optimizer", "parameter dtype", "coding kind", "wire dtype", "bytes per tile", "number of parameters",
                        "number of tiles", "parameter names / shapes"]
                k = next(i for i in range(len(mine)) if other[i] != every[0][i])
                detail = ""
                if k == 8:
                    diff = [(a, b) for a, b in zip(every[0][8], other[8]) if a != b][:1]
                    detail = f": first difference {diff[0] if diff else (len(every[0][8]), len(other[8]))}"
                raise ValueError(f"rank {r} and rank 0 disagree on the {what[k]} ({other[k] if k < 8 else '...'} vs "
                                 f"{every[0][k] if k < 8 else '...'}){detail} — every rank must build the same model, coding and mode")

    def _real_mask(self) -> torch.Tensor:
        """``ntiles x 64`` 32-bit words, bit ``e & 31`` of word ``tile * 64 + (e >> 5)`` set iff element ``e`` of the tile lies in
        its parameter's arena view (:meth:`ParamSlot.view`).  It depends on the layout only, so every rank builds the same one."""
        import numpy as np
        L = self.layout
        real = torch.zeros(L.numel_padded, dtype=torch.bool)
        for s in L.slots:
            s.view(real[s.offset: s.offset + s.numel]).fill_(True)
        words = np.packbits(real.numpy(), bitorder="little").view(np.int32)
        return torch.empty(len(words), dtype=torch.int32, device=self.device).copy_(torch.from_numpy(words))

    def _make_chunks(self):
        """Static chunks of the update pipeline (identical on every rank: they depend on the layout only).

        Chunk ``k`` = arena tiles ``[lo, hi)`` holding whole parameters, at least ``chunk_bytes`` of parameter bytes
        each (the last one takes the remainder).  A chunk is encoded — and, by the ranks that serve it (``_make_plan``),
        gathered / updated / published — as soon as every parameter in it AND in all earlier chunks has produced its
        gradient, while backward keeps running on the later chunks (``/root/reference/ps.py:140-148,159-162``: one collective per
        parameter, consumed as each completes)."""
        L = self.layout
        chunks = L.plan_chunks(self.psz, self.chunk_bytes, single=(not self.pipeline and self.mode != "async"))
        self.chunks = chunks
        self.nchunks = len(chunks)
        self.chunk_tiles = [(c[0].first_tile, c[-1].first_tile + c[-1].ntiles) for c in chunks]
        self._chunk_of = [0] * L.nparams
        for k, c in enumerate(chunks):
            for sl in c:
                self._chunk_of[sl.index] = k

    def _make_plan(self):
        """The serve plan: which rank gathers, updates and publishes which tiles of every span, and how it announces that it is
        done.  Static and identical on every rank: it depends on the layout, the mode and N only.

        The spans are the pipeline chunks (one span over the whole arena when not pipelined; ``async`` never is).
        ``shards[k][r]`` is rank ``r``'s tile range ``(begin, end)`` of span ``k``, or ``None`` when ``r`` does not serve:

        * ``ps`` and ``async`` (and every mode at N = 1): rank 0 serves the whole span;
        * ``allgather``: every rank serves the whole span, publishing into its own parameter arena;
        * ``sharded``: the span ``[lo, hi)`` is split into N contiguous ranges in rank order, ``(hi - lo) // N`` tiles each; the
          remainder goes one tile each to the ``(hi - lo) % N`` ranks starting at ``k % N``, so small chunks do not all land on
          rank 0.  A range may be empty.

        A serving rank keeps optimizer state for its own ranges only, concatenated in span order (``state_tiles`` tiles; every
        tile outside ``sharded``): the update of span ``k`` addresses it with ``state_shift = begin - compact_base``
        (``_mine[k]``).  Tile granularity is exact for every coding: they all decode per tile and read per-parameter scales and
        hyper-parameters by index."""
        n, me = self.size, self.rank
        spans = self.chunk_tiles if self.pipeline else [(0, self.layout.ntiles)]
        self.shards = []                      # per span: (begin, end) or None, per rank
        for k, (lo, hi) in enumerate(spans):
            if self.sharded:
                q, rem = divmod(hi - lo, n)
                ranges, b = [], lo
                for r in range(n):
                    e = b + q + (1 if (r - k) % n < rem else 0)
                    ranges.append((b, e))
                    b = e
            elif self.mode == "allgather":
                ranges = [(lo, hi)] * n
            else:
                ranges = [(lo, hi)] + [None] * (n - 1)
            self.shards.append(ranges)
        self._mine = []                       # per span: (begin, end, state_shift) of this rank, or None
        base = 0
        for ranges in self.shards:
            if ranges[me] is None:
                self._mine.append(None)
                continue
            b, e = ranges[me]
            self._mine.append((b, e, b - base))
            base += e - b
        self.state_tiles = base
        servers = [r for r in range(n) if self.shards[0][r] is not None]
        self.is_server = me in servers
        # GRAD_READY progress goes to the other serving ranks: a rank's own gradient is ordered by its stream.  (Async workers
        # post their gradient to the server from _step_async.)
        self._grad_targets = [self._sig_base[r] for r in servers if r != me] if self.mode != "async" else []
        # The signal of a step's last launch, and what it adds to PARAMS_READY per step on a rank that another rank publishes
        # into: that rank waits for PARAMS_READY >= epoch * _ready_per_step before its next forward (0: it waits for its own
        # comm stream instead).
        if n == 1:
            self._done_signal, self._ready_per_step = SIGNAL_NONE, 0
        elif self.mode == "ps":                       # rank 0 stores the epoch into every rank
            self._done_signal, self._ready_per_step = SIGNAL_PARAMS_READY, 0 if self.is_server else 1
        elif self.mode == "allgather":                # every rank publishes into its own arena
            self._done_signal, self._ready_per_step = SIGNAL_CONSUMED, 0
        elif self.mode == "sharded":                  # every server adds 1 into every rank
            self._done_signal, self._ready_per_step = self.m.SIGNAL_PARAMS_READY_ADD, n
        else:                                         # async: the server signals from _step_async, workers never wait
            self._done_signal, self._ready_per_step = SIGNAL_PARAMS_READY, 0

    def _state_pieces(self, first_tile: int, ntiles: int):
        """``(arena_tile_lo, arena_tile_hi, state_tile_lo)`` for the parts of arena tiles ``[first_tile, first_tile + ntiles)``
        whose optimizer state this (serving) rank keeps.  Pieces next to each other in the arena and in the state are merged,
        so a rank that keeps every tile's state gets one piece (one copy in ``_to_state``)."""
        out = []
        for b, e, shift in self._mine:
            lo, hi = max(b, first_tile), min(e, first_tile + ntiles)
            if lo >= hi:
                continue
            if out and out[-1][1] == lo and out[-1][0] - out[-1][2] == shift:
                out[-1] = (out[-1][0], hi, out[-1][2])
            else:
                out.append((lo, hi, lo - shift))
        return out

    def _to_state(self, full: torch.Tensor, state: torch.Tensor):
        """Copy the arena-indexed ``full`` into ``state`` (compact in mode='sharded')."""
        for lo, hi, c in self._state_pieces(0, self.layout.ntiles):
            state[c * TILE: (c + hi - lo) * TILE].copy_(full[lo * TILE: hi * TILE])

    def _start_step(self):
        """The bookkeeping of a step no gradient has arrived for yet.  Callers decide what happens to the gradients kept
        alive for the previous step (``_keep_prev``) and to its completion event (``_prev_done``)."""
        self._fired: set = set()
        self._keep: List[torch.Tensor] = []
        self._raw_bytes = 0
        self._first_flush_done = False
        self._published = None
        self._step_hyp = None
        self._chunk_items: List[list] = [[] for _ in self.chunks]
        self._chunk_left = [len(c) for c in self.chunks]
        self._next_chunk = 0
        self._carried: set = set()           # parameters with a contribution in the carry this step
        self._acc_items: List[list] = [[] for _ in self.chunks]   # accumulates not yet launched, per chunk
        self._acc_left = [len(c) for c in self.chunks]           # per chunk: parameters yet to fire in this micro-batch
        self._acc_waited = False
        self._mb.reset()

    def _progress(self, epoch: int, chunk: int) -> int:
        """Monotone GRAD_READY value meaning "chunks 0..chunk of step ``epoch`` are in my wire arena"."""
        return (epoch - 1) * self.nchunks + chunk + 1

    # ---------------------------------------------------------------------------------- state
    def _expose_state(self):
        """Make ``opt.state[p]`` views of the flat fp32 state (checkpoint parity, SURVEY §5)."""
        o = self.opt
        bufs = self._state_buffers()
        for s in self.layout.slots:
            st = o.state[s.param]
            sl = slice(s.offset, s.offset + s.numel)
            if self.optim.step_key:
                st.setdefault("step", 0)
            for key, buf in bufs:
                st[key] = s.view(buf[sl])

    def sync_state_to_torch(self):
        o = self.opt
        if self.kind == KIND_QSGD:
            for s in self.layout.slots:
                o.state[s.param]["qsgd_step"] = self._qsgd_step
        if not self.is_server:
            return
        if self.ema is not None:
            # the last average of a step may still run on the comm stream (a rank that waits only for its own comm stream waits
            # for the update, not for the average): the views handed out below are read on the current stream
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
        for s in self.layout.slots:   # SGD too: the first-step momentum rule (ps.py:203-205) needs it on resume
            o.state[s.param]["step"] = self._param_steps[s.index] if self.mode != "async" else self._group_steps[s.group]
        if self.sharded:
            self._gather_state()
        elif self.ema is not None:    # the average is state once it has been taken
            taken = self._ema_taken()
            for s in self.layout.slots:
                if taken:
                    o.state[s.param]["ema"] = s.view(self.ema[s.offset: s.offset + s.numel])
                else:
                    o.state[s.param].pop("ema", None)

    def _ema_taken(self) -> bool:
        """Has the weight average been taken at least once?  (Async counts on the device: this synchronises.)"""
        if self._ema_count is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
            return int(self._ema_count[0].item()) > 0
        return self._ema_n > 0

    def _state_buffers(self, ema: bool = False):
        """``(state key, flat fp32 buffer)`` of every optimizer-state buffer this engine keeps (``ema``: and the average)."""
        out = [(key, getattr(self, buf)) for key, buf, _ in self.optim.buffers] + [("master_param", self.master)]
        if ema:
            out.append(("ema", self.ema))
        return [(k, b) for k, b in out if b is not None]

    def _gather_state(self):
        """mode='sharded' ``state_dict()`` (collective): every rank's compact shards → the full per-parameter state on every
        rank, the values rank 0 holds in mode='ps', as CPU copies.  ``MPI_PS.state_dict`` drops them from ``opt.state`` once
        its dict is built (:meth:`drop_state_copies`), so only the returned dict keeps them."""
        torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
        torch.cuda.synchronize(self.device)
        bufs = self._state_buffers(ema=self.ema is not None and self._ema_taken())
        every = self.world.all_gather_object({k: b.cpu() for k, b in bufs})
        full = {k: torch.zeros(self.layout.numel_padded, dtype=torch.float32) for k, _ in bufs}
        for r, theirs in enumerate(every):
            base = 0
            for ranges in self.shards:
                b, e = ranges[r]
                for k in full:
                    full[k][b * TILE: e * TILE] = theirs[k][base * TILE: (base + e - b) * TILE]
                base += e - b
        o = self.opt
        for s in self.layout.slots:
            for k, flat in full.items():
                o.state[s.param][k] = s.view(flat[s.offset: s.offset + s.numel])

    def drop_state_copies(self):
        """mode='sharded': leave only the step counts in ``opt.state`` — the engine's compact buffers are the live state, and
        full-size copies (gathered for ``state_dict()``, or put there by ``load_state_dict()``) would undo the 1/N."""
        o = self.opt
        for s in self.layout.slots:
            if s.param in o.state:      # a new dict: one that state_dict() already returned keeps its tensors
                o.state[s.param] = {k: v for k, v in o.state[s.param].items()
                                    if k in ("step", "qsgd_step") or not torch.is_tensor(v)}

    def _load_slot(self, s, buf: torch.Tensor, value: torch.Tensor):
        """Write parameter-shaped ``value`` into the state buffer ``buf`` at slot ``s`` (only the tiles this rank keeps)."""
        tmp = torch.zeros(s.ntiles * TILE, dtype=buf.dtype, device=buf.device)
        s.view(tmp[: s.numel]).copy_(value.to(buf.dtype))
        for lo, hi, c in self._state_pieces(s.first_tile, s.ntiles):
            buf[c * TILE: (c + hi - lo) * TILE].copy_(tmp[(lo - s.first_tile) * TILE: (hi - s.first_tile) * TILE])

    def sync_state_from_torch(self, original=None):
        """After ``load_state_dict``: copy loaded tensors back into the flat (fp32) state.

        ``original`` maps ``id(param)`` → the un-cast saved state of that parameter."""
        o = self.opt
        if self.kind == KIND_QSGD:
            for s in self.layout.slots:
                st = original.get(id(s.param), {}) if original is not None else o.state.get(s.param, {})
                if "qsgd_step" in st:
                    self._qsgd_step = int(st["qsgd_step"])
        if self._ema_on:
            # the average resumes when every parameter has one; a checkpoint without it restarts it (the next step copies)
            saved = [(s, original.get(id(s.param), {}) if original is not None else o.state.get(s.param, {}))
                     for s in self.layout.slots]
            have = [torch.is_tensor(st.get("ema")) for _, st in saved]
            if any(have) and not all(have):
                raise ValueError("the checkpoint has a weight average ('ema') for some parameters only")
            self._ema_n = int(all(have))
            if self.ema is not None:
                # the loaded average must land after any average still queued on the comm stream, and before the next one
                cur = torch.cuda.current_stream(self.device)
                cur.wait_stream(self.comm_stream)
                with torch.no_grad():
                    for s, st in saved:
                        if self._ema_n:
                            self._load_slot(s, self.ema, st["ema"])
                    if self._ema_count is not None:
                        self._ema_count.fill_(0)
                        self._ema_count[0] = self._ema_n
                self.comm_stream.wait_stream(cur)
        if not self.is_server:
            return
        with torch.no_grad():
            for s in self.layout.slots:
                st = o.state.get(s.param, {})
                if original is not None and id(s.param) in original:
                    st = original[id(s.param)]
                sl = slice(s.offset, s.offset + s.numel)
                for key, buf in self._state_buffers():
                    if key in st and st[key] is not None:
                        if self.sharded or st[key].data_ptr() != buf[sl].data_ptr():
                            self._load_slot(s, buf, st[key])
                if "step" in st:
                    self._group_steps[s.group] = max(self._group_steps[s.group], int(st["step"]))
                    self._param_steps[s.index] = int(st["step"])
            if self.master is not None:
                # parameters may have been re-loaded by the user: re-seed masters that lack a saved copy
                for s in self.layout.slots:
                    src = original.get(id(s.param), {}) if original is not None else o.state.get(s.param, {})
                    if "master_param" not in src:
                        self._load_slot(s, self.master, s.param.data)
        if any(self._param_steps[s.index] != self._group_steps[s.group] for s in self.layout.slots):
            self._uniform_steps = False
        if self.sharded:
            self.drop_state_copies()
        else:
            self._expose_state()
            for s in self.layout.slots:      # torch's cast copy of the average (state_dict() exposes the live one)
                o.state[s.param].pop("ema", None)

    # ------------------------------------------------------------------------------- backward
    def grad_out(self, param: torch.nn.Parameter) -> Optional[torch.Tensor]:
        """Where the producer of ``param``'s gradient may write it DIRECTLY: a view of this rank's wire arena with the
        parameter's shape and physical layout — or ``None`` (coded wires, other modes).

        With Identity / same-dtype wires the wire tile of a parameter is bit-for-bit its gradient, so a kernel we own
        (fused BN backward, the stem's implicit weight gradient, ``BcastLinear``'s dW GEMM with ``out=``) can skip the
        ``psb_encode_kernel`` copy: ``on_grad`` recognises the pointer and only counts the parameter as arrived.  Safe in
        ``mode='ps'`` and ``mode='sharded'`` only: a rank's backward starts after it observed PARAMS_READY (every server
        finished reading the previous wire tiles); in ``allgather`` mode peers may still be reading them (CONSUMED is awaited
        on the comm stream)."""
        if not self._direct_ok or self._closed or self.accumulating:
            return None                      # (an accumulated step encodes from the carry)
        sl = self.layout.by_id.get(id(param))
        if sl is None:
            return None
        flat = self.wire_arena[sl.first_tile * self.bpt: sl.first_tile * self.bpt + sl.numel * self.psz].view(self.dtype)
        return sl.view(flat)

    def on_grad(self, grad: torch.Tensor, name: str, param: torch.nn.Parameter):
        """Backward hook (``ps.py:98-101``): file the gradient under its chunk; every chunk that is now complete (in
        arena order) is encoded — and on the server gathered / updated / broadcast — right away, under backward."""
        if self._in_ema_weights:
            raise RuntimeError(f"parameter {name!r} got a gradient inside opt.ema_weights(): the parameters hold the average "
                               "there; run backward() outside the block")
        s = self.layout.by_id[id(param)]
        g = grad.detach()
        # a gradient the producer already wrote into the wire arena (grad_out) has nothing to encode
        direct = self._direct_ok and g.data_ptr() == self._wire_ptr + s.first_tile * self.bpt and g.dtype == self.dtype \
            and g.stride() == param.stride()
        if not direct:
            if g.dtype != self.dtype:
                g = g.to(self.dtype)
            if s.strides is not None:
                # custom placement: the encode kernel reads the whole span, padding included (it must be zero)
                if not (g.stride() == param.stride() and g.data_ptr() % 16 == 0 and g.storage_offset() * g.element_size() +
                        s.numel * g.element_size() <= g.untyped_storage().nbytes()):
                    span = torch.zeros(s.numel, dtype=g.dtype, device=g.device)
                    s.view(span).copy_(g)
                    g = span
                else:
                    g = torch.as_strided(g, (s.numel,), (1,))
            elif g.stride() != param.stride() or g.data_ptr() % 16:
                # the arena is in the parameter's physical order: bring the gradient into it
                g = torch.empty_strided(param.shape, param.stride(), dtype=g.dtype, device=g.device).copy_(g)
        if self._mb.fire(s.index):           # a new backward pass: the previous one's gradients are summed first
            self._flush_accumulate()
            self._acc_left = [len(c) for c in self.chunks]
        if s.index in self._fired:
            raise RuntimeError(f"parameter {name!r} produced two gradients before step(); call step() after every backward, "
                               "or run the earlier backwards inside opt.no_sync() to accumulate them")
        if self._no_sync:
            self._accumulate(s, g, param)
            return
        if self._carried:
            self._drop_wire_alias(param)
        self._fired.add(s.index)
        k = self._chunk_of[s.index]
        self._chunk_left[k] -= 1
        self._raw_bytes += s.numel * self.psz
        if direct:
            self.direct_grads += 1
            self.direct_names.add(name)
            if param.grad is not None:
                # AccumulateGrad would add the incoming gradient INTO param.grad in place — and both may alias the same wire
                # tile (zero_grad(set_to_none=False)): drop the old one so the new gradient is assigned, not accumulated
                param.grad = None
        else:
            self._chunk_items[k].append((s, g))
        while self._next_chunk < self.nchunks and self._chunk_left[self._next_chunk] == 0:
            self._flush_chunk(self._next_chunk)

    # ------------------------------------------------------------------------- accumulation
    @property
    def accumulating(self) -> bool:
        """Inside ``no_sync()``, or the carry holds gradients the next ``step()`` has not sent yet."""
        return self._no_sync or bool(self._carried)

    def begin_no_sync(self):
        if self.mode == "async" and self.size > 1 and self.rank == 0:
            return                           # the dedicated server runs no backward
        if self.carry is None:
            L = self.layout
            self.carry = self.residual if self.residual is not None else \
                torch.zeros(L.numel_padded, dtype=torch.float32, device=self.device)
            self._carry_ptr = self.carry.data_ptr()
            self._zeros = torch.zeros(max(s.numel for s in L.slots), dtype=self.dtype, device=self.device)
        self._no_sync = True
        self._mb.cut()

    def end_no_sync(self):
        self._flush_accumulate()
        self._no_sync = False
        self._mb.cut()

    def _drop_wire_alias(self, param):
        """After a direct-placement step ``param.grad`` can still view the wire arena (``zero_grad(set_to_none=False)``):
        AccumulateGrad would add this gradient into a wire tile the server may be reading.  Drop it: the gradient is assigned."""
        g = param.grad
        if g is not None and self._direct_ok and 0 <= g.data_ptr() - self._wire_ptr < self.wire_arena.numel():
            param.grad = None

    def _accumulate(self, s, g, param):
        """A gradient inside ``no_sync()``: queue it for the carry; each chunk is summed once all its parameters fired."""
        self._drop_wire_alias(param)
        self._carried.add(s.index)
        k = self._chunk_of[s.index]
        self._acc_items[k].append((s, g))
        self._acc_left[k] -= 1
        if self._acc_left[k] == 0:
            self._flush_accumulate(k)

    def _flush_accumulate(self, k: Optional[int] = None):
        """carry += the queued gradients (of chunk ``k``, or all), on the compute stream: the gradients need not outlive it."""
        items = []
        for j in (range(self.nchunks) if k is None else (k,)):
            items += self._acc_items[j]
            self._acc_items[j] = []
        if not items:
            return
        if not self._acc_waited:
            self._acc_waited = True
            if self._prev_done is not None:  # the last step's encode zeroed (or wrote the leftover into) the carry on the comm stream
                torch.cuda.current_stream(self.device).wait_event(self._prev_done)
        self.m.accumulate([g for _, g in items], [s.first_tile for s, _ in items], [s.ntiles for s, _ in items],
                          [s.index for s, _ in items], self._tiles_ptr, self._carry_ptr)
        self.launches += (len(items) + 63) // 64

    def _close_accumulation(self):
        """step(): sum what is still queued; parameters that fired only inside no_sync() are encoded from the carry alone."""
        self._flush_accumulate()
        for i in sorted(self._carried - self._fired):
            s = self.layout.slots[i]
            k = self._chunk_of[i]
            self._fired.add(i)
            self._chunk_left[k] -= 1
            self._raw_bytes += s.numel * self.psz
            self._chunk_items[k].append((s, self._zeros[: s.numel]))

    def _event(self, timing: bool = False):
        """A pooled CUDA event (creating one costs more than recording one)."""
        if timing:
            return torch.cuda.Event(enable_timing=True)
        self._ev_i = (self._ev_i + 1) % len(self._ev_pool)
        return self._ev_pool[self._ev_i]

    def _flush_chunk(self, k: int, joined: bool = False, active_ptr: int = 0):
        """Everything chunk ``k`` needs, queued on the comm stream (explicit stream handle: no Python-side stream
        switching): encode its gradients into the wire arena, raise this rank's GRAD_READY progress flag from the
        last encode CTA, and — on a rank that serves the span — launch the fused gather/update/publish kernel for its tiles.

        Must be called in chunk order.  ``joined``: the caller already made the comm stream wait for the compute stream."""
        assert k == self._next_chunk
        self._next_chunk = k + 1
        m, cs, csh = self.m, self.comm_stream, self._cs
        cur = torch.cuda.current_stream(self.device)
        if not joined:
            ev = self._event()
            ev.record(cur)
            cs.wait_event(ev)
        if not self._first_flush_done:
            if self._prev_done is not None:
                # Bound the comm stream's lag to one step: gradients are kept alive (not record_stream'ed, which
                # would make the caching allocator grow and cudaMalloc for several steps) until the step after
                # they were encoded, so the compute stream must not run further ahead than that.
                cur.wait_event(self._prev_done)
            self._first_flush_done = True
            self._before_first_encode()
        epoch = self._epoch + 1
        last = k == self.nchunks - 1
        ends_span = self.pipeline or last             # unpipelined: one span over the whole arena, after the last chunk
        sig = None
        if self._grad_targets and ends_span:
            sig = (self._grad_targets, m.SIG_GRAD_READY + self.rank, self._progress(epoch, k))
        items, self._chunk_items[k] = self._chunk_items[k], []
        if items:
            grads = [g for _, g in items]
            kw = dict(seed=self.spec.seed, step=self._qsgd_step & 0xFFFFFFFF, rank=self.rank,
                      levels=self.spec.levels) if self.kind == KIND_QSGD else {}
            if self.kind == KIND_SIGN:
                kw["real_mask"] = self.real_mask.data_ptr()
            if self._carried:                 # an accumulated step: the encode adds the carry and zeroes it
                kw["keep_leftover"] = self.residual is not None
            m.encode(self.kind, self.wire, grads, [s.first_tile for s, _ in items],
                     [s.ntiles for s, _ in items], [s.index for s, _ in items],
                     self._tiles_ptr, self._wire_ptr, self._scales_ptr, self._amax_ptr,
                     self._carry_ptr if self._carried else self._residual_ptr,
                     self.bpt, self.cap, self._ratio,
                     *((sig[0], sig[1], sig[2], self._sigctr_ptr) if sig else ([], 0, 0, 0)),
                     csh, **kw)
            nb = (len(items) + 63) // 64
            self.launches += nb * (2 if self.kind == KIND_SCALED else 1)
            self._keep.extend(grads)
        elif sig:                                     # nothing fired in this chunk: the flag alone
            m.signal(sig[0], sig[1], sig[2], -1, 0, csh)
            self.launches += 1
        # ---- this rank's share of the span (the serve plan), for every synchronous mode; the async server launches from
        # _step_async.  An empty share (mode='sharded') launches nothing, except the completion signal on the last chunk.
        mine = self._mine[k if self.pipeline else 0] if ends_span and self.mode != "async" else None
        if mine is None or (mine[0] == mine[1] and not last):
            return
        lo, hi, shift = mine
        n, want = self.size, self._progress(epoch, k)
        wait_mask = ((1 << n) - 1) & ~(1 << self.rank)
        prof = self._prof.enabled and hi > lo
        ev_a = self._prof.mark(cs) if prof else None
        if n > 1:
            # The req.Wait() for this chunk is a ONE-WARP kernel, not the update grid: 444 update CTAs spinning on the
            # peers' flags would hold every SM's register file (3 x 256 threads x 77 registers) while this rank's own
            # backward still has chunks k+1.. to produce — the skew between ranks would land on the critical path.
            m.wait_flags(self.arena.local_ptr + self.off_signal, m.SIG_GRAD_READY, wait_mask, want, self.timeout_s, csh)
            self.launches += 1
        if hi == lo:                                  # only mode='sharded' has empty shares: its counted PARAMS_READY alone
            m.signal(self._sig_base, m.SIG_PARAMS_READY, 1, stream=csh, add=True)
            self.launches += 1
            return
        # (epoch, groups, contrib_mask, inv_count, wait_grads, signal_mode, ...); state_shift keeps its default, 0, unless
        # this share's state is stored shifted
        self.plan.launch(epoch, self._get_hypers(), (1 << n) - 1, (1.0 / n) if self.opt.average else 1.0, 0,
                         self._done_signal if last else SIGNAL_NONE,
                         active_ptr=active_ptr, timeout_s=self.timeout_s, wait_mask=wait_mask, stream=csh,
                         tile_begin=lo, tile_end=hi, wait_value=want, param_hyper=self._phyper_ptr,
                         **({"state_shift": shift} if shift else {}))
        self.launches += 1
        if self.ema is not None:
            # the average of the tiles just updated, behind the update: it never delays the PARAMS_READY of the last chunk.  When
            # it reads the fp32 master (memory only the comm stream touches), a rank that waits only for its own comm stream waits
            # for `_published`, not for this launch; reading the parameters, it is waited for, since the user may write them
            if last and self.master is not None:
                self._published = self._event()
                self._published.record(cs)
            m.ema(*self._ema_src, self.dt, self.ema.data_ptr(), self.layout.ntiles, lo, hi, shift, self._ema_weight,
                  self._ema_n == 0, stream=csh, num_sms=self._num_sms)
            self.launches += 1
        if prof:
            self._update_spans.append((ev_a, self._prof.mark(cs)))

    def _before_first_encode(self):
        """Queued on the comm stream before this step's first write into the wire arena."""
        epoch = self._epoch + 1              # the step these gradients belong to
        if self.kind == KIND_SCALED:
            with torch.cuda.stream(self.comm_stream):
                self.amax.zero_()
        if self.size == 1:
            return
        sig = self.arena.local_ptr + self.off_signal
        if self.mode == "allgather" and epoch > 1:
            # every peer must have finished READING our previous wire tiles
            self.m.wait_flags(sig, self.m.SIG_CONSUMED, ((1 << self.size) - 1) & ~(1 << self.rank), epoch - 1,
                              self.timeout_s, self._cs)
            self.launches += 1
        elif self.mode == "async" and self.rank != 0 and epoch > 1:
            self.m.wait_flags(sig, self.m.SIG_ACK, 1, epoch - 1, self.timeout_s, self._cs)
            self.launches += 1

    # ----------------------------------------------------------------------------------- step
    def _get_hypers(self):
        """This step's per-group hyper-parameter tuples (sampled once per step, at the first chunk that needs them)."""
        if self._step_hyp is None:
            self._step_hyp = self._hypers()
            self._phyper_ptr = 0
            if not self._uniform_steps and self.is_server:
                self._phyper_ptr = self._upload_param_hypers()
        return self._step_hyp

    def _upload_param_hypers(self) -> int:
        """Per-parameter {step_size, first_step} (AdamW: {s, c2}) for THIS step, assuming the parameter fires (tiles of parameters that do not
        are skipped through the active mask, so their entries are never read)."""
        o = self.opt
        slot = self._epoch % len(self._phyper_host)       # the comm stream lags the host by at most one step
        h, dev = self._phyper_host[slot], self._phyper_dev[slot]
        for sl in self.layout.slots:
            h[sl.index, 0], h[sl.index, 1] = self.optim.per_param(o.param_groups[sl.group], self._param_steps[sl.index] + 1)
        with torch.cuda.stream(self.comm_stream):
            dev.copy_(h, non_blocking=True)
        return dev.data_ptr()

    def _hypers(self) -> List[List[float]]:
        o = self.opt
        out = []
        for gi in range(len(o.param_groups)):
            self._group_steps[gi] += 1
        first = any(t == 1 for t in self._group_steps)
        cache_key = self.optim.cache_key
        if cache_key is not None:
            # a tuple that only changes with lr schedules / the first step (SGD's): reuse the cached list otherwise
            key = tuple(cache_key(g) for g in o.param_groups)
            if not first and self._hyper_cache is not None and self._hyper_cache[0] == key:
                return self._hyper_cache[1]
        for gi, g in enumerate(o.param_groups):
            out.append(self.optim.group(g, self._group_steps[gi]))
        if cache_key is not None and not first:
            self._hyper_cache = (key, out)
        return out

    def _handle_inactive(self):
        """Parameters whose hook did not fire this step (``p.grad is None``, ``ps.py:178-179``)."""
        L = self.layout
        if len(self._fired) == L.nparams:
            if not self._active_all:
                self.active_host.fill_(1)
                self.active_dev.copy_(self.active_host, non_blocking=True)
                self._active_all = True
                self._last_fired = None
            return 0
        fired = frozenset(self._fired)
        if fired == self._last_fired:        # same frozen / unused set as last step: mask and zeroed tiles still valid
            return self.active_dev.data_ptr()
        self._last_fired = fired
        self.active_host.zero_()
        for i in self._fired:
            self.active_host[i] = 1
        self.active_dev.copy_(self.active_host, non_blocking=True)
        self._active_all = False
        # a tile the server will read must not carry last step's payload
        for s in L.slots:
            if s.index not in self._fired:
                self.wire_arena[s.first_tile * self.bpt: (s.first_tile + s.ntiles) * self.bpt].zero_()
        return self.active_dev.data_ptr()

    def _flush_rest(self, cs, joined: bool):
        """step(): chunks that did not complete during backward (always the last one's tail when every parameter
        fired from the final hook; all of them when some parameter got no gradient, ``ps.py:178-179``)."""
        if self._next_chunk >= self.nchunks:
            if not self._active_all:                  # every parameter fired again: forget the frozen-set cache
                self._active_all, self._last_fired = True, None
            return
        if len(self._fired) == self.layout.nparams and self._active_all:
            active_ptr = 0                            # the common case: every parameter got a gradient
        else:
            with torch.cuda.stream(cs):
                active_ptr = self._handle_inactive()  # before the flag: a tile the server reads must be final
        while self._next_chunk < self.nchunks:
            self._flush_chunk(self._next_chunk, joined=joined, active_ptr=active_ptr)

    def step(self) -> Dict[str, float]:
        t0 = time.time()
        data = {"comm_wait": 0.0, "optim_step_time": 0.0, "decode_time": 0.0,
                "iallgather_prepare_time": 0.0, "isend_time": 0.0}
        if self.mode == "async" and self.size > 1:
            return self._step_async(data)
        self._close_accumulation()
        epoch = self._epoch + 1
        m, cs = self.m, self.comm_stream
        prof = self._prof.enabled
        cur = torch.cuda.current_stream(self.device)
        ev = self._event(timing=prof)
        ev.record(cur)                       # backward is complete up to here
        pending = self._next_chunk < self.nchunks
        if pending:
            cs.wait_event(ev)
        data["code_wait"] = time.time() - t0
        t2 = time.time()
        self._flush_rest(cs, joined=True)
        self._get_hypers()                   # workers too: keeps the per-group step counters aligned with the server
        data["optim_step_time"] = time.time() - t2
        done = self._event()
        done.record(cs)
        t3 = time.time()
        if not self._ready_per_step:
            # nothing is published into this rank but by its own comm stream
            cur.wait_event(self._published if self._published is not None else done)
        elif not self._gates:
            # the req.Wait() of mpi_comms.py:121 — a one-thread kernel on the compute stream (with a gate registered, the
            # first forward GEMM, BcastLinear / the stem, acquires the flag inside its TMA producer instead)
            m.wait_flags(self._sig_base[self.rank], m.SIG_PARAMS_READY, 1, epoch * self._ready_per_step, self.timeout_s)
            self.launches += 1
        data["comm_wait"] = time.time() - t3
        data["chunks"] = self.nchunks
        if prof:
            ev_d = self._prof.mark(cur)
            self._prof.span("dev_step_tail_time", ev, ev_d)     # backward-done → parameters usable, on the compute stream
            if self._update_spans:
                self._prof.span("dev_gather_update_bcast_time", *self._update_spans[-1])   # the LAST chunk's kernel
                self._prof.span("dev_update_pipeline_time", self._update_spans[0][0], self._update_spans[-1][1])
            self._update_spans = []
            data.update(self._prof.harvest())                   # device timings of the most recent COMPLETED step
        self._end_of_step(data, done)
        return data

    def _end_of_step(self, data, done=None):
        L = self.layout
        nfired = max(len(self._fired), 1)
        data["msg_bytes"] = self._raw_bytes / nfired
        wire_bytes = sum(L.slots[i].ntiles for i in self._fired) * self.bpt if self._fired else 0
        data["packaged_bytes"] = wire_bytes / nfired
        data["engine"] = "device"
        data["micro_batches"] = self._mb.n
        self._epoch += 1
        self._qsgd_step += 1
        if self._ema_on:
            self._ema_n += 1
        if len(self._fired) != L.nparams:
            self._uniform_steps = False              # some parameter sat this step out: per-parameter counts diverge from now on
        for i in self._fired:
            self._param_steps[i] += 1
        self._keep_prev = self._keep
        if done is None:                     # comm-stream completion marker of this step (see _flush)
            done = self._event()
            done.record(self.comm_stream)
        self._prev_done = done
        self._start_step()
        if os.environ.get("PSB200_CHECK") == "1":
            self.check()
        elif self.size > 1 and self._epoch % self._err_every == 0:
            self._poll_error()

    def _poll_error(self):
        """Surface device-side time-outs WITHOUT a sync: every ``PSB200_ERROR_POLL`` steps an async copy of SIG_ERROR
        lands in pinned memory; the previous poll's value is read once its event has completed."""
        if self._err_event is not None and self._err_event.query():
            err = int(self._err_host[0])
            if err:
                raise RuntimeError(f"rank {self.rank}: a device-side wait timed out (code {err}) — a peer is stalled or "
                                   f"dead; synchronisation is disabled until recover() (PSB200_DEVICE_TIMEOUT="
                                   f"{self.timeout_s:.0f} s)")
            self._err_event = None
        if self._err_event is None:
            with torch.cuda.stream(self.comm_stream):
                self._err_host.copy_(self.signal[self.m.SIG_ERROR: self.m.SIG_ERROR + 1], non_blocking=True)
                self._err_event = torch.cuda.Event()
                self._err_event.record(self.comm_stream)

    def recover(self):
        """Collective recovery after a surfaced time-out: bring every rank back to a common, clean protocol state so that
        training can continue (the reference has no failure handling at all; a dead rank hangs ``mpirun`` for good).

        A timed-out step leaves the ranks' epoch clocks and progress flags misaligned (the stalled rank never posted its
        chunks; chunks gathered before the stall may already have been applied and published).  So: quiesce, clear every
        rank's signal pad and error slot, restart the epoch / chunk clocks at zero, re-adopt rank 0's parameters (and, in
        ``allgather`` mode where optimizer state is replicated, rank 0's state and step counts — through the slow object
        path: this is a rare event), and re-open.  Optimizer step counts keep counting the failed step."""
        torch.cuda.synchronize(self.device)
        self.world.barrier()                  # every rank is here: nobody launches into the old epoch any more
        with torch.no_grad():
            self.signal.zero_()               # peers only ever store flags into this pad, and all of them are quiescent
            self.counters.zero_()
            self._consumed.zero_()
            self._select_out.zero_()
            if self.carry is not None:
                self.carry.zero_()            # an open accumulation is dropped
        self._err_host.zero_()
        self._err_event = None
        self._epoch = 0
        self._no_sync = False
        self._start_step()
        self._keep_prev = []
        self._prev_done = None
        self._gate_epoch = -1
        self.version = 0
        self._async_pending, self._async_done_workers = [], set()
        self._snap_version = 0
        if self._snap_shadow is not None:
            self._snap_scratch.copy_(torch.tensor([0, -1, 0, 0, 0, 0], dtype=torch.int64))
            self._snap_event = None
        torch.cuda.synchronize(self.device)
        self.world.barrier()                  # all pads are clean before anybody reads a peer's memory
        if self.size > 1:
            L = self.layout
            nbytes = L.numel_padded * self.psz
            with torch.no_grad():
                src = self.arena.tensor(self.off_stage if self.consistent else self.off_param, nbytes, self.dtype, rank=0)
                if self.rank != 0 or self.consistent:
                    self.param_arena.copy_(src)
                if self.consistent and self.rank != 0:
                    self.stage_arena.copy_(src)
                if self.mode == "allgather":
                    bufs = [b for b in (self.master, self.buf0, self.buf1, self.buf2, self.ema) if b is not None]
                    state = self.world.broadcast_object(
                        ([b.cpu() for b in bufs], self._group_steps, self._param_steps, self._uniform_steps)
                        if self.rank == 0 else None, src=0)
                    if self.rank != 0:
                        for b, v in zip(bufs, state[0]):
                            b.copy_(v)
                        self._group_steps, self._param_steps = list(state[1]), list(state[2])
                        self._uniform_steps = bool(state[3])
                        self._hyper_cache = None
            torch.cuda.synchronize(self.device)
            self.world.barrier()

    @contextlib.contextmanager
    def ema_weights(self):
        """Collective: the parameters of every rank hold the weight average, rounded once to their dtype, inside the block, and
        exactly their previous bits after it.

        Order: the comm stream is drained and this rank's last publication acquired (PARAMS_READY), so every parameter arena
        holds the same, final weights; a barrier; each serving rank saves its served tiles of its own arena and publishes its
        average over them (the update's publication modes, so each rank's arena is written by the ranks that write it in a step);
        sync and barrier, so no rank reads before every rank has published.  The exit syncs and barriers first, so no rank is
        still reading the average when a peer writes into its arena, then publishes the saved tiles the same way, syncs and
        barriers again.
        PARAMS_READY and the epoch clocks do not move: a gated forward inside the block or after it finds its flag raised."""
        if self.mode == "async":
            raise RuntimeError("ema_weights() is not available in mode='async' (read the average through state_dict())")
        if not self._ema_on:
            raise RuntimeError("ema_weights() needs an optimizer built with ema_decay")
        err = None
        if self.accumulating:
            err = "ema_weights() during gradient accumulation: call step() first"
        elif self._fired or self._next_chunk:
            err = "ema_weights() between backward() and step(): chunks of the step are in flight; call step() first"
        elif self._ema_n == 0:
            err = ("ema_weights(): no average has been taken yet (call step() first; after load_state_dict(), every rank must "
                   "load a dict that carries the average, e.g. rank 0's)")
        elif self._in_ema_weights:
            err = "ema_weights() is already active"
        raise_collectively(self.world, self.size, err)
        cur = torch.cuda.current_stream(self.device)
        cur.wait_stream(self.comm_stream)
        if self._gated():
            self.m.wait_flags(self._sig_base[self.rank], self.m.SIG_PARAMS_READY, 1, self._epoch * self._ready_per_step,
                              self.timeout_s)
            self.launches += 1
        torch.cuda.synchronize(self.device)
        self.world.barrier()
        saved = None
        if self.is_server:
            saved = torch.empty(self.state_tiles * TILE, dtype=self.dtype, device=self.device)
            self._to_state(self.param_arena, saved)
        self._in_ema_weights = True
        try:
            self._publish(self.ema)
            torch.cuda.synchronize(self.device)
            self.world.barrier()
            yield
        finally:
            # every rank has finished reading the average (its queued work included) before any rank writes into its arena
            torch.cuda.synchronize(self.device)
            self.world.barrier()
            self._publish(saved)
            torch.cuda.synchronize(self.device)
            self.world.barrier()
            self._in_ema_weights = False

    def _publish(self, src: Optional[torch.Tensor]):
        """Publish the compact ``src`` (fp32 average, or saved parameters) over this rank's served tiles into the arenas."""
        if not self.is_server:
            return
        A = self.arena
        dst = [p + self.off_param for p in A.ptrs] if self.bcast == BCAST_UNICAST else []
        mc = A.mc_ptr + self.off_param if self.bcast == BCAST_MULTICAST else 0
        for lo, hi, c in self._state_pieces(0, self.layout.ntiles):
            self.m.publish(src.data_ptr(), _DT[src.dtype], lo - c, self.layout.ntiles, lo, hi, self.dt, self.bcast, dst, mc,
                           A.local_ptr + self.off_param, num_sms=self._num_sms)
            self.launches += 1

    def resync_master(self):
        """Re-seed the fp32 master weights from the (bf16/fp16) parameters — call after changing parameters in place
        behind the optimizer's back (``model.load_state_dict`` without ``opt.load_state_dict``, manual re-init; evaluating
        with the weight average needs none of this: :meth:`ema_weights`): every update writes master → parameters, so
        un-synced edits would be overwritten."""
        if self.master is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.comm_stream)
            with torch.no_grad():
                self._to_state(self.param_arena, self.master)

    # ------------------------------------------------------------------------------ async mode
    def _step_async(self, data):
        o = self.opt
        sig_base = self._sig_base
        cs = self.comm_stream
        cur = torch.cuda.current_stream(self.device)
        if self.rank != 0:
            self._close_accumulation()
            epoch = self._epoch + 1
            ev = self._event()
            ev.record(cur)
            cs.wait_event(ev)
            self._flush_rest(cs, joined=True)        # chunks not yet encoded during backward (+ inactive parameters)
            with torch.cuda.stream(cs):
                if not self._first_flush_done:       # no parameter produced a gradient at all
                    self._first_flush_done = True
                    self._before_first_encode()
                # publish "gradient `epoch` is in my arena" + the parameter version it was computed on (staleness accounting)
                self.m.signal([sig_base[0]], self.m.SIG_GRAD_READY + self.rank, epoch, -1, 0, 0,
                              self.arena.local_ptr + self.off_signal, self.m.SIG_GRAD_VERSION + self.rank)
                self.launches += 1
            if self.consistent:
                data["param_version"] = self._snapshot()
            self._end_of_step(data)
            return data                      # never waits for NEW parameters (inconsistent reads unless consistent=True)
        # ---- rank 0: the server — device-resident: select → (open sequence lock) → update → ack are all queued without
        # looking at their result; results come back through a ring of pinned slots, read when their event has completed.
        # The host only blocks when it is `_async_depth` iterations AHEAD of the GPU (never the other way round). ----
        self._start_step()
        n = self.size
        self._async_harvest(block=False)
        cand = ((1 << n) - 1) & ~1
        for r in self._async_done_workers:
            cand &= ~(1 << r)
        if cand == 0:
            self._async_harvest(block=True, everything=True)
            data.update(self._async_last)
            data["ps_done"] = True
            data["engine"] = "device"
            return data
        quota = max(1, min(o.quota, bin(cand).count("1")))
        t0 = time.time()
        slot = self._async_ring[self._async_i % len(self._async_ring)]
        self._async_i += 1
        self.version += 1
        hyp = self._hypers()
        self.m.select_ready(sig_base[0], self._consumed.data_ptr(), cand, quota, self._select_out.data_ptr(),
                            self.timeout_s, self.version, sig_base if self.consistent else [], self._cs)
        # the contributors and their count come from the select kernel (select_out), not from contrib_mask / inv_count
        self.plan.launch(o.steps, hyp, 0, 1.0, 0, SIGNAL_PARAMS_READY,
                         ack_mask=0, version=self.version, select_out=self._select_out.data_ptr(),
                         average_dynamic=1 if o.average else 0, active_ptr=0, timeout_s=self.timeout_s, stream=self._cs)
        self.launches += 2
        with torch.cuda.stream(cs):
            slot["host"].copy_(self._select_out, non_blocking=True)
        slot["event"].record(cs)
        if self.ema is not None:
            # once per applied update: the select's count gates it, the device counts the first.  Queued behind the slot's event,
            # so harvesting an iteration waits for its update, not for the average
            L = self.layout
            self.m.ema(*self._ema_src, self.dt, self.ema.data_ptr(), L.ntiles, 0, L.ntiles, 0, self._ema_weight, False,
                       select_out=self._select_out.data_ptr(), count=self._ema_count.data_ptr(), stream=self._cs,
                       num_sms=self._num_sms)
            self.launches += 1
        slot["version"] = self.version
        self._async_pending.append(slot)
        if len(self._async_pending) >= self._async_depth:
            self._async_harvest(block=True)          # the host is a full ring ahead of the device: wait for the oldest
        data["comm_wait"] = time.time() - t0
        data.update(self._async_last)                # contributors / staleness / version of the latest COMPLETED update
        data["param_version_queued"] = self.version
        data["ps_done"] = False
        self._epoch += 1
        data["engine"] = "device"
        return data

    def _async_harvest(self, block: bool, everything: bool = False):
        """Consume completed server iterations in order (``block``: wait for the oldest; ``everything``: drain)."""
        n = self.size
        while self._async_pending:
            slot = self._async_pending[0]
            if not slot["event"].query():
                if not block:
                    return
                slot["event"].synchronize()
            self._async_pending.pop(0)
            h = slot["host"]
            mask, cnt, finished = int(h[0]), int(h[1]), int(h[40])
            for r in range(n):
                if finished >> r & 1:
                    self._async_done_workers.add(r)
            contributors = [r for r in range(n) if mask >> r & 1]
            if cnt == 0:
                # nothing was applied (every worker finished, or the select timed out): the kernels returned early, the
                # sequence lock was never opened, no version was published — take the host-side prediction back
                self.version -= 1
                for gi in range(len(self._group_steps)):
                    self._group_steps[gi] -= 1
            else:
                self._async_applied += 1
                self._async_last = {"contributors": contributors, "param_version": slot["version"],
                                    "staleness": {r: int(h[44 + r]) for r in contributors},
                                    "updates_applied": self._async_applied}
            if not everything:
                block = False                        # at most one blocking wait per call

    # ------------------------------------------------------------------ consistent reads (async)
    def _snapshot(self, block: bool = False) -> int:
        """Adopt the newest COMPLETE parameter version from the staging copy — entirely on the device.

        The server writes ``BEGIN = v`` before and ``VERSION = v`` after publishing version ``v`` into the staging arena.
        ``psb_snapshot_fetch`` copies staging → a local shadow buffer iff ``BEGIN == VERSION`` before and ``BEGIN`` is unchanged
        after (every CTA must agree); ``psb_snapshot_commit`` then copies shadow → the live parameter arena.  A vetoed attempt
        leaves the parameters on the previous whole version, so the model never reads a torn set.  No host reads: the adopted
        version comes back through an async copy into pinned memory and is reported one call late (``block=True``: wait)."""
        m = self.m
        cur = torch.cuda.current_stream(self.device)
        if self._snap_shadow is None:
            self._snap_shadow = torch.empty_like(self.param_arena)
            self._snap_scratch = torch.tensor([0, -1, 0, 0, 0, 0], dtype=torch.int64, device=self.device)
            self._snap_host = torch.zeros(1, dtype=torch.int64).pin_memory()
            self._snap_event = None
        nbytes = self.param_arena.numel() * self.psz
        m.snapshot(self.arena.local_ptr + self.off_signal, self.stage_arena.data_ptr(), self._snap_shadow.data_ptr(),
                   self.param_arena.data_ptr(), nbytes, self._snap_scratch.data_ptr(),
                   int(os.environ.get("PSB200_SNAPSHOT_ATTEMPTS", "2")), cur.cuda_stream)
        self.launches += 4
        if self._snap_event is None or self._snap_event.query() or block:
            if self._snap_event is not None and self._snap_event.query():
                self._snap_version = int(self._snap_host[0])
            self._snap_host.copy_(self._snap_scratch[5:6], non_blocking=True)
            self._snap_event = torch.cuda.Event()
            self._snap_event.record(cur)
        if block:
            self._snap_event.synchronize()
            self._snap_version = int(self._snap_host[0])
        return self._snap_version

    # -------------------------------------------------------------- broadcast-gated GEMM support
    def register_gate(self, layer) -> None:
        """A :class:`~pytorch_ps_mpi_b200.ops.linear.BcastLinear` will acquire ``PARAMS_READY`` itself,
        so worker ``step()`` stops queueing the separate wait kernel (the GEMM is the Wait)."""
        self._gates.append(layer)

    def gate(self):
        """``(flag_ptr, epoch)`` the next forward must observe before reading broadcast weights.  Taking it marks the
        current epoch's broadcast as acquired by a gated kernel (see :meth:`ensure_params`).  In ``mode='sharded'`` the flag
        counts servers: the value is ``epoch * N``, on every rank."""
        if not self._gated():
            return 0, 0
        self._gate_epoch = self._epoch
        return self.arena.local_ptr + self.off_signal + 8 * self.m.SIG_PARAMS_READY, self._epoch * self._ready_per_step

    def _gated(self) -> bool:
        """Does the next forward have to acquire PARAMS_READY (the serve plan: another rank publishes into this one)?"""
        return self._ready_per_step > 0 and self._epoch > 0

    def ensure_params(self):
        """For forwards that bypass the gated kernel (eval mode, unsupported shapes) while a gate is registered: queue
        the plain wait kernel on the current stream unless this epoch's broadcast was already acquired."""
        if not self._gated() or not self._gates:
            return
        if self._gate_epoch == self._epoch:
            return
        self._gate_epoch = self._epoch
        self.m.wait_flags(self._sig_base[self.rank], self.m.SIG_PARAMS_READY, 1, self._epoch * self._ready_per_step,
                          self.timeout_s)
        self.launches += 1

    def peer_param_ptr(self, param: torch.Tensor, rank: int) -> int:
        """Address of ``param`` inside rank ``rank``'s parameter arena as mapped in this process."""
        return self.arena.ptrs[rank] + (param.data_ptr() - self.arena.local_ptr)

    # ------------------------------------------------------------------------------ diagnostics
    def check(self):
        """Raise if any bounded spin timed out (forces a device sync; off the hot path)."""
        torch.cuda.synchronize(self.device)
        err = int(self.signal[self.m.SIG_ERROR].item())
        if err:
            raise RuntimeError(f"rank {self.rank}: a device-side wait timed out (code {err}); "
                               "a peer is stalled or dead")

    def close(self):
        if self._closed:
            return
        self._closed = True
        try:
            if self.mode == "async" and self.size > 1 and self.rank != 0:
                with torch.cuda.stream(self.comm_stream):
                    if self._epoch > 0:      # the server must have consumed our last gradient first
                        self.m.wait_flags(self.arena.local_ptr + self.off_signal, self.m.SIG_ACK, 1,
                                          self._epoch, self.timeout_s)
                    self.m.signal([self.arena.ptrs[0] + self.off_signal],
                                  self.m.SIG_GRAD_READY + self.rank, _DONE_EPOCH)
            torch.cuda.synchronize(self.device)
            self.world.barrier()
            if self.consistent:              # everybody leaves with the server's final parameters
                self._snapshot(block=True)
        finally:
            # parameters keep their arena views alive; detach them so the block can be freed
            with torch.no_grad():
                for s in self.layout.slots:
                    s.param.data = s.param.data.clone()
                    if hasattr(s.param, "ps_grad_out"):
                        del s.param.ps_grad_out
                    if s.param.grad is not None and self._direct_ok:
                        s.param.grad = None          # may alias the wire arena that is about to be unmapped
            self.arena.close()
