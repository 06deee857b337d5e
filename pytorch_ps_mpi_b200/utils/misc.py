"""Observability helpers: byte accounting, parameter lookup, step timers."""
from __future__ import annotations

import sys
import time
from typing import Dict, Iterable, List, Optional

import numpy as np
import torch


def bytes_of(obj) -> int:
    """Recursive payload-size estimate of tensors / arrays / containers.

    Parity with ``_bytes_of`` (``/root/reference/ps.py:25-43``) with its documented bug fixed:
    the reference's comment says 2-D arrays were mis-sized (``ps.py:26-27``); here every tensor
    and ndarray counts ``numel * element_size`` and a tensor's ``.grad`` is included.
    """
    if isinstance(obj, torch.Tensor):
        n = obj.element_size() * obj.numel()
        g = obj.grad if obj.requires_grad and obj.is_leaf else None
        return n + (bytes_of(g) if g is not None else 0)
    if isinstance(obj, np.ndarray):
        return int(obj.nbytes)
    if isinstance(obj, dict):
        return sum(bytes_of(v) for v in obj.values())
    if isinstance(obj, (tuple, list)):
        return sum(bytes_of(v) for v in obj)
    if isinstance(obj, (bytes, bytearray, memoryview)):
        return len(obj)
    return sys.getsizeof(obj)


_bytes_of = bytes_of   # the reference's private name


def find_param(params: Iterable[torch.Tensor], name: str) -> torch.Tensor:
    """Look a parameter up by the ``.name`` the optimizer tagged it with (``ps.py:46-50``)."""
    matches = [p for p in params if getattr(p, "ps_name", getattr(p, "name", None)) == name]
    if len(matches) > 1:
        raise ValueError("More than one name found")
    if not matches:
        raise KeyError(f"no parameter named {name!r}")
    return matches[0]


class StepTimer:
    """Wall-clock section timer that accumulates into a dict (the reference's ``data`` dict idiom)."""

    def __init__(self, data: Optional[Dict[str, float]] = None):
        self.data = data if data is not None else {}
        self._t = time.time()

    def lap(self, key: str, accumulate: bool = True) -> float:
        now = time.time()
        dt = now - self._t
        self._t = now
        self.data[key] = self.data.get(key, 0.0) + dt if accumulate else dt
        return dt

    def reset(self):
        self._t = time.time()


class CudaStepTimer:
    """Device-side section timing with CUDA events, read one step late (never forces a sync)."""

    def __init__(self, enabled: bool):
        self.enabled = enabled and torch.cuda.is_available()
        self._pending: List[tuple] = []
        self.last: Dict[str, float] = {}

    def mark(self, stream=None):
        if not self.enabled:
            return None
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(stream)
        return ev

    def span(self, key: str, start, end):
        if self.enabled and start is not None and end is not None:
            self._pending.append((key, start, end))

    def harvest(self) -> Dict[str, float]:
        """Collect every completed span (seconds); incomplete ones stay queued."""
        keep = []
        for key, s, e in self._pending:
            if e.query():
                self.last[key] = s.elapsed_time(e) * 1e-3
            else:
                keep.append((key, s, e))
        self._pending = keep
        return dict(self.last)


def summarize_timings(timings: Iterable[Dict[str, float]]) -> Dict[str, Dict[str, float]]:
    """Aggregate the per-step ``data`` dicts an optimizer keeps in ``opt.timings`` (the list the reference
    declared but never filled, ``/root/reference/ps.py:80``): ``{key: {mean, max, total, n}}`` for numeric keys."""
    acc: Dict[str, List[float]] = {}
    for d in timings:
        for k, v in d.items():
            if isinstance(v, (int, float)) and not isinstance(v, bool):
                acc.setdefault(k, []).append(float(v))
    return {k: {"mean": sum(v) / len(v), "max": max(v), "total": sum(v), "n": len(v)} for k, v in acc.items()}


def dump_chrome_trace(timings: Iterable[Dict[str, float]], path: str, pid: int = 0) -> None:
    """Write the host-side sections of every step as a Chrome / Perfetto trace (``chrome://tracing``)."""
    import json
    events, t = [], 0.0
    for step, d in enumerate(timings):
        for key in ("code_wait", "iallgather_prepare_time", "isend_time", "comm_wait", "decode_time", "optim_step_time"):
            dur = float(d.get(key, 0.0) or 0.0) * 1e6
            if dur > 0:
                events.append({"name": key, "ph": "X", "ts": t, "dur": dur, "pid": pid, "tid": 0, "args": {"step": step}})
                t += dur
    with open(path, "w") as f:
        json.dump({"traceEvents": events, "displayTimeUnit": "ms"}, f)


class MicroBatchCounter:
    """Counts the backward passes summed into one step from hook firings: a new one starts at the first hook after ``reset()`` or
    ``cut()`` (entering or leaving ``no_sync()``), or when a parameter fires again."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.n, self._seen = 0, None

    def cut(self):
        self._seen = None

    def fire(self, key) -> bool:
        """Record a hook firing; True when it opens a new backward pass."""
        if self._seen is not None and key not in self._seen:
            self._seen.add(key)
            return False
        self.n += 1
        self._seen = {key}
        return True


def raise_collectively(world, size: int, err) -> None:
    """A collective refusal: every rank raises ``RuntimeError`` when any rank has a reason ``err`` (the lowest rank's is
    reported), so no rank is left waiting in a collective that the others never reach.  ``err`` is ``None`` or a message."""
    every = world.all_gather_object(err) if size > 1 else [err]
    bad = [(r, e) for r, e in enumerate(every) if e is not None]
    if bad:
        r, e = bad[0]
        raise RuntimeError(e if size == 1 else f"rank {r}: {e}")
