"""Explicit-state model of the device engine's epoch-flag protocol (race / deadlock checker, runs on CPU).

The reference has no race detection at all and assumes "communication is reliable"
(``/root/reference/README.md:17-21``); its ordering comes for free from blocking ``req.Wait()`` calls
(``/root/reference/ps.py:146``, ``/root/reference/mpi_comms.py:110,121``).  Here the waits are epoch flags in a
symmetric signal pad that kernels on two CUDA streams per rank raise and poll (``csrc/kernels/ps_kernels.cu``,
``parallel/device_engine.py``), so the ordering argument has to be made explicitly.  This module makes it
mechanically: it writes down, per rank and per stream, the sequence of device operations ``DeviceEngine`` queues
for ``E`` training steps, and explores EVERY interleaving of those sequences, checking

* **no data race** — a kernel never writes a buffer (wire arena, parameter arena, staging arena) while another
  kernel's access to it is in flight, except where the mode allows it by design (AsySG-InCon's inconsistent
  parameter reads, ``/root/reference/README.md:79-81``),
* **no stale or too-new data** — the server sums exactly the epoch-``e`` gradients, step ``e+1`` runs on exactly
  the epoch-``e`` parameters (synchronous modes), an accepted ``consistent=True`` snapshot is never torn,
* **no lost or duplicated gradient** in async mode, and acknowledgements only for consumed gradients,
* **no deadlock** — some stream can always make progress until every stream has drained.

``compute-sanitizer --tool racecheck`` (``scripts/sanitize.sh``) covers intra-kernel hazards on one GPU; this
covers the cross-GPU protocol, which no tool on the box can see.  The "mutants" in ``tests/test_protocol_model.py``
delete one wait at a time and assert that the checker then finds the race / deadlock, so a green run means
something.

Kernels are modelled as intervals (``acq`` … ``rel``) over named resources, flags as integer slots, CUDA events as
flags.  Operations that can never be disabled again and that nobody can observe the absence of (event records,
satisfied waits, stores into slots that are only ever waited on with ``>=``) are executed eagerly with the
operation before them — a sound partial-order reduction that keeps the state space small enough for exhaustive
search at 2–4 ranks and 2–3 epochs.

CLI: ``python -m pytorch_ps_mpi_b200.parallel.protocol_model --mode ps --ranks 3 --epochs 2``.
"""
from __future__ import annotations

import argparse
import sys
from dataclasses import dataclass, field
from typing import Dict, FrozenSet, Iterable, List, Optional, Sequence, Tuple

__all__ = ["Violation", "Result", "Model", "build_ps", "build_ps_unpipelined", "build_allgather", "build_allgather_unpipelined", "build_async", "build_ps_accumulate", "build_sharded", "build_stem_pipeline", "build_stem_wgrad_pipeline",
           "check", "MODES"]

DONE = 1 << 62          # device_engine._DONE_EPOCH / PSB_DONE_EPOCH


class Violation(Exception):
    """A protocol property failed; ``trace`` is the interleaving (list of ``"proc: op"``) that reaches it."""

    def __init__(self, kind: str, detail: str, trace: List[str]):
        super().__init__(f"{kind}: {detail}")
        self.kind, self.detail, self.trace = kind, detail, trace


@dataclass
class Result:
    states: int
    transitions: int
    finals: int


# --------------------------------------------------------------------------------------------
# model container
# --------------------------------------------------------------------------------------------
@dataclass
class Model:
    """Processes (one per rank and stream), flag slots and resources of one protocol instance."""
    names: List[str] = field(default_factory=list)            # process names
    progs: List[list] = field(default_factory=list)           # op lists (Script) or AsyncServer objects
    flag_ix: Dict[object, int] = field(default_factory=dict)
    res_ix: Dict[object, int] = field(default_factory=dict)
    racy_ok: set = field(default_factory=set)                 # resources whose read/write overlap is allowed
    nregs: int = 4
    final_checks: list = field(default_factory=list)          # callables(state, model) -> Optional[str]

    def flag(self, key) -> int:
        return self.flag_ix.setdefault(key, len(self.flag_ix))

    def res(self, key) -> int:
        return self.res_ix.setdefault(key, len(self.res_ix))

    def add(self, name: str, prog) -> int:
        self.names.append(name)
        self.progs.append(prog)
        return len(self.names) - 1


# Script ops (tuples):
#   ("rec", ev) / ("wev", ev)                  CUDA event record / stream-wait-event
#   ("sig", key, value)                        store `value` into flag slot `key`
#   ("add", key, delta)                        flag slot `key` += delta (a release add: a counting flag)
#   ("wait", key, value)                       spin until slot >= value
#   ("acq", [(res, mode, expect), ...])        a kernel starts accessing resources ('r' / 'w'; expect = version or None)
#   ("rel", [(res, mode, newver), ...])        the kernel finished (a write leaves version `newver`)
#   ("load", reg, key)                         host read of a flag slot into a register
#   ("jne", reg_a, reg_b, target)              if regs differ jump
#   ("jeqc", reg, const_reg, target)           if reg == other reg jump   (alias of the inverse of jne)
#   ("mov", reg_dst, reg_src)
#   ("accept", reg)                            seqlock reader adopts the copy it just made; must be clean & == reg


def _set(t: tuple, i: int, v) -> tuple:
    return t[:i] + (v,) + t[i + 1:]


# state = (locals, flags, vers, infl)
#   locals : tuple per process of (pc, regs tuple, torn flag, version seen at acq)
#   flags  : tuple of ints
#   vers   : tuple of ints (content version per resource)
#   infl   : tuple per resource of a sorted tuple of (proc, mode)


class _Explorer:
    def __init__(self, model: Model, max_states: int):
        self.m = model
        self.max_states = max_states
        self.observed = set()          # flag slots whose stores are visible scheduling points
        for p in model.progs:          # register every slot / resource up front: state tuples have a fixed shape
            if isinstance(p, AsyncServer):
                self.observed |= p.observed(model)
                p.register(model)
                continue
            for op in p:
                k = op[0]
                if k in ("rec", "wev"):
                    model.flag(("ev", op[1]))
                elif k in ("sig", "add", "wait"):
                    model.flag(op[1])
                elif k == "load":
                    self.observed.add(model.flag(op[2]))
                elif k in ("acq", "rel"):
                    for item in op[1]:
                        model.res(item[0])

    # ---- helpers -------------------------------------------------------------------------
    def initial(self):
        m = self.m
        locs = []
        for p in m.progs:
            if isinstance(p, AsyncServer):
                locs.append(p.initial(m))
            else:
                locs.append((0, (0,) * m.nregs, False, -1))
        st = (tuple(locs), (0,) * len(m.flag_ix), (0,) * len(m.res_ix), ((),) * len(m.res_ix))
        for i in range(len(m.progs)):
            st = self._run_eager(st, i)
        return st

    def _eager(self, st, i) -> bool:
        """Is process i's next op one that may be folded into its predecessor?"""
        p = self.m.progs[i]
        if isinstance(p, AsyncServer):
            return False
        pc = st[0][i][0]
        if pc >= len(p):
            return False
        op = p[pc]
        k = op[0]
        if k == "rec":
            return True
        if k == "wev":
            return st[1][self.m.flag(("ev", op[1]))] >= 1
        if k == "wait":
            return st[1][self.m.flag(op[1])] >= op[2]
        if k in ("sig", "add"):
            return self.m.flag(op[1]) not in self.observed
        if k in ("jne", "jeqc", "mov"):
            return True
        return False

    def _run_eager(self, st, i):
        while self._eager(st, i):
            st = self._exec(st, i, [])[0]
        return st

    def enabled(self, st, i) -> bool:
        p = self.m.progs[i]
        if isinstance(p, AsyncServer):
            return p.enabled(st, i, self.m)
        pc = st[0][i][0]
        if pc >= len(p):
            return False
        op = p[pc]
        if op[0] == "wev":
            return st[1][self.m.flag(("ev", op[1]))] >= 1
        if op[0] == "wait":
            return st[1][self.m.flag(op[1])] >= op[2]
        return True

    def finished(self, st, i) -> bool:
        p = self.m.progs[i]
        if isinstance(p, AsyncServer):
            return p.finished(st, i)
        return st[0][i][0] >= len(p)

    # resource access bookkeeping, shared by Script and AsyncServer
    def acquire(self, st, i, items, trace):
        m = self.m
        locs, flags, vers, infl = st
        script = not isinstance(m.progs[i], AsyncServer)
        torn, seen = (locs[i][2], locs[i][3]) if script else (False, -1)
        for res_key, mode, expect in items:
            r = m.res(res_key)
            others = [(q, md) for q, md in infl[r] if q != i]
            overlap = [(q, md) for q, md in others if mode == "w" or md == "w"]
            if overlap:
                if res_key in m.racy_ok:
                    if mode == "r":
                        torn = True                       # my copy overlaps a write
                    else:
                        for q, md in overlap:             # their copies are torn by my write
                            if md == "r":
                                l = locs[q]
                                locs = _set(locs, q, (l[0], l[1], True, l[3]))
                else:
                    q, md = overlap[0]
                    raise Violation("race", f"{m.names[i]} starts {'writing' if mode == 'w' else 'reading'} {res_key} "
                                    f"while {m.names[q]} is {'writing' if md == 'w' else 'reading'} it", trace)
            if expect is not None and vers[r] != expect:
                raise Violation("version", f"{m.names[i]} accesses {res_key} expecting version {expect}, "
                                f"found {vers[r]}", trace)
            if mode == "r":
                seen = vers[r]
            infl = _set(infl, r, tuple(sorted(infl[r] + ((i, mode),))))
        if script:
            locs = _set(locs, i, (locs[i][0], locs[i][1], torn, seen))
        return (locs, flags, vers, infl)

    def release(self, st, i, items):
        m = self.m
        locs, flags, vers, infl = st
        for res_key, mode, newver in items:
            r = m.res(res_key)
            cur = list(infl[r])
            cur.remove((i, mode))
            infl = _set(infl, r, tuple(cur))
            if mode == "w" and newver is not None:
                vers = _set(vers, r, newver)
        return (locs, flags, vers, infl)

    # ---- one transition ------------------------------------------------------------------
    def _exec(self, st, i, trace) -> list:
        m = self.m
        p = m.progs[i]
        if isinstance(p, AsyncServer):
            return p.fire(st, i, self, trace)
        locs, flags, vers, infl = st
        pc, regs, torn, seen = locs[i]
        op = p[pc]
        k = op[0]
        npc = pc + 1
        if k == "rec":
            flags = _set(flags, m.flag(("ev", op[1])), 1)
        elif k in ("wev", "wait"):
            pass
        elif k == "sig":
            flags = _set(flags, m.flag(op[1]), op[2])
        elif k == "add":
            flags = _set(flags, m.flag(op[1]), flags[m.flag(op[1])] + op[2])
        elif k == "acq":
            locs2 = _set(locs, i, (pc, regs, False, -1))
            st2 = self.acquire((locs2, flags, vers, infl), i, op[1], trace)
            locs, flags, vers, infl = st2
            pc_, regs, torn, seen = locs[i]
        elif k == "rel":
            locs, flags, vers, infl = self.release(st, i, op[1])
            pc_, regs, torn, seen = locs[i]
        elif k == "load":
            regs = _set(regs, op[1], flags[m.flag(op[2])])
        elif k == "jne":
            if regs[op[1]] != regs[op[2]]:
                npc = op[3]
        elif k == "jeqc":
            if regs[op[1]] == regs[op[2]]:
                npc = op[3]
        elif k == "mov":
            regs = _set(regs, op[1], regs[op[2]])
        elif k == "accept":
            if torn:
                raise Violation("torn-snapshot", f"{m.names[i]} adopts a copy that overlapped a publish", trace)
            if seen != regs[op[1]]:
                raise Violation("version", f"{m.names[i]} adopts version {seen} believing it is {regs[op[1]]}", trace)
        else:
            raise ValueError(op)
        locs = _set(locs, i, (npc, regs, torn, seen))
        return [(locs, flags, vers, infl)]

    def successors(self, st, i, trace):
        out = []
        for s in self._exec(st, i, trace):
            out.append(self._run_eager(s, i))
        return out

    def describe(self, st, i) -> str:
        p = self.m.progs[i]
        if isinstance(p, AsyncServer):
            return f"{self.m.names[i]}: {p.describe(st, i)}"
        return f"{self.m.names[i]}: {p[st[0][i][0]]}"

    # ---- exhaustive search ---------------------------------------------------------------
    def run(self) -> Result:
        m = self.m
        n = len(m.progs)
        init = self.initial()
        seen = {init}
        stack = [(init, None, None)]
        parent = {init: (None, None)}
        transitions = finals = 0

        def trace_of(st, extra=None):
            t = []
            while st is not None:
                pst, label = parent[st]
                if label is not None:
                    t.append(label)
                st = pst
            t.reverse()
            if extra:
                t.append(extra)
            return t

        work = [init]
        while work:
            st = work.pop()
            progressed = False
            for i in range(n):
                if not self.enabled(st, i):
                    continue
                progressed = True
                label = self.describe(st, i)
                try:
                    succ = self.successors(st, i, None)
                except Violation as v:
                    v.trace = trace_of(st, label)
                    raise
                for s in succ:
                    transitions += 1
                    if s not in seen:
                        if len(seen) >= self.max_states:
                            raise RuntimeError(f"state space larger than {self.max_states}")
                        seen.add(s)
                        parent[s] = (st, label)
                        work.append(s)
            if not progressed:
                if all(self.finished(st, i) for i in range(n)):
                    finals += 1
                    for chk in m.final_checks:
                        msg = chk(st, m)
                        if msg:
                            raise Violation("final", msg, trace_of(st))
                else:
                    stuck = [self.describe(st, i) for i in range(n) if not self.finished(st, i)]
                    raise Violation("deadlock", "no stream can make progress; blocked at " + "; ".join(stuck),
                                    trace_of(st))
        return Result(len(seen), transitions, finals)


# --------------------------------------------------------------------------------------------
# the asynchronous server (rank 0 in mode='async'): select → update → ack, data dependent
# --------------------------------------------------------------------------------------------
class AsyncServer:
    """``DeviceEngine._step_async`` on rank 0 + ``psb_select_kernel`` + the async path of ``psb_update_kernel``.

    local state: (phase, consumed[N], last_served, done_mask, chosen_mask, applied[N], version)
    phases: 0 = select, 1 = update kernel starts, 2 = update kernel ends (+ flags), 3 = finished.
    """

    def __init__(self, n: int, quota: int, consistent: bool, *, ack_current: bool = True, raise_begin: bool = True):
        self.n, self.quota, self.consistent, self.ack_current = n, quota, consistent, ack_current
        self.raise_begin = raise_begin
        self.dest = "stage" if consistent else "params"

    def observed(self, m: Model):
        return {m.flag(("GRAD_READY", 0, r)) for r in range(1, self.n)}

    def register(self, m: Model):
        for r in range(self.n):
            for key in (("GRAD_READY", 0, r), ("ACK", r), ("VERSION", r), ("BEGIN", r)):
                m.flag(key)
            for key in (("wire", r), ("wireA", r), (self.dest, r)):
                m.res(key)

    def initial(self, m: Model):
        return (0, (0,) * self.n, 0, 0, 0, (0,) * self.n, 0)

    def finished(self, st, i):
        return st[0][i][0] == 3

    def _ready(self, st, i, m):
        phase, consumed, last, done, chosen, applied, ver = st[0][i]
        cand = [r for r in range(1, self.n) if not done >> r & 1]
        vals = {r: st[1][m.flag(("GRAD_READY", 0, r))] for r in cand}
        fin = [r for r in cand if vals[r] >= DONE]
        ready = [r for r in cand if vals[r] < DONE and vals[r] > consumed[r]]
        need = min(self.quota, len(cand) - len(fin))
        return cand, vals, fin, ready, need

    def enabled(self, st, i, m):
        phase = st[0][i][0]
        if phase == 0:
            cand, vals, fin, ready, need = self._ready(st, i, m)
            return (not cand) or need == 0 or len(ready) >= need
        return phase in (1, 2)

    def describe(self, st, i):
        return ("select", "update-begin", "update-end", "done")[st[0][i][0]] + f" {st[0][i][1:]}"

    def fire(self, st, i, ex: "_Explorer", trace):
        m = ex.m
        locs, flags, vers, infl = st
        phase, consumed, last, done, chosen, applied, ver = locs[i]
        n = self.n
        if phase == 0:
            cand, vals, fin, ready, need = self._ready(st, i, m)
            if not cand:                                  # `if cand == 0: ps_done`
                return [(_set(locs, i, (3, consumed, last, done, 0, applied, ver)), flags, vers, infl)]
            pick = []
            for k in range(n):                            # rotating priority (psb_select_kernel)
                r = (last + 1 + k) % n
                if r in ready and len(pick) < need:
                    pick.append(r)
            mask = 0
            for r in pick:
                mask |= 1 << r
                consumed = _set(consumed, r, vals[r])
            if pick:
                last = max(pick)
            for r in fin:
                done |= 1 << r
            if not pick:                                  # nothing applied; loop (ps_done once cand empties)
                return [(_set(locs, i, (0, consumed, last, done, 0, applied, ver)), flags, vers, infl)]
            ver += 1
            if self.consistent and self.raise_begin:
                for r in range(n):
                    flags = _set(flags, m.flag(("BEGIN", r)), ver)
            return [(_set(locs, i, (1, consumed, last, done, mask, applied, ver)), flags, vers, infl)]
        if phase == 1:
            items = [(("wire", r), "r", consumed[r]) for r in range(n) if chosen >> r & 1]
            items += [(("wireA", r), "r", consumed[r]) for r in range(n) if chosen >> r & 1]
            # consistent=True publishes into the staging arenas; the workers' live parameters are theirs alone
            items += [((self.dest, r), "w", None) for r in range(n)]
            st2 = ex.acquire((_set(locs, i, (2, consumed, last, done, chosen, applied, ver)), flags, vers, infl),
                             i, items, trace)
            return [st2]
        # phase 2: kernel done → versions, VERSION flags, ACKs
        items = [(("wire", r), "r", None) for r in range(n) if chosen >> r & 1]
        items += [(("wireA", r), "r", None) for r in range(n) if chosen >> r & 1]
        items += [((self.dest, r), "w", ver) for r in range(n)]
        locs, flags, vers, infl = ex.release(st, i, items)
        for r in range(n):
            if self.consistent and not self.raise_begin:
                flags = _set(flags, m.flag(("BEGIN", r)), ver)     # mutant: the lock is only "opened" at the end
            flags = _set(flags, m.flag(("VERSION", r)), ver)
        for r in range(n):
            if chosen >> r & 1:
                e = flags[m.flag(("GRAD_READY", 0, r))] if self.ack_current else consumed[r]
                if e < DONE and e != consumed[r]:
                    raise Violation("ack", f"server acknowledges gradient {e} of rank {r} but consumed {consumed[r]}",
                                    trace)
                flags = _set(flags, m.flag(("ACK", r)), max(flags[m.flag(("ACK", r))], min(e, DONE)))
                applied = _set(applied, r, applied[r] + 1)
        return [(_set(locs, i, (0, consumed, last, done, 0, applied, ver)), flags, vers, infl)]


# --------------------------------------------------------------------------------------------
# protocol instances — each mirrors what DeviceEngine queues; `drop` removes one wait (mutation testing)
# --------------------------------------------------------------------------------------------
def _backward(m: Model, r: int, e: int, comp: list, comm: list, expect, *, prev_done: bool, pre_encode: list):
    """forward+backward of step e on the compute stream, two encode buckets on the comm stream.

    ``pre_encode``: ops ``_before_first_encode`` queues on the comm stream ahead of the first wire write."""
    if prev_done and e > 1:
        # _flush: the compute stream may not run more than one step ahead of the comm stream
        comp.append(("wev", ("done", r, e - 1)))
    # forward + backward read the parameters; the gradients of the first bucket are final at `mid` (a hook fired),
    # the rest at `bwd`.  Gradient tensors are fresh allocations every step (kept alive by DeviceEngine._keep until
    # the step after), hence one resource per epoch.
    comp.append(("acq", [(("params", r), "r", expect), (("gradA", r, e), "w", None)]))
    comp.append(("rel", [(("gradA", r, e), "w", e)]))
    comp.append(("rec", ("mid", r, e)))
    comp.append(("acq", [(("gradB", r, e), "w", None)]))
    comp.append(("rel", [(("params", r), "r", None), (("gradB", r, e), "w", e)]))
    comp.append(("rec", ("bwd", r, e)))                           # step(): backward complete
    comm.append(("wev", ("mid", r, e)))
    comm.extend(pre_encode)
    comm.append(("acq", [(("gradA", r, e), "r", e), (("wireA", r), "w", None)]))
    comm.append(("rel", [(("gradA", r, e), "r", None), (("wireA", r), "w", e)]))
    comm.append(("wev", ("bwd", r, e)))
    comm.append(("acq", [(("gradB", r, e), "r", e), (("wire", r), "w", None)]))
    comm.append(("rel", [(("gradB", r, e), "r", None), (("wire", r), "w", e)]))


def _backward_chunks(m: Model, r: int, e: int, comp: list, *, prev_done: bool):
    """forward + backward of step e on the compute stream, seen by the PIPELINED engine: the arena is two chunks, A (the
    layers whose gradients come first) and B.  Forward reads both; backward reads A's weights while it produces gradA
    (hook fires → ``mid``), then B's weights while it produces gradB (→ ``bwd``)."""
    if prev_done and e > 1:
        comp.append(("wev", ("done", r, e - 1)))                   # _flush_chunk: at most one step ahead of the comm stream
    comp.append(("acq", [(("paramsA", r), "r", e - 1), (("paramsB", r), "r", e - 1), (("gradA", r, e), "w", None)]))
    comp.append(("rel", [(("paramsA", r), "r", None), (("gradA", r, e), "w", e)]))
    comp.append(("rec", ("mid", r, e)))
    comp.append(("acq", [(("gradB", r, e), "w", None)]))
    comp.append(("rel", [(("paramsB", r), "r", None), (("gradB", r, e), "w", e)]))
    comp.append(("rec", ("bwd", r, e)))


def _chunk_final(m: Model, n: int, epochs: int):
    def final(st, mm):
        for p in range(n):
            for c in ("paramsA", "paramsB"):
                if st[2][mm.res((c, p))] != epochs:
                    return f"rank {p} ends on {c} version {st[2][mm.res((c, p))]}, expected {epochs}"
    m.final_checks.append(final)


def build_ps(n: int, epochs: int, drop: Optional[str] = None) -> Model:
    """``mode='ps'`` with the per-chunk update pipeline (``DeviceEngine._flush_chunk``): rank 0 gathers / updates /
    publishes chunk A as soon as every rank's GRAD_READY progress value says "chunk A of step e is in my arena" — while
    every rank's backward is still running on chunk B — then chunk B, then raises PARAMS_READY.  GRAD_READY carries the
    monotone value ``(e-1)*2 + chunk + 1``.

    ``drop``: ``'params_ready'`` (workers do not wait for the broadcast), ``'grad_ready'`` (the server does not wait for
    chunk B's flags), ``'grad_ready_a'`` (nor for chunk A's), ``'bwd_event'`` (the last encode does not wait for backward),
    ``'mid_event'`` (chunk A is encoded / flagged before its gradients exist), ``'progress_off_by_one'`` (chunk B's update
    waits for chunk A's value) — each must be caught."""
    m = Model()
    prog = lambda e, c: (e - 1) * 2 + c + 1      # noqa: E731
    for r in range(n):
        comp, comm = [], []
        for e in range(1, epochs + 1):
            if r != 0 and e > 1 and drop != "params_ready":
                comp.append(("wait", ("PARAMS_READY", r), e - 1))      # psb_wait_kernel (or the gated first GEMM)
            if r == 0 and e > 1:
                comp.append(("wev", ("done", 0, e - 1)))               # cur.wait_event(done)
            _backward_chunks(m, r, e, comp, prev_done=(r != 0))
            for c, (ev, grad, wire, par) in enumerate((("mid", "gradA", "wireA", "paramsA"), ("bwd", "gradB", "wire", "paramsB"))):
                if not ((drop == "bwd_event" and ev == "bwd") or (drop == "mid_event" and ev == "mid")):
                    comm.append(("wev", (ev, r, e)))
                comm.append(("acq", [((grad, r, e), "r", e), ((wire, r), "w", None)]))      # psb_encode_kernel, chunk c
                comm.append(("rel", [((grad, r, e), "r", None), ((wire, r), "w", e)]))
                if r != 0:
                    comm.append(("sig", ("GRAD_READY", 0, r), prog(e, c)))                    # its last CTA raises the flag
                    continue
                skip = (drop == "grad_ready" and c == 1) or (drop == "grad_ready_a" and c == 0)
                if not skip:
                    want = prog(e, 0) if (drop == "progress_off_by_one" and c == 1) else prog(e, c)
                    for p in range(1, n):
                        comm.append(("wait", ("GRAD_READY", 0, p), want))
                reads = [((wire, p), "r", e) for p in range(n)]                               # psb_update_kernel, chunk c
                comm.append(("acq", reads + [((par, p), "w", None) for p in range(n)]))
                comm.append(("rel", [(k, md, None) for k, md, _ in reads] + [((par, p), "w", e) for p in range(n)]))
            if r == 0:
                for p in range(n):
                    comm.append(("sig", ("PARAMS_READY", p), e))                              # raised by the LAST chunk's kernel
            comm.append(("rec", ("done", r, e)))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)
    _chunk_final(m, n, epochs)
    return m


def build_ps_accumulate(n: int, epochs: int, drop: Optional[str] = None) -> Model:
    """``mode='ps'`` (pipelined, two chunks) with gradient accumulation: every step is one backward inside ``no_sync()`` and a
    final one.  The carry of each chunk is a resource: the no_sync backward's gradients are added into it by an accumulate
    launch on the COMPUTE stream (``DeviceEngine._flush_accumulate``; the first of a step waits for the comm stream's ``done``
    of the previous step, whose encodes zeroed the carry); the final backward's encode on the comm stream reads and zeroes it.
    After a direct-placement step ``param.grad`` may still view the wire tile; the hook drops it, so AccumulateGrad assigns the
    final gradient instead of adding it into the tile after the encode wrote it.

    ``drop``: ``'prev_done'`` (the first accumulate does not wait for the previous step's encodes), ``'alias'`` (the hook keeps a
    ``param.grad`` that views the wire tile: AccumulateGrad adds into it after the final encode) — each must be caught."""
    m = Model()
    prog = lambda e, c: (e - 1) * 2 + c + 1      # noqa: E731
    for r in range(n):
        comp, comm = [], []
        for e in range(1, epochs + 1):
            if r != 0 and e > 1:
                comp.append(("wait", ("PARAMS_READY", r), e - 1))
            if r == 0 and e > 1:
                comp.append(("wev", ("done", 0, e - 1)))
            # micro-batch 1, inside no_sync(): its gradients are fresh tensors, summed into the carry on the compute stream
            comp.append(("acq", [(("paramsA", r), "r", e - 1), (("paramsB", r), "r", e - 1), (("accg", r, e), "w", None)]))
            comp.append(("rel", [(("paramsA", r), "r", None), (("paramsB", r), "r", None), (("accg", r, e), "w", e)]))
            if e > 1 and drop != "prev_done":
                comp.append(("wev", ("done", r, e - 1)))
            comp.append(("acq", [(("accg", r, e), "r", e), (("carryA", r), "w", 2 * e - 2), (("carryB", r), "w", 2 * e - 2)]))
            comp.append(("rel", [(("accg", r, e), "r", None), (("carryA", r), "w", 2 * e - 1), (("carryB", r), "w", 2 * e - 1)]))
            # the final backward: the pipelined chunks, each encoded with its carry
            _backward_chunks(m, r, e, comp, prev_done=(r != 0))
            if drop == "alias" and r != 0:
                # AccumulateGrad adds the chunk-B gradient into param.grad, which still views the wire tile
                comp.append(("acq", [(("wire", r), "w", None)]))
                comp.append(("rel", [(("wire", r), "w", None)]))
            for c, (ev, grad, wire, par, carry) in enumerate((("mid", "gradA", "wireA", "paramsA", "carryA"),
                                                              ("bwd", "gradB", "wire", "paramsB", "carryB"))):
                comm.append(("wev", (ev, r, e)))
                comm.append(("acq", [((grad, r, e), "r", e), ((carry, r), "w", 2 * e - 1), ((wire, r), "w", None)]))
                comm.append(("rel", [((grad, r, e), "r", None), ((carry, r), "w", 2 * e), ((wire, r), "w", e)]))
                if r != 0:
                    comm.append(("sig", ("GRAD_READY", 0, r), prog(e, c)))
                    continue
                for p in range(1, n):
                    comm.append(("wait", ("GRAD_READY", 0, p), prog(e, c)))
                reads = [((wire, p), "r", e) for p in range(n)]
                comm.append(("acq", reads + [((par, p), "w", None) for p in range(n)]))
                comm.append(("rel", [(k, md, None) for k, md, _ in reads] + [((par, p), "w", e) for p in range(n)]))
            if r == 0:
                for p in range(n):
                    comm.append(("sig", ("PARAMS_READY", p), e))
            comm.append(("rec", ("done", r, e)))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)
    _chunk_final(m, n, epochs)
    return m


def build_sharded(n: int, epochs: int, drop: Optional[str] = None) -> Model:
    """``mode='sharded'`` (pipelined, two chunks A and B): rank ``s`` serves shard ``s`` of each chunk.  Every rank encodes
    its whole gradient and raises its GRAD_READY progress in every peer's pad; the owner of a shard waits for every peer's
    progress, reads shard ``s`` of every rank's wire chunk and writes parameter shard ``s`` on every rank.  After its chunk-B
    shard each rank adds 1 to every rank's PARAMS_READY, and the next step's forward waits for ``>= e * N`` (every rank,
    rank 0 included).  Parameter and wire resources are per shard.

    ``drop``: ``'params_ready'`` (no wait before the forward), ``'count_short'`` (wait for ``e * (N - 1)`` only),
    ``'grad_ready'`` (the owner of B's shard 0 skips one peer's wait), ``'signal_server_only'`` (GRAD_READY goes to rank 0
    only, as in mode='ps') — each must be caught."""
    m = Model()
    prog = lambda e, c: (e - 1) * 2 + c + 1      # noqa: E731
    for r in range(n):
        comp, comm = [], []
        peers = [p for p in range(n) if p != r]
        for e in range(1, epochs + 1):
            if e > 1 and drop != "params_ready":
                comp.append(("wait", ("PARAMS_READY", r), (e - 1) * (n - 1 if drop == "count_short" else n)))
            if e > 1:
                comp.append(("wev", ("done", r, e - 1)))                   # _flush_chunk: at most one step ahead
            pa = [(("paramsA", s, r), "r", e - 1) for s in range(n)]
            pb = [(("paramsB", s, r), "r", e - 1) for s in range(n)]
            comp.append(("acq", pa + pb + [(("gradA", r, e), "w", None)]))
            comp.append(("rel", [(k, md, None) for k, md, _ in pa] + [(("gradA", r, e), "w", e)]))
            comp.append(("rec", ("mid", r, e)))
            comp.append(("acq", [(("gradB", r, e), "w", None)]))
            comp.append(("rel", [(k, md, None) for k, md, _ in pb] + [(("gradB", r, e), "w", e)]))
            comp.append(("rec", ("bwd", r, e)))
            for c, (ev, grad, wire, par) in enumerate((("mid", "gradA", "wireA", "paramsA"), ("bwd", "gradB", "wireB", "paramsB"))):
                comm.append(("wev", (ev, r, e)))
                mine = [((wire, r, s), "w", None) for s in range(n)]           # the encode writes the whole chunk
                comm.append(("acq", [((grad, r, e), "r", e)] + mine))
                comm.append(("rel", [((grad, r, e), "r", None)] + [(k, "w", e) for k, _, _ in mine]))
                for p in ([0] if drop == "signal_server_only" and r != 0 else [] if drop == "signal_server_only" else peers):
                    comm.append(("sig", ("GRAD_READY", p, r), prog(e, c)))
                for p in peers:
                    if not (drop == "grad_ready" and c == 1 and r == 0 and p == peers[-1]):
                        comm.append(("wait", ("GRAD_READY", r, p), prog(e, c)))
                reads = [((wire, p, r), "r", e) for p in range(n)]           # psb_update_kernel over my shard of chunk c
                comm.append(("acq", reads + [((par, r, p), "w", None) for p in range(n)]))
                comm.append(("rel", [(k, md, None) for k, md, _ in reads] + [((par, r, p), "w", e) for p in range(n)]))
            for p in range(n):
                comm.append(("add", ("PARAMS_READY", p), 1))                  # SIGNAL_PARAMS_READY_ADD of the last launch
            comm.append(("rec", ("done", r, e)))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)

    def final(st, mm):
        for p in range(n):
            for c in ("paramsA", "paramsB"):
                for s in range(n):
                    v = st[2][mm.res((c, s, p))]
                    if v != epochs:
                        return f"rank {p} ends on {c} shard {s} version {v}, expected {epochs}"
    m.final_checks.append(final)
    return m


def build_ps_unpipelined(n: int, epochs: int, drop: Optional[str] = None) -> Model:
    """``mode='ps'``, ``pipeline=False``: rank 0 gathers, updates and publishes in ONE launch inside ``step()``.

    ``drop``: ``'params_ready'`` (workers do not wait for the broadcast), ``'grad_ready'`` (the server does not
    wait for the gradients), ``'bwd_event'`` (the last encode does not wait for backward) — each must be caught."""
    m = Model()
    for r in range(n):
        comp, comm = [], []
        for e in range(1, epochs + 1):
            if r != 0 and e > 1 and drop != "params_ready":
                comp.append(("wait", ("PARAMS_READY", r), e - 1))      # psb_wait_kernel on the compute stream
            if r == 0 and e > 1:
                comp.append(("wev", ("done", 0, e - 1)))               # cur.wait_event(done)
            _backward(m, r, e, comp, comm, e - 1, prev_done=(r != 0), pre_encode=[])
            if drop == "bwd_event":
                comm.remove(("wev", ("bwd", r, e)))
            if r != 0:
                comm.append(("sig", ("GRAD_READY", 0, r), e))          # fused into the last encode launch
                comm.append(("rec", ("done", r, e)))
            else:
                if drop != "grad_ready":
                    for p in range(1, n):
                        comm.append(("wait", ("GRAD_READY", 0, p), e))
                reads = [((w, p), "r", e) for p in range(n) for w in ("wireA", "wire")]
                writes = [(("params", p), "w", None) for p in range(n)]
                comm.append(("acq", reads + writes))
                comm.append(("rel", [(k, md, None) for k, md, _ in reads] + [(("params", p), "w", e) for p in range(n)]))
                for p in range(n):
                    comm.append(("sig", ("PARAMS_READY", p), e))
                comm.append(("rec", ("done", 0, e)))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)

    def final(st, mm):
        for p in range(n):
            if st[2][mm.res(("params", p))] != epochs:
                return f"rank {p} ends on parameter version {st[2][mm.res(('params', p))]}, expected {epochs}"
    m.final_checks.append(final)
    return m


def build_allgather(n: int, epochs: int, drop: Optional[str] = None) -> Model:
    """``mode='allgather'`` with the per-chunk pipeline: every rank pulls all ranks' wire tiles of chunk A and updates chunk A
    of its own replica while backward still runs on chunk B, then chunk B (signal_mode 2 on the last chunk).

    ``drop``: ``'consumed'`` (re-encode without waiting for the readers), ``'grad_ready'`` (chunk B's flags),
    ``'grad_ready_a'`` (chunk A's flags)."""
    m = Model()
    prog = lambda e, c: (e - 1) * 2 + c + 1      # noqa: E731
    for r in range(n):
        comp, comm = [], []
        peers = [p for p in range(n) if p != r]
        for e in range(1, epochs + 1):
            if e > 1:
                comp.append(("wev", ("done", r, e - 1)))               # cur.wait_event(done)
            _backward_chunks(m, r, e, comp, prev_done=False)
            for c, (ev, grad, wire, par) in enumerate((("mid", "gradA", "wireA", "paramsA"), ("bwd", "gradB", "wire", "paramsB"))):
                comm.append(("wev", (ev, r, e)))
                if c == 0 and e > 1 and drop != "consumed":
                    comm.extend(("wait", ("CONSUMED", r, p), e - 1) for p in peers)          # _before_first_encode
                comm.append(("acq", [((grad, r, e), "r", e), ((wire, r), "w", None)]))
                comm.append(("rel", [((grad, r, e), "r", None), ((wire, r), "w", e)]))
                for p in peers:
                    comm.append(("sig", ("GRAD_READY", p, r), prog(e, c)))
                if not ((drop == "grad_ready" and c == 1) or (drop == "grad_ready_a" and c == 0)):
                    for p in peers:
                        comm.append(("wait", ("GRAD_READY", r, p), prog(e, c)))
                reads = [((wire, p), "r", e) for p in range(n)]
                comm.append(("acq", reads + [((par, r), "w", None)]))
                comm.append(("rel", [(k, md, None) for k, md, _ in reads] + [((par, r), "w", e)]))
            for p in range(n):
                comm.append(("sig", ("CONSUMED", p, r), e))
            comm.append(("rec", ("done", r, e)))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)
    _chunk_final(m, n, epochs)
    return m


def build_allgather_unpipelined(n: int, epochs: int, drop: Optional[str] = None) -> Model:
    """``mode='allgather'``, ``pipeline=False`` (one chunk): every rank pulls all wire tiles and updates its own replica in one
    launch (signal_mode 2).  This is where the CONSUMED wait is load-bearing: with >= 2 pipelined chunks the in-order comm
    streams already imply it (the checker accepts the pipelined model without it), with one chunk they do not.

    ``drop``: ``'consumed'`` (re-encode without waiting for the readers), ``'grad_ready'``."""
    m = Model()
    for r in range(n):
        comp, comm = [], []
        peers = [p for p in range(n) if p != r]
        for e in range(1, epochs + 1):
            if e > 1:
                comp.append(("wev", ("done", r, e - 1)))               # cur.wait_event(done)
            pre = []
            if e > 1 and drop != "consumed":
                pre = [("wait", ("CONSUMED", r, p), e - 1) for p in peers]
            _backward(m, r, e, comp, comm, e - 1, prev_done=False, pre_encode=pre)
            for p in peers:
                comm.append(("sig", ("GRAD_READY", p, r), e))
            if drop != "grad_ready":
                for p in peers:
                    comm.append(("wait", ("GRAD_READY", r, p), e))
            reads = [((w, p), "r", e) for p in range(n) for w in ("wireA", "wire")]
            comm.append(("acq", reads + [(("params", r), "w", None)]))
            comm.append(("rel", [(k, md, None) for k, md, _ in reads] + [(("params", r), "w", e)]))
            for p in range(n):
                comm.append(("sig", ("CONSUMED", p, r), e))
            comm.append(("rec", ("done", r, e)))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)

    def final(st, mm):
        for p in range(n):
            if st[2][mm.res(("params", p))] != epochs:
                return f"rank {p} ends on parameter version {st[2][mm.res(('params', p))]}, expected {epochs}"
    m.final_checks.append(final)
    return m



def build_async(n: int, epochs: int, quota: int = 1, consistent: bool = False, drop: Optional[str] = None) -> Model:
    """``mode='async'`` (AsySG-InCon, ``/root/reference/README.md:57-81``): workers post gradients and never wait for
    parameters; rank 0 serves ``quota`` gradients per update from ANY source.

    ``drop``: ``'ack'`` (a worker re-encodes without waiting for the server to consume), ``'final_ack'`` (a worker
    posts DONE without waiting for its last gradient to be consumed), ``'recheck'`` (the ``consistent=True`` reader
    does not re-read BEGIN after its copy), ``'server_begin'`` (the server raises BEGIN only after publishing).
    ``'begin'`` (the reader skips the BEGIN == VERSION pre-check) is NOT a bug — the model shows the re-check alone
    is sufficient; the pre-check only saves a wasted copy."""
    m = Model()
    if not consistent:
        for r in range(n):
            m.racy_ok.add(("params", r))                               # inconsistent reads are the point
    else:
        for r in range(n):
            m.racy_ok.add(("stage", r))                                # guarded by the sequence lock instead
    srv = AsyncServer(n, quota, consistent, raise_begin=(drop != "server_begin"))
    m.add("r0.server", srv)
    A, B, C, SNAP = 0, 1, 2, 3
    for r in range(1, n):
        comp, comm = [], []
        for e in range(1, epochs + 1):
            pre = [("wait", ("ACK", r), e - 1)] if (e > 1 and drop != "ack") else []
            _backward(m, r, e, comp, comm, None, prev_done=True, pre_encode=pre)
            comm.append(("sig", ("GRAD_READY", 0, r), e))
            comm.append(("rec", ("done", r, e)))
            if consistent:                                             # DeviceEngine._snapshot on the host thread
                top = len(comp)
                comp.append(("load", A, ("VERSION", r)))
                if drop != "begin":
                    comp.append(("load", B, ("BEGIN", r)))
                    comp.append(("jne", A, B, top))
                skip_ix = len(comp)
                comp.append(None)                                      # patched below: nothing new → skip the copy
                # the snapshot overwrites the live parameters the NEXT forward reads; both are on this stream
                comp.append(("acq", [(("stage", r), "r", None), (("params", r), "w", None)]))
                comp.append(("rel", [(("stage", r), "r", None), (("params", r), "w", None)]))
                if drop != "recheck":
                    comp.append(("load", C, ("BEGIN", r)))
                    comp.append(("jne", C, A, top))
                comp.append(("accept", A))
                comp.append(("mov", SNAP, A))
                comp[skip_ix] = ("jeqc", A, SNAP, len(comp))
        if drop != "final_ack":
            comm.append(("wait", ("ACK", r), epochs))                  # DeviceEngine.close()
        comm.append(("sig", ("GRAD_READY", 0, r), DONE))
        m.add(f"r{r}.compute", comp)
        m.add(f"r{r}.comm", comm)
    def final(st, mm):
        applied = st[0][0][5]
        for r in range(1, n):
            if applied[r] != epochs:
                return f"server applied {applied[r]} gradients of rank {r}, expected {epochs}"
    m.final_checks.append(final)
    return m


def build_stem_pipeline(n: int = 1, epochs: int = 4, drop: Optional[str] = None) -> Model:
    """Intra-CTA pipeline of the fused stem kernel (``csrc/kernels/stem_kernels.cu::psb_stem_fwd_kernel``): the builder
    warpgroup (cp.async patch loads + A-tile builds), the two MMA + epilogue warpgroups (wgmma on their 64 rows of A[buf],
    then staging + BatchNorm column sums from registers) and the TMA unit executing the bulk stores, over ``epochs`` tiles.
    mbarrier phase waits are modelled as counts (``wait(parity)`` at tile ``i`` of a double-buffered resource == "at least
    ``i // 2`` completions", exact because nothing can run two phases ahead).  ``a_empty`` takes one arrival per MMA
    warpgroup (two slots here); named barrier 2 (256 threads) is a pair of sig / wait per warpgroup.  ``n`` is unused.

    ``drop``: ``'a_empty'`` (builders do not wait for the wgmmas that read the A buffer), ``'store_wait'`` (the staging
    tile is rewritten while the bulk store still reads it), ``'staging_bar'`` (no named barrier before the staging writes,
    so warpgroup 1 does not wait for warpgroup 0's ``cp.async.bulk.wait_group.read``).  (The named barriers between the
    four builder warps are below this model's resolution: they are one process here.)"""
    m = Model()
    T = epochs
    builder, store = [], []
    cons = [[], []]
    for i in range(T):
        b = i & 1
        k = i // 2
        # ---- builders (4 warps in lock step through named barrier 1) ----
        if i == 0:
            builder.append(("acq", [(("patch", 0), "w", None)]))                    # load_patch(t0)
        if i + 1 < T:
            builder.append(("acq", [(("patch", b ^ 1), "w", None)]))                  # cp.async of tile i+1
        builder.append(("rel", [(("patch", b), "w", i)]))                            # cp.async.wait_group + barrier
        if drop != "a_empty":
            builder.append(("wait", ("a_empty", b, 0), k))
            builder.append(("wait", ("a_empty", b, 1), k))
        builder.append(("acq", [(("patch", b), "r", i), (("A", b), "w", None)]))     # build_row
        builder.append(("rel", [(("patch", b), "r", None), (("A", b), "w", i)]))
        builder.append(("sig", ("a_full", b), k + 1))
        # ---- MMA + epilogue warpgroups c = 0, 1 ----
        for c in range(2):
            q = cons[c]
            q.append(("wait", ("a_full", b), k + 1))
            q.append(("acq", [(("A", b), "r", i)]))                                  # wgmma + wait_group 0
            q.append(("rel", [(("A", b), "r", None)]))
            q.append(("sig", ("a_empty", b, c), k + 1))
            if c == 0 and drop != "store_wait" and i >= 2:
                q.append(("wait", ("st_done",), i - 1))                              # cp.async.bulk.wait_group.read 1
            if drop != "staging_bar":
                q.append(("sig", ("bar_pre", c), i + 1))                              # named barrier 2
                q.append(("wait", ("bar_pre", 1 - c), i + 1))
            q.append(("acq", [(("O", b, c), "w", None)]))                              # this warpgroup's 64 staged rows
            q.append(("rel", [(("O", b, c), "w", i)]))
            q.append(("sig", ("bar_post", c), i + 1))                                 # named barrier 2
            q.append(("wait", ("bar_post", 1 - c), i + 1))
            if c == 0:
                q.append(("sig", ("st_issued",), i + 1))
            q.append(("acq", [(("O", b, 0), "r", i), (("O", b, 1), "r", i)]))       # BatchNorm column sums (all rows)
            q.append(("rel", [(("O", b, 0), "r", None), (("O", b, 1), "r", None)]))
        # ---- the TMA unit executing the bulk stores, in order ----
        store.append(("wait", ("st_issued",), i + 1))
        store.append(("acq", [(("O", b, 0), "r", i), (("O", b, 1), "r", i)]))
        store.append(("rel", [(("O", b, 0), "r", None), (("O", b, 1), "r", None)]))
        store.append(("sig", ("st_done",), i + 1))
    m.add("builders", builder)
    m.add("mma_epi_0", cons[0])
    m.add("mma_epi_1", cons[1])
    m.add("tma_store", store)
    return m


def build_stem_wgrad_pipeline(n: int = 1, epochs: int = 4, drop: Optional[str] = None) -> Model:
    """Intra-CTA pipeline of ``psb_stem_wgrad_kernel``: the builder warpgroup fills A[buf] and its thread 0 issues the gy
    TMA load into G[buf] after the ``empty`` wait (the TMA unit is a process of its own); the MMA warpgroup accumulates every
    tile into register-resident accumulators, frees the pair after ``wgmma.wait_group 0`` and finally writes the CTA's
    partial from its registers (program order, no barrier).  ``drop``: ``'empty'`` (the builders do not wait for the wgmmas
    before refilling A and G), ``'g_full'`` (the MMA warpgroup does not wait for the gy bytes)."""
    m = Model()
    T = epochs
    builder, gtma, mma = [], [], []
    for i in range(T):
        b, k = i & 1, i // 2
        if i == 0:
            builder.append(("acq", [(("patch", 0), "w", None)]))
        if i + 1 < T:
            builder.append(("acq", [(("patch", b ^ 1), "w", None)]))
        builder.append(("rel", [(("patch", b), "w", i)]))
        if drop != "empty":
            builder.append(("wait", ("empty", b), k))
        builder.append(("sig", ("g_issue", b), k + 1))                               # thread 0: expect_tx + TMA load
        builder.append(("acq", [(("patch", b), "r", i), (("A", b), "w", None)]))
        builder.append(("rel", [(("patch", b), "r", None), (("A", b), "w", i)]))
        builder.append(("sig", ("a_full", b), k + 1))
        gtma.append(("wait", ("g_issue", b), k + 1))
        gtma.append(("acq", [(("G", b), "w", None)]))                                 # cp.async.bulk.tensor load of gy
        gtma.append(("rel", [(("G", b), "w", i)]))
        gtma.append(("sig", ("g_full", b), k + 1))
        mma.append(("wait", ("a_full", b), k + 1))
        if drop != "g_full":
            mma.append(("wait", ("g_full", b), k + 1))
        mma.append(("acq", [(("A", b), "r", i), (("G", b), "r", i)]))
        mma.append(("rel", [(("A", b), "r", None), (("G", b), "r", None)]))
        mma.append(("sig", ("empty", b), k + 1))
    m.add("builders", builder)
    m.add("gy_tma", gtma)
    m.add("mma", mma)
    return m


MODES = {"ps": build_ps, "ps_unpipelined": build_ps_unpipelined, "allgather": build_allgather,
         "allgather_unpipelined": build_allgather_unpipelined, "async": build_async, "stem_pipeline": build_stem_pipeline,
         "stem_wgrad_pipeline": build_stem_wgrad_pipeline, "ps_accumulate": build_ps_accumulate, "sharded": build_sharded}


def check(mode: str, n: int, epochs: int, max_states: int = 2_000_000, **kw) -> Result:
    """Exhaustively explore ``mode`` for ``n`` ranks × ``epochs`` steps; raises :class:`Violation` on a failure."""
    return _Explorer(MODES[mode](n, epochs, **kw), max_states).run()


def main(argv: Optional[Sequence[str]] = None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--mode", choices=sorted(MODES), default="ps",
                    help="engine protocols (ps / allgather / async) or the kernel pipelines (stem_*; --epochs = tiles)")
    ap.add_argument("--ranks", type=int, default=3)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--quota", type=int, default=1)
    ap.add_argument("--consistent", action="store_true")
    ap.add_argument("--drop", default=None, help="delete one wait (mutation): see the build_* docstrings")
    a = ap.parse_args(argv)
    kw = {"drop": a.drop}
    if a.mode == "async":
        kw.update(quota=a.quota, consistent=a.consistent)
    try:
        res = check(a.mode, a.ranks, a.epochs, **kw)
    except Violation as v:
        print(f"VIOLATION {v}")
        for line in v.trace[-25:]:
            print("   ", line)
        return 1
    print(f"ok: mode={a.mode} ranks={a.ranks} epochs={a.epochs} states={res.states} "
          f"transitions={res.transitions} final_states={res.finals}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
