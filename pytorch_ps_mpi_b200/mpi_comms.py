"""L1/L2 communication façade with the reference's signatures (generic-object host path).

Everything ``/root/reference/mpi_comms.py`` exports is here under the same name and call
shape — ``to_np``, ``to_torch``, ``compress``, ``decompress``, ``igather``/``irecv`` (worker→PS
gather, ``mpi_comms.py:60-117``), ``ibroadcast``/``irecv1`` (PS→worker broadcast,
``mpi_comms.py:120-133``), ``class Iallgather`` (``mpi_comms.py:144-174``), ``trim_msg``,
``print_summary``, ``format_for_send``, ``to_mpi``/``to_mpi_v`` and the module globals ``comm``,
``rank``, ``size``, ``max_bytes`` — but re-designed:

* the wire format is :mod:`pytorch_ps_mpi_b200.serialization` (pickled skeleton + raw tensor
  bytes + explicit length header) instead of pickle+blosc+32-byte sentinel in 10x slots,
* the transport is :mod:`pytorch_ps_mpi_b200.parallel.transport` (native shm rings / gloo)
  instead of mpi4py, so only the root allocates receive space and only as much as arrives,
* non-root ``irecv`` completes its request (the reference leaked it, ``mpi_comms.py:109-117``),
* ``to_torch`` preserves dtypes (the reference cast everything to float32, ``mpi_comms.py:48``),
* ``Iallgather.prepare`` exchanges all P sizes in ONE message, not P collectives
  (``mpi_comms.py:150-158``).

This path serves arbitrary Python objects and user codings.  Dense tensors on the GPU never come
through here: they use the symmetric-memory kernels in :mod:`pytorch_ps_mpi_b200.parallel`.
"""
from __future__ import annotations

import functools
import time
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import runtime, serialization
from .parallel import transport as _tp
from .serialization import compress, decompress  # noqa: F401  (re-exported, reference names)

__all__ = [
    "comm", "to_np", "to_torch", "compress", "decompress", "igather", "irecv", "ibroadcast",
    "irecv1", "Iallgather", "trim_msg", "print_summary", "format_for_send", "to_mpi", "to_mpi_v",
    "max_bytes", "BYTE", "ANY_SOURCE", "isend_obj", "irecv_obj", "barrier",
]

comm = runtime.COMM_WORLD          # ``MPI.COMM_WORLD`` stand-in (mpi_comms.py:11)
BYTE = "BYTE"                      # ``MPI.BYTE`` stand-in for to_mpi / to_mpi_v
ANY_SOURCE = _tp.ANY_SOURCE

#: per-``name`` bytes of the largest gathered message seen (the reference's sticky slot size,
#: ``mpi_comms.py:15,82-83``; informational here — nothing is over-allocated from it)
max_bytes: Dict[Any, int] = {}

_SENTINEL = b"\x29" * 32


def __getattr__(name):   # module-level ``rank`` / ``size`` resolve lazily (mpi_comms.py:12-13)
    if name == "rank":
        return runtime.world().rank
    if name == "size":
        return runtime.world().size
    raise AttributeError(name)


# ---------------------------------------------------------------------------------------
# host staging helpers (C9 / C10)
# ---------------------------------------------------------------------------------------
_NP_UNSUPPORTED = (torch.bfloat16, torch.float8_e4m3fn, torch.float8_e5m2)


def to_np(d):
    """Recursive tensor→ndarray staging (``mpi_comms.py:32-43``).  bf16/fp8 upcast to float32."""
    if isinstance(d, torch.Tensor):
        t = d.detach()
        if t.is_cuda:
            t = t.cpu()
        if t.dtype in _NP_UNSUPPORTED:
            t = t.float()
        return t.numpy()
    if isinstance(d, dict):
        return {k: to_np(v) for k, v in d.items()}
    if isinstance(d, list):
        return list(map(to_np, d))
    if isinstance(d, tuple):
        return tuple(map(to_np, d))
    if isinstance(d, map):
        return map(to_np, d)
    return d


def to_torch(d, cuda: bool = False):
    """Recursive ndarray→tensor (dtype preserving) with optional async H2D (``mpi_comms.py:46-58``)."""
    if isinstance(d, np.ndarray):
        d = torch.from_numpy(d) if d.flags.writeable else torch.from_numpy(d.copy())
    if isinstance(d, torch.Tensor):
        if cuda and torch.cuda.is_available() and not d.is_cuda:
            d = d.cuda(non_blocking=True)
        return d
    if isinstance(d, dict):
        return {k: to_torch(v, cuda=cuda) for k, v in d.items()}
    if isinstance(d, list):
        return list(map(functools.partial(to_torch, cuda=cuda), d))
    if isinstance(d, tuple):
        return tuple(map(functools.partial(to_torch, cuda=cuda), d))
    if isinstance(d, map):
        return map(functools.partial(to_torch, cuda=cuda), d)
    return d


def trim_msg(msg):
    """Return ``msg`` up to the 32-byte ``0x29`` sentinel (``mpi_comms.py:96-104``).

    Kept for API parity; framed messages carry a length header and never need it.
    """
    i = bytes(msg).find(_SENTINEL) if not isinstance(msg, (bytes, bytearray)) else msg.find(_SENTINEL)
    if i == -1:
        raise Exception("trim_msg error; end of msg not found")
    return msg[:i]


def print_summary(flat_dict):
    """Debug pretty-printer: shapes for tensors/arrays, values otherwise (``mpi_comms.py:176-184``)."""
    string = "    {"
    for k, v in flat_dict.items():
        if isinstance(v, (torch.Tensor, np.ndarray)):
            string += f"{k}: {tuple(v.shape)}, "
        else:
            string += f"{k}: {v}, "
    string += "}"
    print(string)
    return string


def format_for_send(obj, level: int = 0):
    """Serialise + frame an object → ``(packaged, {'msg_bytes', 'packaged_bytes'})`` (``mpi_comms.py:186-193``)."""
    packaged, raw_len = serialization.dumps_framed(obj, level=level)
    return packaged, {"msg_bytes": raw_len, "packaged_bytes": len(packaged)}


def _unpack(msg, cuda: bool = False, numpy: bool = False):
    obj = serialization.loads(serialization.unframe_view(msg))      # tensors are views into `msg` (kept alive by them)
    return to_np(obj) if numpy else to_torch(obj, cuda=cuda)


def to_mpi_v(v, counts, dtype=BYTE):
    displacements = [sum(counts[:i]) for i in range(len(counts))]
    return (v, (counts, displacements), dtype)


def to_mpi(v, dtype=BYTE):
    return (v, dtype)


# ---------------------------------------------------------------------------------------
# requests / sequencing
# ---------------------------------------------------------------------------------------
_seq = 0
_TAG_P2P = 1 << 28


def _next_tag() -> int:
    """Every collective takes the next tag on every rank (same call order everywhere, as in MPI)."""
    global _seq
    _seq = (_seq + 1) % (1 << 27)
    return _seq


class _Multi(_tp.Request):
    """A request that completes when all of its parts do."""

    def __init__(self, parts: Sequence[_tp.Request]):
        self.parts = list(parts)
        self._results: Optional[list] = None

    def Wait(self, timeout=None):
        if self._results is None:
            self._results = [p.Wait(timeout) for p in self.parts]
        return self._results

    def Test(self):
        return all(p.Test() for p in self.parts)

    wait, test = Wait, Test


def barrier():
    _tp.get_transport().barrier()


# ---------------------------------------------------------------------------------------
# worker → PS gather (C11a-c)
# ---------------------------------------------------------------------------------------
class _GatherRecv:
    """Receive-side handle of an ``igather`` (the reference's pre-sized ``recv`` bytearray)."""

    def __init__(self, root: int, local, reqs):
        self.root, self.local, self.reqs = root, local, reqs


def igather(obj, name="", root: int = 0, level: int = 0):
    """Post a gather of a Python object to ``root`` (``mpi_comms.py:60-93``).

    Returns ``(recv, req, timings)`` with the reference's timing keys.
    """
    tr = _tp.get_transport()
    t = [time.time()]
    if level <= 0:
        # level 0: serialise + frame in ONE pass over one buffer — there is no separate compression stage to time, so
        # compress_time is reported as exactly 0.0 (the reference's level-0 blosc pass is a memcpy, mpi_comms.py:18-26)
        send, _ = serialization.dumps_framed(obj, level=0)
        t += [time.time()]
        t += [t[-1]]
    else:
        raw = serialization.dumps(obj)                          # pickle_time: the serialisation alone
        t += [time.time()]
        send = serialization.frame(raw, level=level)            # compress_time: byte-shuffle + deflate
        t += [time.time()]
    max_bytes[name] = max(max_bytes.get(name, 0), len(send))
    tag = _next_tag()
    t += [time.time()]
    if tr.rank == root:
        parts = [tr.irecv(src=r, tag=tag) for r in range(tr.size) if r != root]
        recv = _GatherRecv(root, send, parts)
        req = _Multi(parts)
    else:
        recv = _GatherRecv(root, None, [])
        req = tr.isend(root, send, tag=tag)
        recv.keep = send
    t += [time.time()]
    return recv, req, {"pickle_time": t[1] - t[0], "compress_time": t[2] - t[1],
                       "alloc_time": t[3] - t[2], "igather_time": t[4] - t[3],
                       "alloc_bytes": len(send) if tr.rank != root else 0}


def irecv(recv: _GatherRecv, req, name="", cuda: bool = False):
    """Complete a gather: list of every rank's object at the root, ``None`` elsewhere (``mpi_comms.py:107-117``)."""
    tr = _tp.get_transport()
    got = req.Wait()
    if tr.rank != recv.root:
        return None
    msgs: List[Any] = []
    it = iter(got)
    for r in range(tr.size):
        msgs.append(recv.local if r == recv.root else next(it))
    return [_unpack(m, cuda=cuda) for m in msgs]


# ---------------------------------------------------------------------------------------
# PS → worker broadcast (C11d-e)
# ---------------------------------------------------------------------------------------
def ibroadcast(obj, root: int = 0, level: int = 0):
    """Post a broadcast of ``root``'s object (``mpi_comms.py:127-133``).  Returns ``(send, req)``."""
    tr = _tp.get_transport()
    tag = _next_tag()
    if tr.rank == root:
        send, _ = serialization.dumps_framed(obj, level=level)
        req = _Multi([tr.isend(r, send, tag=tag) for r in range(tr.size) if r != root])
        return send, req
    req = tr.irecv(src=root, tag=tag)
    return None, req


def irecv1(recv, req, cuda: bool = False):
    """Complete a broadcast and return the root's object on every rank (``mpi_comms.py:120-124``)."""
    got = req.Wait()
    msg = recv if recv is not None else got
    return _unpack(msg, cuda=cuda)


# ---------------------------------------------------------------------------------------
# variable-size all-gather (C12)
# ---------------------------------------------------------------------------------------
class _CountsReq(_tp.Request):
    """Shared completion of the one-message size exchange behind ``Iallgather.prepare``."""

    def __init__(self, owner: "_SizeExchange", i: int, counts: np.ndarray):
        self.owner, self.i, self.counts = owner, i, counts

    def Wait(self, timeout=None):
        self.owner.complete()
        return self.counts

    def Test(self):
        return self.owner.done or self.owner.req.Test()

    wait, test = Wait, Test


class _SizeExchange:
    def __init__(self, tr, my_counts: List[int]):
        self.tr, self.done = tr, False
        self.mine = np.asarray(my_counts, dtype=np.int64)
        self.table = np.zeros((len(my_counts), tr.size), dtype=np.int64)
        self.table[:, tr.rank] = self.mine
        tag = _next_tag()
        self._sends = [tr.isend(r, self.mine.tobytes(), tag=tag) for r in range(tr.size) if r != tr.rank]
        self._srcs = [r for r in range(tr.size) if r != tr.rank]
        self.req = _Multi([tr.irecv(src=r, tag=tag) for r in self._srcs])

    def complete(self):
        if self.done:
            return
        for r, buf in zip(self._srcs, self.req.Wait()):
            self.table[:, r] = np.frombuffer(bytes(buf), dtype=np.int64)
        for s in self._sends:
            s.Wait()
        self.done = True


class Iallgather:
    """Variable-size all-gather of byte blobs (``mpi_comms.py:144-174``)."""

    def __init__(self):
        w = runtime.world()
        self.comm = comm
        self.rank = w.rank
        self.size = w.size

    def _get_counts(self, rank_size):
        return self.prepare([rank_size])[0]

    def prepare(self, counts: Sequence[int]):
        """Exchange message lengths; returns ``[(req, counts_i)]`` — ``counts_i`` valid after ``req.Wait()``."""
        tr = _tp.get_transport()
        ex = _SizeExchange(tr, list(counts))
        return [(_CountsReq(ex, i, ex.table[i]), ex.table[i]) for i in range(len(counts))]

    def send(self, send, counts):
        tr = _tp.get_transport()
        tag = _next_tag()
        peers = [r for r in range(tr.size) if r != tr.rank]
        sends = [tr.isend(r, send, tag=tag) for r in peers]
        recvs = [tr.irecv(src=r, tag=tag) for r in peers]
        handle = {"local": send, "peers": peers, "sends": sends}
        return handle, _Multi(recvs), counts

    def recv(self, recv, req, counts, cuda: bool = False):
        tr = _tp.get_transport()
        got = req.Wait()
        by_rank: List[Any] = [None] * tr.size
        by_rank[tr.rank] = recv["local"]
        for r, m in zip(recv["peers"], got):
            by_rank[r] = m
        for s in recv["sends"]:
            s.Wait()
        if counts is not None and len(counts) == tr.size:
            for r, m in enumerate(by_rank):
                if int(counts[r]) not in (0, len(m)):
                    raise ValueError(f"Iallgather.recv: rank {r} announced {int(counts[r])} bytes, got {len(m)}")
        return [_unpack(m, numpy=True) for m in by_rank]


# ---------------------------------------------------------------------------------------
# point-to-point object messaging (async AsySG-InCon spec, README.md:65-76)
# ---------------------------------------------------------------------------------------
def isend_obj(obj, dst: int, tag: int = 0, level: int = 0):
    tr = _tp.get_transport()
    send, _ = serialization.dumps_framed(obj, level=level)
    req = tr.isend(dst, send, tag=_TAG_P2P + tag)
    req._keep = send
    return req


class _ObjRecv(_tp.Request):
    def __init__(self, inner, cuda):
        self.inner, self.cuda, self.source = inner, cuda, -1

    def Wait(self, timeout=None):
        msg = self.inner.Wait(timeout)
        self.source = self.inner.source
        return _unpack(msg, cuda=self.cuda)

    def Test(self):
        return self.inner.Test()

    wait, test = Wait, Test


def irecv_obj(src: int = ANY_SOURCE, tag: int = 0, cuda: bool = False):
    """Non-blocking receive of a Python object, ``src=ANY_SOURCE`` allowed (README.md:68)."""
    tr = _tp.get_transport()
    return _ObjRecv(tr.irecv(src=src, tag=_TAG_P2P + tag), cuda)
