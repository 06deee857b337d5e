#!/usr/bin/env python
"""Host transport micro-benchmark (CPU only): ping-pong latency and one-way bandwidth between two ranks, for the native
shm transport and the gloo fallback.  ``python bench/transport_pingpong.py`` → JSON lines on stdout and in
``bench_out/transport_pingpong.jsonl``."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def body(rank, size, transport, out_path):
    os.environ["PSB200_TRANSPORT"] = transport
    import torch
    torch.set_num_threads(1)
    import pytorch_ps_mpi_b200 as ps
    from pytorch_ps_mpi_b200.parallel.transport import get_transport
    ps.runtime.init()
    tr = get_transport()
    res = []
    for nbytes in (8, 1 << 10, 64 << 10, 1 << 20, 16 << 20, 64 << 20):
        buf = bytearray(nbytes)
        reps = 2000 if nbytes <= (64 << 10) else (200 if nbytes <= (1 << 20) else 20)
        tr.barrier()
        # ping-pong
        t0 = time.perf_counter()
        for _ in range(reps):
            if rank == 0:
                tr.isend(1, buf, tag=7).Wait()
                tr.irecv(1, tag=8).Wait()
            else:
                tr.irecv(0, tag=7).Wait()
                tr.isend(0, buf, tag=8).Wait()
        rtt = (time.perf_counter() - t0) / reps
        tr.barrier()
        # one-way stream: rank 0 sends, rank 1 receives, one ack at the end
        t0 = time.perf_counter()
        if rank == 0:
            reqs = [tr.isend(1, buf, tag=9) for _ in range(reps)]
            for r in reqs:
                r.Wait()
            tr.irecv(1, tag=10).Wait()
        else:
            for _ in range(reps):
                tr.irecv(0, tag=9).Wait()
            tr.isend(0, b"k", tag=10).Wait()
        dt = time.perf_counter() - t0
        if rank == 0:
            res.append({"transport": transport, "bytes": nbytes, "half_rtt_us": rtt / 2 * 1e6,
                        "stream_GBps": nbytes * reps / dt / 1e9})
    tr.barrier()
    if rank == 0:
        with open(out_path, "a") as f:
            for r in res:
                f.write(json.dumps(r) + "\n")


def main():
    from pytorch_ps_mpi_b200.launch import spawn
    out = os.path.join(ROOT, "bench_out", "transport_pingpong.jsonl")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    open(out, "w").close()
    for transport in ("shm", "gloo"):
        spawn(body, 2, args=(transport, out), timeout=600)
    print(open(out).read(), end="")


if __name__ == "__main__":
    main()
