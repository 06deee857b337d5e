#!/usr/bin/env python
"""A few rounds of the fused PS round (encode → flag → psb_update_kernel → PARAMS_READY) on a synthetic parameter vector,
for profiling ONE rank of a multi-GPU job under ncu with a handful of metrics (NVLink rx/tx bytes, DRAM bytes, duration):

    python -m torch.distributed.run --nproc-per-node 8 bench/update_probe.py --mb 64 --reduce auto

(rank 0 runs under ``ncu --metrics …``, the other ranks run plain; epoch flags are monotone and the update is a pure
function of the restored state, so ncu's kernel replay on rank 0 is safe — replays see the peers' flags already raised.)
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pytorch_ps_mpi_b200 as ps   # noqa: E402
from bandwidth_sweep import code_of   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=float, default=64)
    ap.add_argument("--piece-mb", type=float, default=8)
    ap.add_argument("--reduce", default="auto")
    ap.add_argument("--code", default="identity")
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    w = ps.runtime.init()
    dev = w.device
    n = int(a.mb * (1 << 20)) // 2
    piece = int(a.piece_mb * (1 << 20)) // 2
    shapes = [piece] * (n // piece) + ([n % piece] if n % piece else [])
    params = [torch.nn.Parameter(torch.zeros(m, device=dev, dtype=torch.bfloat16)) for m in shapes]
    grads = [torch.randn(m, device=dev).bfloat16() for m in shapes]
    code = code_of(a.code)
    opt = ps.SGD([(f"v{i}", p) for i, p in enumerate(params)], params, lr=1e-3, momentum=0.9, code=code, mode="ps",
                 engine="device", reduce=a.reduce)
    eng = opt._engine
    order = [(s.param, s.name, next(i for i, q in enumerate(params) if q is s.param)) for s in eng.layout.slots]
    for _ in range(a.rounds):
        for p, name, i in order:
            eng.on_grad(grads[i], name, p)
        opt.step()
        torch.cuda.synchronize(dev)
        w.barrier()
    eng.check()
    if w.rank == 0:
        print("probe ok", {"mb": a.mb, "chunks": eng.nchunks, "reduce": eng.reduce, "bcast": eng.bcast, "wire_bytes": eng.bpt * eng.layout.ntiles})
    opt.close()
    ps.runtime.shutdown()


if __name__ == "__main__":
    main()
