#!/usr/bin/env python
"""Time the gradient encode of one step on ONE GPU: ``psb_encode_kernel`` over a whole arena of bf16 gradients, per coding,
with CUDA events around many back-to-back calls.  ``Scale`` includes its abs-max pre-pass (two launches per bucket); block-wise
QSGD and block-wise sign are one launch per bucket; error-feedback sign also reads and rewrites the fp32 residual arena.
``accumulate`` times ``psb_accumulate_kernel`` (``no_sync()``: carry += gradient) on the same arena: it moves the same HBM bytes
as the error-feedback sign encode, less the 272-byte wire tiles, so it is that encode's natural bound.  Repeat codes in
``--codes`` to alternate them within one run.  Achieved bytes/s = bytes moved / time, against the H100 SXM's 3.35 TB/s HBM3
(data sheet).  One JSON line per (arena, coding).

    python bench/encode_timing.py --codes qsgd:7,qsgd:127,scale:int8 --arenas resnet18,bert_base
    python bench/encode_timing.py --codes sign,accumulate,sign,accumulate,sign:noef
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bandwidth_sweep import code_of   # noqa: E402
from pytorch_ps_mpi_b200.codings import KIND_SCALED, KIND_SIGN   # noqa: E402
from pytorch_ps_mpi_b200.ops import ext   # noqa: E402
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout   # noqa: E402

HBM_TBS = 3.35
ARENAS = {"resnet18": 11_689_512, "bert_base": 109_482_240}    # parameters (torchvision ResNet-18, BERT-base uncased)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--codes", default="qsgd:7,qsgd:127,scale:int8")
    ap.add_argument("--arenas", default="resnet18,bert_base")
    ap.add_argument("--piece-mb", type=float, default=8.0, help="largest gradient tensor")
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    m = ext.cuda()
    dev = torch.device("cuda", 0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    for arena in a.arenas.split(","):
        n = ARENAS[arena]
        piece = int(a.piece_mb * (1 << 20)) // 2
        shapes = [piece] * (n // piece) + ([n % piece] if n % piece else [])
        params = [torch.nn.Parameter(torch.zeros(s, device=dev, dtype=torch.bfloat16)) for s in shapes]
        grads = [torch.randn(s, device=dev).bfloat16() for s in shapes]
        L = FlatLayout([{"params": params}], {id(p): f"p{i}" for i, p in enumerate(params)})
        tiles = L.tile_table_fast().to(dev)
        order = [(L.by_id[id(p)], g) for p, g in zip(params, grads)]
        carry = torch.zeros(L.numel_padded, dtype=torch.float32, device=dev)
        mask = torch.full((L.ntiles * 64,), -1, dtype=torch.int32, device=dev)   # every element real (no custom placement)
        for c in a.codes.split(","):
            if c == "accumulate":
                def acc(step):
                    m.accumulate([g for _, g in order], [s.first_tile for s, _ in order], [s.ntiles for s, _ in order],
                                 [s.index for s, _ in order], tiles.data_ptr(), carry.data_ptr())
                report(arena, n, c, time_it(acc, a.iters), n * 2 + 2 * 4 * L.numel_padded, 0, 1, card)
                continue
            spec = code_of(c).device_spec()
            wire = spec.resolved_wire(torch.bfloat16)
            bpt = spec.bytes_per_tile(torch.bfloat16)
            arena_w = torch.zeros(L.ntiles * bpt, dtype=torch.uint8, device=dev)
            scales = torch.zeros(L.nparams, dtype=torch.float32, device=dev)
            amax = torch.zeros(L.nparams, dtype=torch.int32, device=dev)
            kw = dict(seed=spec.seed, step=0, rank=0, levels=spec.levels) if spec.levels else {}
            if spec.kind == KIND_SIGN:
                kw["real_mask"] = mask.data_ptr()
            res = carry.data_ptr() if spec.error_feedback else 0

            def enc(step):
                if spec.kind == KIND_SCALED:
                    amax.zero_()
                if "step" in kw:
                    kw["step"] = step
                m.encode(spec.kind, wire, [g for _, g in order], [s.first_tile for s, _ in order], [s.ntiles for s, _ in order],
                         [s.index for s, _ in order], tiles.data_ptr(), arena_w.data_ptr(), scales.data_ptr(), amax.data_ptr(), res,
                         bpt, spec.tile_capacity(), 1.0, **kw)

            read = n * 2 * (2 if spec.kind == KIND_SCALED else 1)        # Scale reads the gradient twice (abs-max, encode)
            read += 4 * L.numel_padded if res else 0                     # the residual, read and rewritten
            written = L.ntiles * bpt + (4 * L.numel_padded if res else 0)
            report(arena, n, c, time_it(enc, a.iters), read, written, 2 if spec.kind == KIND_SCALED else 1, card)


def time_it(fn, iters):
    """µs per call: CUDA events around ``iters`` back-to-back calls after 5 warm-up calls."""
    for i in range(5):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(iters):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3


def report(arena, n, code, us, read, written, launches, card):
    gbs = (read + written) / us / 1e3
    print(json.dumps({"arena": arena, "params": n, "code": code, "us": round(us, 1), "bytes_read": read,
                      "bytes_written": written, "GBs": round(gbs, 1), "hbm_fraction": round(gbs / (HBM_TBS * 1e3), 3),
                      "launches_per_bucket": launches, "card": card}), flush=True)


if __name__ == "__main__":
    main()
