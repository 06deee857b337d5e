#!/usr/bin/env python
"""Gradient accumulation (``MPI_PS.no_sync()``) on ONE GPU.  One JSON line per measurement:

* ``psb_accumulate_kernel`` (carry += gradient, fp32) over a whole arena of bf16 gradients, timed with CUDA events over many
  back-to-back calls.  HBM bytes from shapes: 2 (bf16 gradient read) + 4 + 4 (fp32 carry read and written) per arena element,
  tile padding included, against the H100 SXM's 3.35 TB/s HBM3 (data sheet).
* ResNet-18, bf16, batch 256 per step on the device engine: one backward of 256 against four backwards of 64 (three inside
  ``no_sync()``), milliseconds per step between CUDA events after a warm-up; and the same forwards and backwards of a plain
  model without the engine (``engine: false``), which separates the cost of the accumulation from that of small batches.
  cuDNN is set up as ``bench.py`` sets it (deterministic, no autotuning).
* The card's name and power limit, read in the same run.

    python bench/accumulate_timing.py [--arenas resnet18,bert_base] [--steps 20] [--warmup 5]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_ps_mpi_b200 as ps   # noqa: E402
from pytorch_ps_mpi_b200 import models, runtime   # noqa: E402
from pytorch_ps_mpi_b200.ops import ext   # noqa: E402
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout   # noqa: E402

HBM_TBS = 3.35
ARENAS = {"resnet18": 11_689_512, "bert_base": 109_482_240}    # parameters (torchvision ResNet-18, BERT-base uncased)


def kernel_timing(arena, iters, piece_mb, dev):
    m = ext.cuda()
    n = ARENAS[arena]
    piece = int(piece_mb * (1 << 20)) // 2
    shapes = [piece] * (n // piece) + ([n % piece] if n % piece else [])
    params = [torch.nn.Parameter(torch.zeros(s, device=dev, dtype=torch.bfloat16)) for s in shapes]
    grads = [torch.randn(s, device=dev).bfloat16() for s in shapes]
    L = FlatLayout([{"params": params}], {id(p): f"p{i}" for i, p in enumerate(params)})
    tiles = L.tile_table_fast().to(dev)
    carry = torch.zeros(L.numel_padded, dtype=torch.float32, device=dev)
    slots = [L.by_id[id(p)] for p in params]
    args = ([s.first_tile for s in slots], [s.ntiles for s in slots], [s.index for s in slots], tiles.data_ptr(),
            carry.data_ptr())
    for _ in range(3):
        m.accumulate(grads, *args)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        m.accumulate(grads, *args)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    nbytes = 10 * L.numel_padded
    return {"what": "accumulate_kernel", "arena": arena, "params": n, "launches_per_call": (len(grads) + 63) // 64,
            "us": round(us, 2), "hbm_bytes": nbytes, "achieved_TBps": round(nbytes / us / 1e6, 3),
            "share_of_hbm_peak": round(nbytes / us / 1e6 / HBM_TBS, 3)}


def step_timing(micro, batch, steps, warmup, dev, engine=True):
    torch.manual_seed(0)
    model = models.resnet18(num_classes=1000).to(dev).to(memory_format=torch.channels_last).bfloat16()
    named = list(model.named_parameters())
    if engine:
        opt = ps.SGD(named, [p for _, p in named], lr=0.01, momentum=0.9, code=ps.Identity(), engine="device")
    else:
        opt = None
    mb = batch // micro
    g = torch.Generator(device=dev).manual_seed(1)
    xs = [torch.randn(mb, 3, 224, 224, device=dev, generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
          for _ in range(micro)]
    ys = [torch.randint(0, 1000, (mb,), device=dev, generator=g) for _ in range(micro)]

    def one_step():
        model.zero_grad(set_to_none=True)
        for i in range(micro):
            with opt.no_sync() if opt is not None and i < micro - 1 else contextlib.nullcontext():
                torch.nn.functional.cross_entropy(model(xs[i]).float(), ys[i]).backward()
        return opt.step()[1] if opt is not None else {"micro_batches": micro}

    for _ in range(warmup):
        one_step()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for s in range(steps):
        data = one_step()
        ev[s + 1].record()
    torch.cuda.synchronize()
    per = sorted(ev[s].elapsed_time(ev[s + 1]) for s in range(steps))
    if opt is not None:
        opt._engine.check()
        opt.close()
    assert data["micro_batches"] == micro
    return {"what": "resnet18_step", "engine": engine, "batch": batch, "micro_batches": micro, "micro_batch": mb, "steps": steps,
            "ms_per_step_median": round(per[len(per) // 2], 3), "ms_per_step_min": round(per[0], 3),
            "ms_per_step_max": round(per[-1], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arenas", default="resnet18,bert_base")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--piece-mb", type=float, default=8.0, help="largest gradient tensor")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--micro", default="1,4", help="micro-batches per step to compare")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("accumulate_timing needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    for arena in a.arenas.split(","):
        print(json.dumps(kernel_timing(arena, a.iters, a.piece_mb, dev)), flush=True)
    runtime.init()
    for micro in (int(x) for x in a.micro.split(",")):
        for engine in (True, False):
            print(json.dumps(step_timing(micro, a.batch, a.steps, a.warmup, dev, engine)), flush=True)
    runtime.shutdown()


if __name__ == "__main__":
    main()
