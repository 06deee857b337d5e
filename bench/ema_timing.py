#!/usr/bin/env python
"""The weight average (``ema_decay``) on ONE GPU.  One JSON line per measurement:

* ``psb_ema_kernel`` over a whole arena (fp32 master and fp32 average: 4 + 4 + 4 bytes per arena element, tile padding
  included), alternated with ``psb_accumulate_kernel`` (bf16 gradient + fp32 carry: 2 + 4 + 4 bytes), which moves comparable
  bytes; CUDA events over many back-to-back calls; achieved bytes/s against the H100 SXM's 3.35 TB/s HBM3 (data sheet).
* ResNet-18, bf16, PS-SGD at N = 1 on the device engine: the average off, on (``ema_decay``), and the user-side workaround
  (``ensure_params()`` + ``AveragedModel.update_parameters`` on the compute stream after every step), alternated in rounds;
  milliseconds per step between CUDA events after a warm-up.  cuDNN is set up as ``bench.py`` sets it.
* The card's name and power limit, read in the same run.

    python bench/ema_timing.py [--arenas resnet18,bert_base] [--rounds 3] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

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
    master = torch.randn(L.numel_padded, dtype=torch.float32, device=dev)
    ema = torch.zeros(L.numel_padded, dtype=torch.float32, device=dev)
    slots = [L.by_id[id(p)] for p in params]
    acc_args = ([s.first_tile for s in slots], [s.ntiles for s in slots], [s.index for s in slots], tiles.data_ptr(),
                carry.data_ptr())

    def run_ema(first=False):
        m.ema(master.data_ptr(), 0, 1, ema.data_ptr(), L.ntiles, 0, L.ntiles, 0, 1.0 - 0.999, first)

    def run_acc():
        m.accumulate(grads, *acc_args)

    run_ema(True)
    for _ in range(3):
        run_ema()
        run_acc()
    torch.cuda.synchronize()
    out = []
    for what, fn, bpe in (("ema_kernel", run_ema, 12), ("accumulate_kernel", run_acc, 10)) * 3:   # alternated
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        nbytes = bpe * L.numel_padded
        out.append({"what": what, "arena": arena, "params": n, "us": round(us, 2), "hbm_bytes": nbytes,
                    "achieved_TBps": round(nbytes / us / 1e6, 3), "share_of_hbm_peak": round(nbytes / us / 1e6 / HBM_TBS, 3)})
    return out


def step_timing(variant, batch, steps, warmup, dev):
    torch.manual_seed(0)
    model = models.resnet18(num_classes=1000).to(dev).to(memory_format=torch.channels_last).bfloat16()
    named = list(model.named_parameters())
    opt = ps.SGD(named, [p for _, p in named], lr=0.01, momentum=0.9, code=ps.Identity(), engine="device",
                 ema_decay=0.999 if variant == "ema_decay" else None)
    avg = AveragedModel(model, multi_avg_fn=get_ema_multi_avg_fn(0.999), use_buffers=False) if variant == "user_side" else None
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(batch, 3, 224, 224, device=dev, generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device=dev, generator=g)

    def one_step():
        model.zero_grad(set_to_none=True)
        torch.nn.functional.cross_entropy(model(x).float(), y).backward()
        opt.step()
        if avg is not None:
            opt._engine.ensure_params()
            avg.update_parameters(model)

    for _ in range(warmup):
        one_step()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    ev[0].record()
    for s in range(steps):
        one_step()
        ev[s + 1].record()
    torch.cuda.synchronize()
    per = sorted(ev[s].elapsed_time(ev[s + 1]) for s in range(steps))
    opt._engine.check()
    opt.close()
    return {"what": "resnet18_step", "variant": variant, "batch": batch, "steps": steps,
            "ms_per_step_median": round(per[len(per) // 2], 3), "ms_per_step_min": round(per[0], 3),
            "ms_per_step_max": round(per[-1], 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arenas", default="resnet18,bert_base")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--piece-mb", type=float, default=8.0, help="largest parameter tensor")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3, help="alternated rounds of the three step variants")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ema_timing needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    for arena in a.arenas.split(","):
        for row in kernel_timing(arena, a.iters, a.piece_mb, dev):
            print(json.dumps(row), flush=True)
    runtime.init()
    for _ in range(a.rounds):
        for variant in ("off", "ema_decay", "user_side"):
            print(json.dumps(step_timing(variant, a.batch, a.steps, a.warmup, dev)), flush=True)
    runtime.shutdown()


if __name__ == "__main__":
    main()
