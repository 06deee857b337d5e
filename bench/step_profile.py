#!/usr/bin/env python
"""Per-kernel profile of the headline training step on ONE GPU (``bench.py --gpus 1``'s model, data, cuDNN flags, device
engine and ``attach``), written to ``--out``:

- ``kernels.txt``: every kernel of the recorded steps, aggregated by name (total / calls / mean, per step);
- ``categories.json``: per-step totals for cuDNN fprop / dgrad / wgrad, our ``psb_*`` kernels and the other ATen kernels;
- ``wgrad_by_shape.txt``: cuDNN weight-gradient time per convolution shape (``aten::convolution_backward`` input shapes).

The kernel table and the category totals come from a run with CUDA activity only.  The per-shape attribution needs the
operator that launched each kernel, so it is a second, separate run with CPU activity and input shapes recorded as well.

    python bench/step_profile.py --out bench_out/step_profile [--model resnet18] [--steps 10]
"""
import argparse
import collections
import importlib.util
import json
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _bench_module():
    spec = importlib.util.spec_from_file_location("_bench_main", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def category(name: str) -> str:
    n = name.lower()
    if "psb_" in n:
        return "ours (psb_*)"
    if "wgrad" in n:
        return "cudnn wgrad"
    if "dgrad" in n:
        return "cudnn dgrad"
    if "fprop" in n or "implicit_convolve" in n:
        return "cudnn fprop"
    if "cudnn" in n or "xmma" in n or "cutlass" in n or n.startswith("sm90_") or "gemm" in n:
        return "library gemm/other cudnn"
    return "other aten"


def kernel_events(prof):
    return [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_out/step_profile")
    ap.add_argument("--model", default="resnet18", choices=["resnet18", "resnet50"])
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10, help="steps recorded in each profiled run")
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    os.makedirs(a.out, exist_ok=True)
    bench = _bench_module()
    import pytorch_ps_mpi_b200 as ps

    w = ps.runtime.init()
    device = w.device
    ps.runtime.bind_to_gpu_numa_node(device)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    args = argparse.Namespace(model=a.model, batch=a.batch, code="identity", seq=128)
    model, make_batch, loss_fn, _ = bench.build(args, device, ps)
    gen0 = torch.Generator().manual_seed(7)
    xb, yb = (t.to(device) for t in make_batch(gen0))
    for _ in range(2):
        loss_fn(xb, yb).backward()
        model.zero_grad(set_to_none=True)
    named = list(model.named_parameters())
    opt = ps.SGD(named, [p for _, p in named], code=bench.make_code(ps, "identity"), mode="ps", engine="device",
                 average=True, lr=0.05, momentum=0.9, weight_decay=1e-4)
    model.attach(opt)
    gen = torch.Generator().manual_seed(1234)
    batches = [tuple(t.to(device) for t in make_batch(gen)) for _ in range(4)]

    def step(i):
        x, y = batches[i % len(batches)]
        opt.zero_grad(set_to_none=True)
        loss_fn(x, y).backward()
        opt.step()

    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize(device)

    # run 1: CUDA activity only -> kernel table + categories
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            step(i)
        torch.cuda.synchronize(device)
    by_name = collections.defaultdict(lambda: [0.0, 0])
    for e in kernel_events(prof):
        by_name[e.name][0] += e.time_range.elapsed_us()
        by_name[e.name][1] += 1
    cats = collections.defaultdict(float)
    total = 0.0
    rows = sorted(by_name.items(), key=lambda kv: -kv[1][0])
    with open(os.path.join(a.out, "kernels.txt"), "w") as f:
        f.write(f"{'us/step':>10} {'calls/step':>10} {'us/call':>9}  category | kernel\n")
        for name, (us, n) in rows:
            cats[category(name)] += us / a.steps
            total += us / a.steps
            f.write(f"{us / a.steps:10.1f} {n / a.steps:10.1f} {us / n:9.1f}  {category(name)} | {name[:200]}\n")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    summary = {"model": a.model, "batch": a.batch, "steps_recorded": a.steps, "card": card,
               "kernel_us_per_step": round(total, 1), "categories_us_per_step": {k: round(v, 1) for k, v in sorted(cats.items())}}

    # run 2: CPU + CUDA with input shapes -> cuDNN wgrad per convolution shape
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True) as prof2:
        for i in range(a.steps):
            step(i)
        torch.cuda.synchronize(device)
    per_shape = collections.defaultdict(lambda: [0.0, 0.0, 0, 0.0])

    def walk(ev, acc):
        for k in ev.kernels:
            acc.append(k)
        for c in ev.cpu_children:
            walk(c, acc)

    for ev in prof2.events():
        if ev.name != "aten::convolution_backward" or ev.device_type != torch.autograd.DeviceType.CPU:
            continue
        ks = []
        walk(ev, ks)
        shp = ev.input_shapes
        key = f"dy{shp[0]} x{shp[1]} w{shp[2]}" if len(shp) > 2 else str(shp)
        for k in ks:
            c = category(k.name)
            if c == "cudnn wgrad":
                per_shape[key][0] += k.duration / a.steps
            elif c == "cudnn dgrad":
                per_shape[key][1] += k.duration / a.steps
            else:
                per_shape[key][3] += k.duration / a.steps
        per_shape[key][2] += 1
    with open(os.path.join(a.out, "wgrad_by_shape.txt"), "w") as f:
        f.write(f"{'wgrad us/step':>14} {'dgrad us/step':>14} {'other us/step':>14} {'convs/step':>10}  "
                "shape (grad output, input, weight)\n")
        for key, (wg, dg, n, other) in sorted(per_shape.items(), key=lambda kv: -kv[1][0]):
            f.write(f"{wg:14.1f} {dg:14.1f} {other:14.1f} {n / a.steps:10.1f}  {key}\n")
    summary["wgrad_by_shape_us_per_step"] = {k: round(v[0], 1) for k, v in per_shape.items()}
    with open(os.path.join(a.out, "categories.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))
    opt.close()
    ps.runtime.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
