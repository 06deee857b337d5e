#!/usr/bin/env python
"""Per-server update work with and without a sharded parameter server, on one GPU.

``mode='ps'`` runs the fused gather / optimizer / publish kernel (``psb_update_kernel``) over the whole arena on rank 0;
``mode='sharded'`` runs it on every rank over a 1/N range of each chunk, with compact optimizer state (``state_shift``).
This times one launch sequence over the whole arena of BERT-base and ResNet-18 (bf16 parameters, fp32 masters, Identity
bf16 wire, SGD with momentum, Adam and AdamW) against one over a contiguous 1/N of it with compact state, for N = 2, 4, 8.  One rank,
so the gather reads only the local wire arena: this is the server's own work, not the NVLink ingress.  Before every timed
launch a 256 MB buffer is written, so the launch starts with a cold L2 (50 MB on the H100), as it does in a training step
where backward has run in between; each launch is timed on its own, and the median and the range are reported.

``--ab adam,adamw`` instead compares two optimizers' whole-arena launches, alternating blocks of ``--iters`` launches of each
for ``--rounds`` rounds, so that both see the same share of whatever else runs on the machine.

    python bench/shard_update_timing.py [--iters 30] [--optims sgd,adam,adamw] [--out bench_out/shard_update.json]
    python bench/shard_update_timing.py --ab adam,adamw [--rounds 6]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch_ps_mpi_b200 import models   # noqa: E402
from pytorch_ps_mpi_b200.codings import TILE   # noqa: E402
from pytorch_ps_mpi_b200.ops import ext   # noqa: E402
from pytorch_ps_mpi_b200.parallel import device_engine as de   # noqa: E402
from pytorch_ps_mpi_b200.parallel.layout import FlatLayout   # noqa: E402


def arena_of(name):
    model = models.bert_base() if name == "bert_base" else models.resnet18(num_classes=1000)
    return FlatLayout([{"params": list(model.parameters())}], {})


def time_update(m, layout, optim, lo, hi, compact, iters, flush):
    """Per-launch times (µs) of ``iters`` update launches over tiles [lo, hi), each after an L2 flush, CUDA events around each."""
    dev = torch.device("cuda")
    nt = layout.ntiles
    n_state = (hi - lo) * TILE if compact else nt * TILE
    shift = lo if compact else 0
    wire = torch.randn(nt * TILE, device=dev).mul_(1e-3).bfloat16()
    params = torch.randn(nt * TILE, device=dev).bfloat16()
    scales = torch.ones(max(layout.nparams, 1), device=dev)
    signal = torch.zeros(512, dtype=torch.int64, device=dev)
    counters = torch.zeros(8, dtype=torch.int32, device=dev)
    tiles = layout.tile_table_fast().to(dev)
    master = torch.randn(n_state, device=dev)
    bufs = [torch.zeros(n_state, device=dev) for _ in range(1 if optim == "sgd" else 2)]
    P = m.UpdatePlan()
    P.kind, P.wire, P.opt = 0, 1, de._OPTIMS[optim].code
    P.grid = min(nt, m.update_max_grid(P.kind, P.wire, P.opt))
    P.set_rank_ptrs(0, wire.data_ptr(), scales.data_ptr(), params.data_ptr(), signal.data_ptr())
    P.configure(1, 0, nt, TILE * 2, 0, 1, de.BCAST_LOCAL, de.REDUCE_P2P, 0, 0, params.data_ptr(), master.data_ptr(),
                bufs[0].data_ptr(), bufs[1].data_ptr() if len(bufs) > 1 else 0, 0, tiles.data_ptr(), signal.data_ptr(),
                counters.data_ptr(), counters.data_ptr() + 4)
    if optim == "adam":
        hyper = [[1e-3, 0.0, 0.0, 0.0, 0.9, 0.999, 1e-8, 1e-3, 0.0, 0.0, 0.0]]
    elif optim == "adamw":
        hyper = [de._adamw_group({"lr": 1e-3, "weight_decay": 1e-2, "betas": (0.9, 0.999), "eps": 1e-8}, 10)]
    else:
        hyper = [[1e-3, 0.0, 0.9, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]]

    def launch():
        P.launch(1, hyper, 1, 1.0, 0, de.SIGNAL_NONE, tile_begin=lo, tile_end=hi, wait_value=0, state_shift=shift)

    for _ in range(5):
        launch()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in evs:
        flush.add_(1.0)                                  # evicts the arena from L2
        a.record()
        launch()
        b.record()
    torch.cuda.synchronize()
    return [a.elapsed_time(b) * 1000.0 for a, b in evs]


def stat(ts):
    ts = sorted(ts)
    return {"median": round(ts[len(ts) // 2], 1), "min": round(ts[0], 1), "max": round(ts[-1], 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--optims", default="sgd,adam,adamw")
    ap.add_argument("--ab", default=None, help="two optimizers to compare on the whole arena, alternating (e.g. adam,adamw)")
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    m = ext.cuda()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    flush = torch.zeros(64 << 20, device="cuda")        # 256 MB
    rows = []
    if a.ab:
        pair = a.ab.split(",")
        for name in ("resnet18", "bert_base"):
            layout = arena_of(name)
            nt = layout.ntiles
            per = {o: [] for o in pair}
            for _ in range(a.rounds):
                for o in pair:
                    per[o] += time_update(m, layout, o, 0, nt, False, a.iters, flush)
            row = {"arena": name, "tiles": nt, "rounds": a.rounds, **{f"{o}_us": stat(per[o]) for o in pair}}
            rows.append(row)
            print(json.dumps(dict(row, card=card)), flush=True)
    for name in (() if a.ab else ("bert_base", "resnet18")):
        layout = arena_of(name)
        nt = layout.ntiles
        for optim in a.optims.split(","):
            row = {"arena": name, "tiles": nt, "optim": optim,
                   "full_us": stat(time_update(m, layout, optim, 0, nt, False, a.iters, flush))}
            for n in (2, 4, 8):
                q = nt // n
                lo = q * (n // 2)                          # a middle shard: the compact state starts at tile lo
                row[f"shard_1/{n}_us"] = stat(time_update(m, layout, optim, lo, lo + q, True, a.iters, flush))
            rows.append(row)
            print(json.dumps(dict(row, card=card)), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
