#!/usr/bin/env python
"""Every epilogue of the wgmma GEMM (``psb_bcast_gemm_kernel``, ``bcast_gemm.cu``) next to cuBLAS; needs a GPU.

``epi0`` direct fragment stores, ``epi1`` staged full-line stores, ``epi3`` TMA store (N % 8 == 0).  Numerics are checked against
an fp32 matmul first; CUDA-event timing, L2 flushed, one JSON line per (shape, variant).
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch_ps_mpi_b200.ops.linear import bcast_linear   # noqa: E402

TWO_CTA = 2
VARIANTS = [("prod", TWO_CTA)]            # epilogue selector 0 = the production choice (TMA store if N % 8 == 0, else staged)
for epi, sel in ((0, 4), (1, 1), (3, 3)):   # kernel template EPI → selector bits of `variant`
    VARIANTS.append((f"epi{epi}", TWO_CTA | sel << 4))

SHAPES = [("bert.ffn_in", 16384, 3072, 768), ("bert.qkv", 16384, 2304, 768), ("bert.ffn_out", 16384, 768, 3072),
          ("mlp.fc1", 8192, 4096, 784), ("stem", 256 * 112 * 112 // 8, 64, 176), ("square4096", 4096, 4096, 4096),
          ("ragged", 1000, 328, 264), ("ragged.unaligned_n", 515, 330, 72)]


def bench(fn, flush, iters=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2] * 1e-3


def main():
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    out = open(os.path.join(ROOT, "bench_out", "gemm_variants.jsonl"), "w")
    bad = 0
    for name, M, N, K in SHAPES:
        torch.manual_seed(0)
        x = (torch.randn(M, K, device=dev) / K ** 0.5).bfloat16()
        w = torch.randn(N, K, device=dev).bfloat16()
        b = torch.randn(N, device=dev)
        ref = torch.relu(x.float() @ w.float().t() + b)
        t_lib = bench(lambda: torch.nn.functional.linear(x, w), flush)
        fl = 2.0 * M * N * K
        for tag, v in VARIANTS:
            if (v >> 4) & 15 == 3 and N % 8:
                continue
            rec = {"shape": name, "M": M, "N": N, "K": K, "variant": tag, "code": v}
            if (v >> 8) == 0:             # a storing variant: numerics first (bias + ReLU exercised too)
                y = bcast_linear(x, w, b, relu=True, variant=v).float()
                err = (y - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)
                rec["max_rel_err"] = err
                if not err < 2e-2:
                    bad += 1
                    rec["FAILED"] = True
            t = bench(lambda: bcast_linear(x, w, variant=v), flush)
            rec.update(us=t * 1e6, tflops=fl / t / 1e12, cublas_us=t_lib * 1e6)
            line = json.dumps(rec)
            print(line, flush=True)
            out.write(line + "\n")
            out.flush()
    out.close()
    if bad:
        print(f"{bad} variant(s) FAILED the numerics check", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
