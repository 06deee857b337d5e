#!/usr/bin/env python
"""wgmma ``bcast_gemm`` vs cuBLAS (torch.matmul) on the first-forward-GEMM shapes of the zoo.

CUDA-event timing after warm-up, L2 flushed between iterations (256 MB memset), fraction of the
MEASURED bf16 peak in MEASURED_PEAKS.json if present, else of the H100 SXM data sheet's dense bf16 rate (989 TFLOP/s at
700 W).  One JSON line per shape."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch_ps_mpi_b200.ops.linear import bcast_linear   # noqa: E402


def peak_tflops():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"], "measured"
    except Exception:
        return 989.0, "H100 SXM data sheet, dense bf16"


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
    peak, how = peak_tflops()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    shapes = [("mlp.fc1 b=4096", 4096, 512, 784), ("bert.qkv b*s=16384", 16384, 2304, 768),
              ("bert.ffn_in b*s=16384", 16384, 3072, 768), ("bert.ffn_out b*s=16384", 16384, 768, 3072),
              ("square 8192", 8192, 8192, 8192), ("bert.decoder 16384x30522", 16384, 30528, 768)]
    for name, M, N, K in shapes:
        x = (torch.randn(M, K, device=dev) / K ** 0.5).bfloat16()
        w = torch.randn(N, K, device=dev).bfloat16()
        t_ours = bench(lambda: bcast_linear(x, w, variant=2), flush)
        t_1cta = bench(lambda: bcast_linear(x, w, variant=1), flush)
        t_lib = bench(lambda: torch.nn.functional.linear(x, w), flush)
        fl = 2.0 * M * N * K
        print(json.dumps({"shape": name, "M": M, "N": N, "K": K, "ours_us": t_ours * 1e6, "ours_1cta_us": t_1cta * 1e6, "cublas_us": t_lib * 1e6,
                          "ours_tflops": fl / t_ours / 1e12, "cublas_tflops": fl / t_lib / 1e12,
                          "ours_frac_of_peak": fl / t_ours / 1e12 / peak, "peak_tflops": peak, "peak_source": how}), flush=True)


if __name__ == "__main__":
    main()
