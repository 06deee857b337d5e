#!/usr/bin/env python
"""Validate and time the EXPERIMENTAL fused stem kernels (``csrc/kernels/stem_kernels.cu``) — needs a GPU.

Sections (``--only a,b,...``; default all):

* ``numerics``        ``stem_fwd`` vs ``F.conv2d`` in fp32 on several image sizes (borders, odd heights, partial tiles) and
                      its BatchNorm sums vs sums of its own bf16 output;
* ``wgrad``           weight gradient of the fused autograd path (im2col rebuilt in backward) vs the default path;
* ``wgrad_implicit``  ``psb_stem_wgrad_kernel`` (MN-major wgmma operands) vs a fp32 reference, + timing at batch 256;
* ``model``           one ResNet-18 forward/backward with the fused stem vs the default path;
* ``timing``          batch 256, 224x224: stem + BN1 forward, default vs fused (CUDA events, L2 flushed);
* ``tail``            ResNet-18's stem tail (BN1 + ReLU + max-pool on 256x64x112x112): the unfused chain against the fused
                      kernels, forward and backward — bit-identical results, the least HBM bytes each moves (from the shapes),
                      time (CUDA events, L2 flushed) and achieved bandwidth as a share of the data sheet's 3.35 TB/s.

Exit code 1 if any check fails.  One JSON line per check on stdout, appended to ``bench_out/stem_fused_check.jsonl``.
A device-side trap kills the CUDA context, so on first contact run one section per process, each under ``timeout``:
``for s in numerics wgrad wgrad_implicit model timing; do timeout 300 python bench/stem_fused_check.py --only $s; done``
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pytorch_ps_mpi_b200.models import resnet as resnet_mod          # noqa: E402
from pytorch_ps_mpi_b200.ops import ext                              # noqa: E402
from pytorch_ps_mpi_b200.ops import stem as stem_mod                 # noqa: E402
from pytorch_ps_mpi_b200.ops.batchnorm import FusedBatchNormAct2d    # noqa: E402
from pytorch_ps_mpi_b200.ops.stem import _w2d, stem_conv, stem_conv_fused, stem_wgrad_implicit   # noqa: E402

BAD = 0
DEV = None


def emit(**rec):
    global BAD
    if rec.get("ok") is False:
        BAD += 1
    line = json.dumps(rec)
    print(line, flush=True)
    os.makedirs(os.path.join(ROOT, "bench_out"), exist_ok=True)
    with open(os.path.join(ROOT, "bench_out", "stem_fused_check.jsonl"), "a") as f:
        f.write(line + "\n")


def cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def bench(fn, iters=10):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
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
    return ts[len(ts) // 2]


def weight():
    torch.manual_seed(0)
    return (torch.randn(64, 3, 7, 7, device=DEV) * 0.05).bfloat16()


def sec_numerics():
    m, w = ext.cuda(), weight()
    for (n, h, wd) in [(2, 224, 224), (3, 64, 64), (1, 30, 40), (5, 17, 8), (2, 225, 256), (300, 32, 32)]:
        x = cl(torch.randn(n, 3, h, wd, device=DEV).bfloat16())
        y, sums = m.stem_fwd(x, _w2d(w), True)
        ref = F.conv2d(x.float(), w.float(), stride=2, padding=3)
        err = (y.float() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)
        yf = y.float()
        s_ref = torch.cat([yf.sum((0, 2, 3)), (yf * yf).sum((0, 2, 3))])
        serr = ((sums - s_ref).abs() / (s_ref.abs() + 1.0)).max().item()
        emit(check="numerics", shape=[n, h, wd], max_rel_err=err, sums_rel_err=serr,
             channels_last=bool(y.is_contiguous(memory_format=torch.channels_last)), ok=bool(err < 2e-2 and serr < 1e-3))


def sec_wgrad():
    w = weight()
    x = cl(torch.randn(8, 3, 224, 224, device=DEV).bfloat16())
    gy = cl(torch.randn(8, 64, 112, 112, device=DEV).bfloat16())
    wa, wb = w.clone().requires_grad_(True), w.clone().requires_grad_(True)
    stem_conv(x, wa).backward(gy)
    stem_conv_fused(x, wb)[0].backward(gy)
    gerr = (wa.grad.float() - wb.grad.float()).abs().max().item() / max(wa.grad.float().abs().max().item(), 1e-6)
    emit(check="wgrad", max_rel_diff=gerr, ok=bool(gerr < 1e-2))


def sec_wgrad_implicit():
    m = ext.cuda()
    for (n, h, wd) in [(8, 224, 224), (2, 64, 64), (1, 30, 40), (3, 17, 8), (2, 33, 256)]:
        xs = cl(torch.randn(n, 3, h, wd, device=DEV).bfloat16())
        oh, ow = (h - 1) // 2 + 1, (wd - 1) // 2 + 1
        g = cl(torch.randn(n, 64, oh, ow, device=DEV).bfloat16())
        ref = g.permute(0, 2, 3, 1).reshape(-1, 64).float().t() @ m.im2col_stem(xs).float()     # [64,176]
        got = stem_wgrad_implicit(xs, g).float()
        e = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-6)
        emit(check="wgrad_implicit", shape=[n, h, wd], max_rel_err=e, ok=bool(e < 1e-2))
    xs = cl(torch.randn(256, 3, 224, 224, device=DEV).bfloat16())
    g = cl(torch.randn(256, 64, 112, 112, device=DEV).bfloat16())
    t_impl = bench(lambda: stem_wgrad_implicit(xs, g))
    t_gemm = bench(lambda: g.permute(0, 2, 3, 1).reshape(-1, 64).t() @ m.im2col_stem(xs))
    emit(check="wgrad_timing", batch=256, implicit_ms=t_impl, im2col_plus_gemm_ms=t_gemm, ok=True)


def sec_model():
    res = {}
    for tag, fused, implicit in (("default", False, False), ("fused", True, False), ("fused+implicit_wgrad", True, True)):
        torch.manual_seed(1)
        net = resnet_mod.resnet18(num_classes=100).to(DEV).bfloat16().to(memory_format=torch.channels_last).train()
        resnet_mod._FUSED_STEM, stem_mod._IMPLICIT_WGRAD = fused, implicit
        xi = cl(torch.randn(16, 3, 224, 224, device=DEV).bfloat16())
        tgt = torch.randint(0, 100, (16,), device=DEV)
        loss = F.cross_entropy(net(xi).float(), tgt)
        loss.backward()
        res[tag] = (loss.item(), net.conv1.weight.grad.float().norm().item(), net.bn1.running_var.float().mean().item())
    resnet_mod._FUSED_STEM, stem_mod._IMPLICIT_WGRAD = False, False
    ref = res["default"]
    ok = all(abs(v[0] - ref[0]) < 5e-2 and abs(v[1] - ref[1]) < 5e-2 * max(ref[1], 1e-3) and abs(v[2] - ref[2]) < 1e-2
             for v in res.values())
    emit(check="model", results=res, ok=bool(ok))


def sec_timing():
    m, w = ext.cuda(), weight()
    x = cl(torch.randn(256, 3, 224, 224, device=DEV).bfloat16())
    bn = FusedBatchNormAct2d(64, relu=True).to(DEV).bfloat16().train()
    w2 = _w2d(w)
    with torch.no_grad():
        t_default = bench(lambda: bn(stem_conv(x, w)))
        t_fused = bench(lambda: (lambda ys: bn(ys[0], sums=ys[1]))(stem_conv_fused(x, w)))
        t_kernel = bench(lambda: m.stem_fwd(x, w2, True))
        t_conv_only = bench(lambda: stem_conv(x, w))
    emit(check="timing", batch=256, default_stem_bn_ms=t_default, fused_stem_bn_ms=t_fused, fused_kernel_ms=t_kernel,
         default_conv_only_ms=t_conv_only, ok=True)


def sec_tail():
    m = ext.cuda()
    N, C, H, W = 256, 64, 112, 112
    T = N * C * H * W * 2                     # the stem output (bf16)
    P, A, M = T // 4, T // 8, T // 16         # pooled output, 1-byte taps, 1-bit ReLU mask
    torch.manual_seed(0)
    x = cl(torch.randn(N, C, H, W, device=DEV).bfloat16())
    xf = x.float()
    sums = torch.cat([xf.sum((0, 2, 3)), (xf * xf).sum((0, 2, 3))])
    del xf
    g = (torch.randn(C, device=DEV) * 0.5 + 1.0).bfloat16()
    b = (torch.randn(C, device=DEV) * 0.5).bfloat16()
    dp = cl(torch.randn(N, C, H // 2, W // 2, device=DEV).bfloat16())
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)

    def fwd_unfused():
        y, mean, rstd, mask = m.bn_forward_presummed(x, None, g, b, rm, rv, 1e-5, 0.1, True, sums)
        return (*m.maxpool_forward(y), mean, rstd, mask)

    def fwd_fused():
        return m.bn_forward_presummed(x, None, g, b, rm, rv, 1e-5, 0.1, True, sums, pool=True)

    pu, au, mean, rstd, mask = fwd_unfused()
    pf, _, _, af = fwd_fused()
    bwd_unfused = lambda: m.bn_backward(m.maxpool_backward(dp, au, H, W), x, mask, g, mean, rstd, True, False)   # noqa: E731
    bwd_fused = lambda: m.bn_backward(dp, x, x, g, mean, rstd, True, False, pool_arg=af)                        # noqa: E731
    du, df = bwd_unfused(), bwd_fused()
    same = (torch.equal(pu.view(torch.int16), pf.view(torch.int16))
            and all(torch.equal(u.view(torch.int16), f.view(torch.int16)) for u, f in zip((du[0], du[2], du[3]), (df[0], df[2], df[3]))))
    rows = {"fwd_unfused": (fwd_unfused, 2 * T + M + T + P + A), "fwd_fused": (fwd_fused, T + P + A),
            "bwd_unfused": (bwd_unfused, P + A + T + 2 * T + M + 3 * T + M), "bwd_fused": (bwd_fused, T + P + A + 2 * T + P + A)}
    out = {}
    for name, (fn, nbytes) in rows.items():
        ms = bench(fn, iters=20)
        out[name] = {"ms": ms, "min_bytes_MB": nbytes / 1e6, "GB_per_s": nbytes / ms / 1e6, "share_of_3.35TBps": nbytes / ms / 3.35e9}
    emit(check="tail", shape=[N, C, H, W], bit_identical=bool(same), **out, ok=bool(same))


SECTIONS = {"numerics": sec_numerics, "wgrad": sec_wgrad, "wgrad_implicit": sec_wgrad_implicit, "model": sec_model,
            "timing": sec_timing, "tail": sec_tail}


def main():
    global DEV
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=",".join(SECTIONS))
    only = [s for s in ap.parse_args().only.split(",") if s]
    DEV = torch.device("cuda", 0)
    for name in only:
        SECTIONS[name]()
    if BAD:
        print(f"{BAD} check(s) FAILED", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
