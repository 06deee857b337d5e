#!/usr/bin/env python
"""Write SASS evidence of the built objects into ``profiles/sm90a/`` (git-ignored; CPU only, needs cuobjdump):

    python scripts/dump_sass.py            # after __graft_entry__.build()

* ``profiles/sm90a/sass/<kernel>.sass``   the full listing of one instantiation of every named hot-path kernel
* ``profiles/sm90a/sass_mnemonics_<obj>.txt`` opcode histogram per object file (what proves wgmma / TMA / multimem: HGMMA,
                                          UTMALDG(.MULTICAST) / UTMASTG, LDGMC…HPADD (multimem.ld_reduce), *.STRONG.SYS)
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "pytorch_ps_mpi_b200", "_build")
OUT = os.path.join(ROOT, "profiles", "sm90a")

# (object, regex on the demangled function header, output name)
KERNELS = [
    ("ps_kernels.o", r"psb_update_kernel<0, 1, 0>", "psb_update_kernel_dense_bf16_sgd"),
    ("ps_kernels.o", r"psb_update_kernel<2, 1, 1>", "psb_update_kernel_topk_bf16_adam"),
    ("ps_kernels.o", r"psb_encode_kernel<2, 1, false>", "psb_encode_kernel_topk_bf16"),
    ("ps_kernels.o", r"psb_select_kernel", "psb_select_kernel"),
    ("ps_kernels.o", r"psb_snapshot_fetch", "psb_snapshot_fetch"),
    ("bcast_gemm.o", r"psb_bcast_gemm_kernel<128, 2, 3>", "psb_bcast_gemm_kernel_pair_tma_store"),
    ("bcast_gemm.o", r"psb_bcast_gemm_kernel<128, 1, 3>", "psb_bcast_gemm_kernel_1cta_tma_store"),
    ("stem_kernels.o", r"psb_stem_fwd_kernel", "psb_stem_fwd_kernel"),
    ("stem_kernels.o", r"psb_stem_wgrad_kernel", "psb_stem_wgrad_kernel"),
    ("bn_kernels.o", r"psb_bn_bwd_reduce<true, true>", "psb_bn_bwd_reduce_relu_masked"),
    ("pool_kernels.o", r"psb_maxpool_bwd_quads", "psb_maxpool_bwd_quads"),
]


def sass(obj):
    exe = "cuobjdump" if subprocess.run(["which", "cuobjdump"], stdout=subprocess.PIPE).returncode == 0 else "/usr/local/cuda/bin/cuobjdump"
    raw = subprocess.run([exe, "-sass", os.path.join(OBJ, obj)], stdout=subprocess.PIPE, text=True, check=True).stdout
    dem = subprocess.run(["c++filt"], input=raw, stdout=subprocess.PIPE, text=True).stdout
    return dem


def main():
    os.makedirs(os.path.join(OUT, "sass"), exist_ok=True)
    cache = {}
    for obj, rx, name in KERNELS:
        path = os.path.join(OBJ, obj)
        if not os.path.exists(path):
            print("skip", obj, "(not built)")
            continue
        text = cache.setdefault(obj, sass(obj))
        blocks = re.split(r"(?m)^\s*Function : ", text)
        hit = next((b for b in blocks[1:] if re.search(rx, b.splitlines()[0])), None)
        if hit is None:
            print("NOT FOUND", obj, rx)
            continue
        with open(os.path.join(OUT, "sass", name + ".sass"), "w") as f:
            f.write("Function : " + hit)
        print(f"{name}: {len(hit.splitlines())} lines")
    for obj, text in cache.items():
        ops = collections.Counter()
        for line in text.splitlines():
            m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d\s+)?([A-Z][A-Z0-9_.]+)", line)
            if m:
                ops[m.group(1)] += 1
        with open(os.path.join(OUT, f"sass_mnemonics_{obj[:-2]}.txt"), "w") as f:
            for op, n in ops.most_common():
                f.write(f"{n:7d} {op}\n")


if __name__ == "__main__":
    sys.exit(main())
