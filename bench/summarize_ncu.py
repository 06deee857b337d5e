#!/usr/bin/env python
"""Summarise an .ncu-rep (captured with Nsight Compute) into a small text file.

    python bench/summarize_ncu.py prof_update.ncu-rep psb_update_kernel.ncu.txt
"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tmem.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "launch__waves_per_multiprocessor",
    "lts__t_bytes.sum", "l1tex__t_bytes.sum", "smsp__cycles_active.avg",
    "smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio",
]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    lines = [f"# ncu --set full --clock-control none --import-source on   ({rep})", ""]
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")]
        lines.append(f"## {name}")
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                lines.append(f"{k:85s} {r[i]:>16s} {units[i]}")
        lines.append("")
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], stdout=subprocess.PIPE, text=True).stdout
    srows = list(csv.reader(io.StringIO(src)))
    if len(srows) > 2:
        sh = srows[0]
        def col(n):
            return sh.index(n) if n in sh else None
        c_src, c_samp = col("Source"), col("# Samples") if col("# Samples") is not None else col("Warp Stall Sampling (All Samples)")
        if c_src is not None and c_samp is not None:
            top = sorted((r for r in srows[1:] if len(r) > c_samp and r[c_samp].replace(".", "").isdigit()),
                         key=lambda r: -float(r[c_samp]))[:15]
            lines.append("## hottest source/SASS lines by warp-stall samples")
            for r in top:
                lines.append(f"{r[c_samp]:>8s}  {r[c_src][:140]}")
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[:60]))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
