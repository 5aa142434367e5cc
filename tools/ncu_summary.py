#!/usr/bin/env python3
"""Summarises an .ncu-rep (one `ncu --set full` capture of k_mix_voices) into a text
file: headline metrics, stall mix, and stall samples per
barrier-delimited code region.   usage: ncu_summary.py <file.ncu-rep> <out.txt>"""
import csv
import io
import subprocess
import sys

rep, out = sys.argv[1], sys.argv[2]


def page(name, extra=()):
    txt = subprocess.run(["ncu", "-i", rep, "--page", name, "--csv", *extra], capture_output=True,
                         text=True).stdout
    return list(csv.reader(io.StringIO(txt)))


lines = []
raw = page("raw")
hdr, units, vals = raw[0], raw[1], raw[2]
want = ["Kernel Name", "gpu__time_duration.sum", "launch__grid_size", "launch__block_size",
        "launch__registers_per_thread", "launch__occupancy_limit_registers",
        "launch__occupancy_limit_shared_mem", "launch__shared_mem_per_block_dynamic",
        "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
        "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__bytes_read.sum.per_second",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]
lines.append(f"# ncu summary of {rep}\n")
for h, u, v in zip(hdr, units, vals):
    if h in want or h.startswith("smsp__average_warps_issue_stalled") and h.endswith("per_issue_active.ratio"):
        lines.append(f"{h:95s} {u:14s} {v}")

sass = page("source", ["--print-source", "sass"])
h = sass[1]
si, src, ie = h.index("Warp Stall Sampling (All Samples)"), h.index("Source"), h.index("Instructions Executed")
data = []
for r in sass[2:]:
    try:
        data.append((int(r[si]), r[src], int(r[ie])))
    except Exception:
        pass
tot = sum(d[0] for d in data) or 1
lines.append("\n# stall samples per BAR.SYNC-delimited region (0: per-voice setup + phase table, "
             "then window fill, resample, ..., FIR, write-back)")
seg = acc = ex = start = 0
for i, d in enumerate(data):
    acc += d[0]
    ex += d[2]
    if "BAR.SYNC" in d[1] or i == len(data) - 1:
        lines.append(f"region {seg:2d} sass[{start:5d}-{i:5d}] samples {acc:6d} ({acc / tot * 100:5.1f}%) "
                     f"warp-instructions {ex:10d}")
        seg += 1
        acc = ex = 0
        start = i + 1
lines.append("\n# top 15 instructions by stall samples")
for i, d in sorted(enumerate(data), key=lambda x: -x[1][0])[:15]:
    lines.append(f"{d[0]:6d} {d[0] / tot * 100:5.1f}%  exec={d[2]:9d}  {d[1][:90]}")
open(out, "w").write("\n".join(lines) + "\n")
print("\n".join(lines))
