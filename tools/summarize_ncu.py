#!/usr/bin/env python
"""Turn ncu outputs into small text summaries.

  python tools/summarize_ncu.py launches launches.csv > launches_<tag>.txt
  python tools/summarize_ncu.py full prof.ncu-rep   > <kernel>_<tag>.txt
"""
import collections
import csv
import io
import re
import subprocess
import sys

KEYS = [
    "Kernel Name", "Grid Size", "Block Size", "gpu__time_duration.sum", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem",
    "sm__cycles_elapsed.max", "smsp__cycles_active.avg", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
    "smsp__average_warp_latency_issue_stalled_long_scoreboard.pct", "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
]


def launches(path):
    with open(path) as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    agg, total, seq = collections.OrderedDict(), 0.0, []
    for row in csv.DictReader(lines):
        try:
            t = float(row["Metric Value"])
        except (ValueError, KeyError):
            continue
        unit = row["Metric Unit"]
        t = t / 1e3 if unit == "ns" else (t * 1e3 if unit == "ms" else t)
        name = re.sub(r"\(.*", "", re.sub(r"<.*", "", row["Kernel Name"])).replace("void ", "")[:80]
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += t
        total += t
        seq.append((name, row.get("Grid Size"), t))
    print(f"# ncu --metrics gpu__time_duration.sum --clock-control none : {len(seq)} launches, {total:.1f} us total (serialised, cold cache)")
    print(f"# {'us':>10} {'launches':>8} {'share':>6}  kernel")
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{t:12.1f} {n:8d} {100 * t / total:5.1f}%  {k}")
    ours = sum(t for k, (n, t) in agg.items() if k.startswith("pfb::"))
    print(f"# this library's kernels (pfb::*): {ours:.1f} us = {100 * ours / total:.1f}% of the step; the rest is torch/cuDNN (encoders, pre-processing)")
    print("# --- first refinement iteration, launch by launch ---")
    started = False
    for name, grid, t in seq:
        if "corr_lookup" in name or "onthefly" in name:
            if started:
                break
            started = True
        if started:
            print(f"{t:10.1f} us  grid {grid:>16}  {name}")


def full(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    idx = [i for i, h in enumerate(hdr) if h in KEYS]
    print(f"# ncu --set full --clock-control none : {path}")
    for r in rows[2:]:
        print("----")
        for i in idx:
            print(f"  {hdr[i]} [{units[i]}] = {r[i]}")


if __name__ == "__main__":
    {"launches": launches, "full": full}[sys.argv[1]](sys.argv[2])
