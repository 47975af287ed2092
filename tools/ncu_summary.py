#!/usr/bin/env python
"""Summarise an .ncu-rep (raw page) or an ncu launch-list CSV into text summaries.
    python tools/ncu_summary.py raw  x.ncu-rep > x_ncu.txt
    python tools/ncu_summary.py list launches.csv > x_launches.txt
"""
import collections
import csv
import subprocess
import sys

KEEP = ("gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__cluster", "sm__cycles_elapsed.max", "dram__bytes_read.sum",
        "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tc_cycles_active.avg.pct_of_peak_sustained_active", "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.sum.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "lts__t_sector_hit_rate.pct", "l1tex__throughput.avg.pct_of_peak_sustained_active",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio")


def raw(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    for vals in rows[2:]:
        name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
        print("kernel:", name)
        for h, u, v in zip(hdr, units, vals):
            if h in KEEP or any(h.startswith(k) for k in ("launch__cluster",)):
                print("  %-82s %-16s %s" % (h, u, v))


def launches(path):
    rows = list(csv.reader(open(path)))
    hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
    h = rows[hi]
    ki, vi = h.index("Kernel Name"), h.index("Metric Value")
    agg = collections.OrderedDict()
    for r in rows[hi + 1:]:
        if len(r) <= vi:
            continue
        k = r[ki].split("(")[0][-70:]
        a = agg.setdefault(k, [0, 0.0])
        a[0] += 1
        a[1] += float(r[vi].replace(",", ""))
    tot = sum(a[1] for a in agg.values())
    print("# per-kernel device time from `ncu --metrics gpu__time_duration.sum --clock-control none` (cold-cache, serialised: compare shares)")
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%-72s launches=%4d total=%11.3f ms  avg=%9.3f ms  share=%5.1f%%" % (k, n, t / 1e6, t / 1e6 / n, 100 * t / tot))


if __name__ == "__main__":
    {"raw": raw, "list": launches}[sys.argv[1]](sys.argv[2])
