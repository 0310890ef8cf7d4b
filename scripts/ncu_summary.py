#!/usr/bin/env python
"""Summarise an .ncu-rep (run here, no GPU needed): key metrics of each profiled launch + the SASS lines with the most
stall samples.  usage: python scripts/ncu_summary.py prof.ncu-rep > prof.md"""
import csv
import io
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
hdr, units = rows[0], rows[1]
keys = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "smsp__inst_executed.sum", "sm__cycles_elapsed.avg", "sm__cycles_active.avg",
        "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_static",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio", "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio"]
print(f"# ncu summary of `{rep}`\n")
for r in rows[2:]:
    print(f"## {r[hdr.index('Kernel Name')][:110]}\n")
    print("| metric | value | unit |\n|---|---|---|")
    for k in keys:
        if k in hdr:
            print(f"| {k} | {r[hdr.index(k)]} | {units[hdr.index(k)]} |")
    print()
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(src)))
h = None
for i, r in enumerate(rows):
    if "Source" in r and "# Samples" in r:
        h = i
        break
if h is not None:
    hdr = rows[h]
    ix = {n: i for i, n in enumerate(hdr)}
    data = [r for r in rows[h + 1:] if len(r) == len(hdr)]
    stalls = [n for n in hdr if n.startswith("stall_") and "Not Issued" not in n]
    tot = sum(int(r[ix["# Samples"]]) for r in data)
    agg = sorted(((s, sum(int(r[ix[s]]) for r in data)) for s in stalls), key=lambda x: -x[1])
    print(f"## warp-state samples ({tot} total)\n")
    print(", ".join(f"{s}={v}" for s, v in agg if v))
    print("\n## SASS instructions with the most samples\n")
    print("| samples | executed | avg threads | instruction | top stalls |\n|---|---|---|---|---|")
    for r in sorted(data, key=lambda r: -int(r[ix["# Samples"]]))[:25]:
        st = sorted(((s, int(r[ix[s]])) for s in stalls if int(r[ix[s]]) > 0), key=lambda x: -x[1])[:2]
        print(f"| {r[ix['# Samples']]} | {r[ix['Instructions Executed']]} | {r[ix['Avg. Threads Executed']]} | `{r[ix['Source']].strip()[:70]}` | {st} |")
