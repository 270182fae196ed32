#!/usr/bin/env python3
"""Key figures of `ncu --set full` reports as a markdown table.
usage: python tools/ncu_summary.py label=path.ncu-rep [label=path ...]"""
import csv
import io
import subprocess
import sys

KEYS = [("gpu__time_duration.sum", "kernel time [ms]"),
        ("launch__registers_per_thread", "registers / thread"),
        ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active [% of 64/SM]"),
        ("smsp__inst_executed.sum", "warp instructions"),
        ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy [%]"),
        ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "fp32 (fma) pipe cycles active [%]"),
        ("sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "fp64 pipe cycles active [%]"),
        ("l1tex__throughput.avg.pct_of_peak_sustained_active", "L1TEX / shared-memory pipe throughput [%]"),
        ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "shared-memory wavefronts [% of peak]"),
        ("lts__t_sector_hit_rate.pct", "L2 sector hit rate [%]"),
        ("dram__bytes_read.sum", "DRAM read"),
        ("dram__bytes_write.sum", "DRAM write"),
        ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait / issue"),
        ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short scoreboard / issue"),
        ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long scoreboard / issue"),
        ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall math pipe throttle / issue"),
        ("smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "stall branch resolving / issue"),
        ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "stall not selected / issue")]


def load(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    return {h: (v, u) for h, u, v in zip(hdr, units, vals)}, vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else ""


cols = [a.split("=", 1) for a in sys.argv[1:]]
data = [(lab, *load(p)) for lab, p in cols]
print("| metric | " + " | ".join(lab for lab, _, _ in data) + " |")
print("|---|" + "---|" * len(data))
for key, name in KEYS:
    cells = []
    for _, d, _ in data:
        v, u = d.get(key, ("", ""))
        try:
            f = float(v)
            cells.append(f"{f:.4g} {u}".strip() if u not in ("%", "inst", "") else f"{f:.4g}")
        except ValueError:
            cells.append(v)
    print(f"| {name} | " + " | ".join(cells) + " |")
print()
for lab, _, kn in data:
    print(f"* `{lab}`: `{kn[:160]}`")
