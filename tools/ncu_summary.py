#!/usr/bin/env python
"""Key metrics of an ncu report as text:  python tools/ncu_summary.py out/x.ncu-rep > x.txt"""
import csv
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_active",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_tensor_subpipe_imma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor_subpipe_dmma.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
        "sm__cycles_elapsed.max", "smsp__cycles_active.avg"]
rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
H, U = rows[0], rows[1]
print(f"# ncu --set full --clock-control none --import-source on   ({rep.split('/')[-1]})")
for r in rows[2:]:
    print("kernel:", r[H.index("Kernel Name")][:110], " grid", r[H.index("Grid Size")], " block", r[H.index("Block Size")])
    for w in WANT:
        if w in H:
            print(f"  {w:90s} {r[H.index(w)]:>18s} {U[H.index(w)]}")
