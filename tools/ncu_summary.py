#!/usr/bin/env python3
"""Summarise an .ncu-rep (ncu --set full) into a few numbers: DRAM traffic, issue activity, stall reasons.
usage: python tools/ncu_summary.py x.ncu-rep > x.summary.txt"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.per_cycle_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "l1tex__data_pipe_lsu_wavefronts.sum.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    name_col = hdr.index("Kernel Name")
    print(f"# {path}  (ncu --set full --clock-control none)")
    for r in rows[2:]:
        print(f"\n== {r[name_col]}")
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                print(f"  {k:84s} {r[i]:>18s} {units[i]}")
        try:
            rd, wr = hdr.index("dram__bytes_read.sum"), hdr.index("dram__bytes_write.sum")
            f = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}
            tot = float(r[rd]) * f[units[rd]] + float(r[wr]) * f[units[wr]]
            print(f"  {'traffic = dram read + write':84s} {tot/1e9:18.4f} GB")
        except Exception:
            pass


if __name__ == "__main__":
    main(sys.argv[1])
