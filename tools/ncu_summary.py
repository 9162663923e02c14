#!/usr/bin/env python3
"""Condense an Nsight Compute report into a handful of lines.

    ncu --set full --clock-control none --import-source on -k regex:fmha -c 6 -o out/x  python bench/attn_bench.py ...
    python tools/ncu_summary.py out/x.ncu-rep [kernel-name-substring] > ncu_x.txt

Reads the report with ``ncu -i ... --page raw --csv`` (works without a GPU) and prints, per selected kernel launch,
the metrics the profiling recipe asks for: duration, issue / tensor-pipe / memory utilisation, DRAM traffic, occupancy
limits and the warp-stall breakdown.
"""
import csv
import io
import subprocess
import sys

KEEP = [
    "gpu__time_duration.sum",
    "smsp__inst_executed.sum",
    "sm__issue_active.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_tensor",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_subpipe",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "launch__registers_per_thread",
    "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem",
    "launch__grid_size",
    "launch__block_size",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__inst_executed_pipe_xu.sum",
    "sm__inst_executed_pipe_xu",
    "lts__t_sectors.avg.pct_of_peak_sustained_elapsed",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "dram__bytes_read.sum",
    "dram__bytes_write.sum",
    "smsp__average_warps_issue_stalled",
]


def main():
    rep = sys.argv[1]
    want = sys.argv[2] if len(sys.argv) > 2 else ""
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    header, units, data = rows[0], rows[1], rows[2:]
    name_col = header.index("Kernel Name")
    seen = {}
    for row in data:
        name = row[name_col]
        if want and want not in name:
            continue
        seen[name] = seen.get(name, 0) + 1
        if seen[name] > 1:   # first launch of each kernel is enough (the bench repeats it)
            continue
        print("== {}".format(name[:150]))
        for col, (metric, unit) in enumerate(zip(header, units)):
            if any(metric.startswith(k) for k in KEEP) and row[col] not in ("", "n/a"):
                print("{:<86s} {} {}".format(metric, row[col], unit))
        print()


if __name__ == "__main__":
    main()
