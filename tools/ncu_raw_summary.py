#!/usr/bin/env python
"""Condense `ncu -i X.ncu-rep --page raw --csv` (one captured launch of `ncu --set full`) into the handful of counters the docs quote.
    ncu -i gemm_pair.ncu-rep --page raw --csv > gemm_pair_raw.csv
    python tools/ncu_raw_summary.py gemm_pair_raw.csv "command line of the capture" > profiles/ncu_gemm_pair.txt
"""
import csv
import sys

KEEP = (
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor.sum", "sm__inst_executed_pipe_tensor.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "lts__t_sector_hit_rate.pct", "launch__registers_per_thread", "launch__cluster_dim_x", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "smsp__inst_executed.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
)


def main():
    rows = list(csv.reader(open(sys.argv[1], errors="replace")))
    hi = next(i for i, r in enumerate(rows) if r and r[0] == "ID")
    names = rows[hi]
    if "Metric Name" in names:  # long format (one row per metric): fold the first launch into name -> (value, unit)
        im, iu, iv, ik = names.index("Metric Name"), names.index("Metric Unit"), names.index("Metric Value"), names.index("Kernel Name")
        first = rows[hi + 1][0]
        data = [r for r in rows[hi + 1:] if len(r) > iv and r[0] == first]
        kernel = data[0][ik]
        names = [r[im] for r in data]
        units = [r[iu] for r in data]
        vals = [r[iv] for r in data]
        col = {n: i for i, n in enumerate(names)}
    else:  # wide format of `--page raw`: names, units, then one row per launch
        units, vals = rows[hi + 1], rows[hi + 2]
        col = {n: i for i, n in enumerate(names)}
        kernel = vals[col["Kernel Name"]] if "Kernel Name" in col else ""
    if len(sys.argv) > 2:
        print(sys.argv[2])
    print(f"kernel: {kernel}")
    shown = set()
    for n in KEEP:
        if n in col:
            print(f"{n:<96}{vals[col[n]]} {units[col[n]]}")
            shown.add(n)
    for n in names:  # every warp-stall reason and every tensor-pipe counter the report holds
        if n in shown or n not in col:
            continue
        if ("issue_stalled" in n and n.endswith("per_issue_active.ratio")) or "pipe_tensor" in n or "tmem" in n:
            print(f"{n:<96}{vals[col[n]]} {units[col[n]]}")


if __name__ == "__main__":
    main()
