#!/usr/bin/env python
"""Summarise an .ncu-rep (raw page) into the handful of numbers the roofline argument needs.
usage: python tools/ncu_summary.py prof.ncu-rep > summary.txt"""
import csv, subprocess, sys
KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_bytes.sum", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__warps_eligible.avg.per_cycle_active",
    "l1tex__throughput.avg.pct_of_peak_sustained_active", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "smsp__sass_average_branch_targets_threads_uniform.pct", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__cycles_active.avg", "sm__cycles_elapsed.max",
]
rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, units, data = rows[0], rows[1], rows[2:]
for r in data:
    print("=" * 100)
    print("kernel:", r[hdr.index("Kernel Name")])
    for k in KEYS:
        if k in hdr:
            i = hdr.index(k)
            print(f"  {k:75s} {r[i]:>16s} {units[i]}")
    stalls = []
    for i, k in enumerate(hdr):
        if "issue_stalled" in k and k.endswith("_per_warp_active.pct"):
            try:
                stalls.append((float(r[i]), k.replace("smsp__average_warp_latency_", "").replace("smsp__warp_issue_stalled_", "")))
            except ValueError:
                pass
    for v, k in sorted(stalls, reverse=True)[:6]:
        print(f"  stall {k:69s} {v:16.2f} %")
