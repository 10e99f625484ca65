#!/usr/bin/env python
"""Turns an `ncu --set full` report into a short text summary.
usage: python profiles/summarize_ncu.py prof.ncu-rep > <name>.txt"""
import csv
import io
import subprocess
import sys

RAW = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
       "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
       "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__waves_per_multiprocessor",
       "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
       "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
       "sm__inst_executed_pipe_tma.avg.pct_of_peak_sustained_active", "smsp__thread_inst_executed_per_inst_executed.ratio"]
DETAILS = ["Executed Ipc Active", "Executed Ipc Elapsed", "Issue Slots Busy", "One or More Eligible", "Active Warps Per Scheduler",
           "Eligible Warps Per Scheduler", "Theoretical Occupancy", "Achieved Occupancy", "L2 Hit Rate", "L1/TEX Hit Rate",
           "Static Shared Memory Per Block", "Grid Size", "Block Size"]


def run(args):
    return subprocess.run(["ncu", "-i", sys.argv[1], *args], capture_output=True, text=True).stdout


def main():
    raw = list(csv.reader(io.StringIO(run(["--page", "raw", "--csv"]))))
    H, units, rows = raw[0], raw[1], raw[2:]
    det = list(csv.reader(io.StringIO(run(["--page", "details", "--csv"]))))
    DH = det[0]
    di = {k: DH.index(k) for k in ("ID", "Metric Name", "Metric Value", "Metric Unit")}
    print(f"# ncu --set full --clock-control none summary of {sys.argv[1]}")
    print("# (per-launch values; captured under the profiler, so durations are cold-cache/serialised: compare shares, not absolutes)")
    for n, r in enumerate(rows):
        print(f"\n== launch {n}: {r[H.index('Kernel Name')][:110]}")
        for m in RAW:
            if m in H:
                i = H.index(m)
                print(f"  {m:72s} {r[i]:>16s} {units[i]}")
        for d in det[1:]:
            if d[di['ID']] == str(n) and d[di['Metric Name']] in DETAILS:
                print(f"  {d[di['Metric Name']]:72s} {d[di['Metric Value']]:>16s} {d[di['Metric Unit']]}")
        rd, wr = float(r[H.index('dram__bytes_read.sum')]), float(r[H.index('dram__bytes_write.sum')])
        ur, uw = units[H.index('dram__bytes_read.sum')], units[H.index('dram__bytes_write.sum')]
        mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
        print(f"  {'traffic = dram read + write':72s} {(rd * mult[ur] + wr * mult[uw]) / 1e6:16.3f} MB")


if __name__ == "__main__":
    main()
