"""Prints the metrics the roofline discussion uses from an ncu report (`ncu --set full` capture), one block per profiled launch.
Usage: python tools/ncu_summary.py x.ncu-rep > profiles/rNN_ncu_x_summary.txt"""
import csv
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "launch__registers_per_thread", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
        "launch__waves_per_multiprocessor", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_active",
        "l1tex__t_sector_hit_rate.pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "l1tex__m_xbar2l1tex_read_bytes.sum.per_second", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio"]
out = subprocess.run(["ncu", "-i", sys.argv[1], "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, units = rows[0], rows[1]
unit = dict(zip(hdr, units))
print(f"# {sys.argv[1]} (ncu --set full --clock-control none; cold-cache, serialised replays)")
for r in rows[2:]:
    d = dict(zip(hdr, r))
    print(f"{d.get('Kernel Name', '')[:90]}  grid {d.get('Grid Size', '')} block {d.get('Block Size', '')}")
    for k in KEYS:
        if k in d and d[k] != "":
            print(f"    {k:85s} {d[k]:>16s} {unit.get(k, '')}")
