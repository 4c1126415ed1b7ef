#!/usr/bin/env python
"""Summarise an `ncu --set full` report (read here, on the CPU box) into one CSV row per captured launch with the metrics the
roofline record needs: duration, DRAM bytes read / written, DRAM and tensor-pipe utilisation, issue activity, registers, grid.

  python tools/ncu_summary.py results/prof.ncu-rep summary.csv

The report is exported with `ncu -i <rep> --page raw --csv` (first row metric names, second row units)."""
import csv
import io
import subprocess
import sys

WANT = [
    ("Kernel Name", "kernel"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__registers_per_thread", "regs"),
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram_read"),
    ("dram__bytes_write.sum", "dram_write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"),
    ("dram__throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct2"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor_pct"),
    ("sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active", "tensor_hmma_pct"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor_inst"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm_pct"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue_active_pct"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved_occupancy_pct"),
    ("lts__t_sector_hit_rate.pct", "l2_hit_pct"),
    ("l1tex__t_sector_hit_rate.pct", "l1_hit_pct"),
    ("smsp__average_warp_latency_issue_stalled_long_scoreboard.ratio", "stall_long_scoreboard"),
    ("smsp__average_warp_latency_issue_stalled_barrier.ratio", "stall_barrier"),
    ("smsp__average_warp_latency_issue_stalled_no_instruction.ratio", "stall_no_instruction"),
    ("smsp__average_warp_latency_issue_stalled_lg_throttle.ratio", "stall_lg_throttle"),
    ("smsp__average_warp_latency_issue_stalled_math_pipe_throttle.ratio", "stall_math_throttle"),
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    # skip any non-CSV preamble lines
    start = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    header, units, data = rows[start], rows[start + 1], rows[start + 2:]
    col = {name: i for i, name in enumerate(header)}
    picked = [(src, dst) for src, dst in WANT if src in col]
    with open(out, "w", newline="") as f:
        w = csv.writer(f)
        w.writerow([dst + (f" [{units[col[src]]}]" if units[col[src]] else "") for src, dst in picked])
        for r in data:
            if len(r) < len(header):
                continue
            w.writerow([r[col[src]] for src, dst in picked])
    print(f"{len(data)} launches -> {out}; columns: {[d for _, d in picked]}")
    missing = [src for src, _ in WANT if src not in col]
    if missing:
        print("not in this report:", missing)


if __name__ == "__main__":
    main()
