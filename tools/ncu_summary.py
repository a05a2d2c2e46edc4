#!/usr/bin/env python
"""Summarise an .ncu-rep (read with `ncu -i ... --page raw --csv`) into a handful of numbers per kernel."""
import csv
import io
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram % of peak"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 % of peak"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM % of peak"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe active %"),
    ("sm__inst_executed_pipe_tensor.sum", "tensor pipe inst"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("launch__registers_per_thread", "registers/thread"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smem bank conflicts"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall math_pipe_throttle"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_scoreboard"),
    ("smsp__average_warps_issue_stalled_sleeping_per_issue_active.ratio", "stall sleeping"),
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    ki = hdr.index("Kernel Name")
    for r in data:
        print(f"### {r[ki][:150]}")
        for key, label in WANT:
            if key in hdr:
                i = hdr.index(key)
                print(f"  {label:28s} {r[i]:>18s} {units[i]}")
        print()


if __name__ == "__main__":
    main(sys.argv[1])
