"""Summarise an .ncu-rep (ncu --set full) into a small text table for profiles/.

    python tools/ncu_summary.py prof.ncu-rep > profiles/pair_kernels_ncu.txt
"""
import csv
import io
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "duration"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "active threads / instruction"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots busy"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM throughput"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "FMA pipe"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "ALU pipe"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "LSU pipe"),
    ("l1tex__throughput.avg.pct_of_peak_sustained_active", "L1/TEX throughput"),
    ("l1tex__t_sector_hit_rate.pct", "L1 sector hit rate"),
    ("lts__t_sector_hit_rate.pct", "L2 sector hit rate"),
    ("lts__throughput.avg.pct_of_peak_sustained_elapsed", "L2 throughput"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "DRAM throughput"),
    ("dram__bytes_read.sum", "DRAM read"),
    ("dram__bytes_write.sum", "DRAM write"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy"),
    ("launch__registers_per_thread", "registers / thread"),
    ("launch__grid_size", "grid"),
    ("launch__block_size", "block"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard (warps/issue)"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait"),
    ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "stall not_selected"),
    ("smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "stall branch_resolving"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_scoreboard"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall math_pipe_throttle"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "stall lg_throttle"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall mio_throttle"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
]


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    print(f"# ncu --set full --clock-control none summary of {rep}")
    for r in rows[2:]:
        print()
        print("kernel:", r[hdr.index("Kernel Name")])
        for key, label in WANT:
            if key in hdr:
                i = hdr.index(key)
                print(f"  {label:38s} {r[i]:>16s} {units[i]:10s}  [{key}]")


if __name__ == "__main__":
    main()
