#!/usr/bin/env python
"""Extracts the judged metrics of one kernel from an .ncu-rep into a small CSV.
usage: python tools/ncu_summary.py <x>.ncu-rep <x>_ncu.csv"""
import csv
import subprocess
import sys

KEEP = """gpu__time_duration.sum dram__bytes_read.sum dram__bytes_write.sum gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed
sm__throughput.avg.pct_of_peak_sustained_elapsed launch__registers_per_thread launch__grid_size launch__block_size
launch__occupancy_limit_registers launch__occupancy_limit_shared_mem sm__warps_active.avg.per_cycle_active smsp__inst_executed.sum
smsp__issue_active.avg.pct_of_peak_sustained_active smsp__thread_inst_executed_per_inst_executed.ratio
sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active
sm__inst_executed_pipe_tma.avg.pct_of_peak_sustained_active l1tex__t_requests_pipe_lsu_mem_local_op_ld.sum
l1tex__t_requests_pipe_lsu_mem_local_op_st.sum smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio
smsp__average_warps_issue_stalled_wait_per_issue_active.ratio smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio
smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio
smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio
smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio
smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active
lts__t_bytes.sum l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum""".split()


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as f:
        f.write("kernel,metric,unit,value\n")
        for vals in rows[2:]:
            name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
            for i, h in enumerate(hdr):
                if h in KEEP:
                    f.write(f"{name.split('(')[0]},{h},{units[i]},{vals[i]}\n")
    print(open(out).read())


if __name__ == "__main__":
    main()
