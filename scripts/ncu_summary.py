#!/usr/bin/env python
"""Summarise .ncu-rep files into <name>.md: per captured launch the
duration, DRAM traffic, issue/ALU utilisation, occupancy and the top stall reasons."""
import csv, io, subprocess, sys

WANT = [
    ("gpu__time_duration.sum", "duration"), ("launch__grid_size", "grid"), ("launch__block_size", "block"),
    ("launch__registers_per_thread", "regs"), ("dram__bytes_read.sum", "dram_read"), ("dram__bytes_write.sum", "dram_write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram_pct"), ("lts__t_sector_hit_rate.pct", "l2_hit_pct"),
    ("l1tex__t_sector_hit_rate.pct", "l1_hit_pct"), ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps_active_pct"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue_active_pct"),
    ("sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "alu_pipe_pct"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "lsu_pipe_pct"),
    ("sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "fma_pipe_pct"),
    ("sm__inst_executed_pipe_fmaheavy.avg.pct_of_peak_sustained_active", "fmaheavy_pipe_pct"),
    ("sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "alu_cycles_pct"),
    ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "fma_cycles_pct"),
    ("launch__occupancy_limit_shared_mem", "occ_limit_smem_blocks"), ("launch__occupancy_limit_registers", "occ_limit_regs_blocks"),
    ("sm__maximum_warps_per_active_cycle_pct", "theoretical_occupancy_pct"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "threads_per_inst"), ("smsp__inst_executed.sum", "warp_insts"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall_long_scoreboard"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall_short_scoreboard"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall_wait"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall_barrier"),
    ("smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "stall_branch"),
    ("smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio", "stall_no_inst"),
    ("smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio", "stall_math_throttle"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall_mio_throttle"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "stall_lg_throttle"),
    ("smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio", "stall_not_selected"),
]


def main(rep, out, title):
    txt = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units = rows[0], rows[1]
    with open(out, "w") as f:
        f.write(f"# {title}\n\nsource: `{rep}` (ncu --set full --clock-control none)\n\n")
        for r in rows[2:]:
            name = r[hdr.index("Kernel Name")].split("(")[0]
            f.write(f"## {name}  (launch id {r[hdr.index('ID')]})\n\n| metric | value | unit |\n|---|---|---|\n")
            for key, label in WANT:
                if key in hdr:
                    i = hdr.index(key)
                    f.write(f"| {label} | {r[i]} | {units[i]} |\n")
            f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else sys.argv[1])
