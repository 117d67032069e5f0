"""Summarise an .ncu-rep (no GPU needed to read it) into a small text file.
usage: python scripts/ncu_summary.py prof.ncu-rep name.summary.txt"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum",
    "dram__bytes_read.sum",
    "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct",
    "l1tex__t_sector_hit_rate.pct",
    "lts__t_sectors_srcunit_tex_op_read.sum",
    "lts__t_sectors_srcunit_tex_op_write.sum",
    "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
    "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
    "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread",
    "launch__grid_size",
    "launch__block_size",
    "launch__waves_per_multiprocessor",
    "launch__occupancy_limit_registers",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_dispatch_stall_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_no_instruction_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_imc_miss_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_drain_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_sleeping_per_issue_active.ratio",
    "smsp__warps_eligible.avg.per_cycle_active",
    "smsp__warps_active.avg.per_cycle_active",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__inst_executed_op_shared_ld.sum",
    "smsp__inst_executed_op_shared_st.sum",
    "smsp__inst_executed_pipe_fp64.sum",
    "smsp__inst_executed_pipe_fma.sum",
    "smsp__inst_executed_pipe_alu.sum",
    "smsp__inst_executed_pipe_lsu.sum",
    "sm__inst_executed_pipe_fp64.avg.pct_of_peak_sustained_active",
    "sm__cycles_elapsed.max",
    "launch__shared_mem_per_block_dynamic",
    "nvltx__bytes.sum",
    "nvlrx__bytes.sum",
]


def main(rep, out):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    lines = [f"# ncu summary of {rep}", "# (ncu --set full --clock-control none; per launch)"]
    for r in rows[2:]:
        name = r[hdr.index("Kernel Name")] if "Kernel Name" in hdr else "?"
        lines.append(f"\n## {name[:150]}")
        for k in KEYS:
            if k in hdr:
                i = hdr.index(k)
                lines.append(f"{k:85s} {r[i]:>16s} {units[i]}")
        if "dram__bytes_read.sum" in hdr:
            def val(k):
                i = hdr.index(k)
                v = float(r[i].replace(",", ""))
                u = units[i].lower()
                return v * {"gbyte": 1e9, "mbyte": 1e6, "kbyte": 1e3, "byte": 1}.get(u, 1)
            t_i = hdr.index("gpu__time_duration.sum")
            t = float(r[t_i].replace(",", "")) * {"us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1}.get(units[t_i].lower(), 1e-6)
            tr = val("dram__bytes_read.sum") + val("dram__bytes_write.sum")
            lines.append(f"{'traffic = dram read + write (bytes)':85s} {tr:16.0f}")
            lines.append(f"{'dram GB/s under ncu clocks':85s} {tr / t / 1e9:16.1f}")
    open(out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
