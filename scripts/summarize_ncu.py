"""Summarises an .ncu-rep (captured with `ncu --set full`) into a small text file: one block per kernel launch
with the metrics DESIGN.md / bench.py refer to.

    python scripts/summarize_ncu.py prof.ncu-rep summary.txt ["free-text note"]
"""
import csv
import io
import subprocess
import sys

METRICS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts_mem_lgds.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct", "sm__inst_executed.sum",
    "smsp__thread_inst_executed_per_inst_executed.ratio", "smsp__sass_average_branch_targets_threads_uniform.pct",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_membar_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    note = sys.argv[3] if len(sys.argv) > 3 else ""
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    with open(out, "w") as f:
        f.write(f"# {rep}\n# {note}\n# source: ncu --set full --clock-control none (one capture; per-launch values)\n\n")
        for d in data:
            f.write(d[hdr.index("Kernel Name")] + "\n")
            for m in METRICS:
                if m in hdr:
                    i = hdr.index(m)
                    f.write(f"    {m:88s} {d[i]:>20s} {units[i]}\n")
            f.write("\n")
    print("wrote", out)


if __name__ == "__main__":
    main()
