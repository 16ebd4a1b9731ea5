"""Summarise an .ncu-rep into a small text table.
    python tools/ncu_summary.py prof.ncu-rep
"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem", "smsp__inst_executed.sum",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    print(f"# {path}  (ncu --set full --clock-control none; per-launch values, cold caches, serialised)")
    for r in rows[2:]:
        print("\n== " + r[idx["Kernel Name"]].split("(")[0] + f"   [launch id {r[idx['ID']]}]")
        for k in KEYS:
            if k in idx and r[idx[k]] not in ("", "n/a"):
                print(f"  {k:84s} {r[idx[k]]:>18s} {units[idx[k]]}")


if __name__ == "__main__":
    main(sys.argv[1])
