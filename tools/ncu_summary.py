"""Summarise an .ncu-rep (raw page) into a small text table.
   python tools/ncu_summary.py x.ncu-rep > x.txt"""
import csv
import subprocess
import sys

WANT = [
    "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "gpu__time_duration.sum",
    "sm__cycles_elapsed.max", "smsp__inst_executed.sum", "sm__inst_executed_pipe_tensor.sum",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__average_warp_latency_per_inst_issued.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
]


def main(path):
    out = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    ki = hdr.index("Kernel Name")
    print("# source: %s (ncu --set full --clock-control none --cache-control none; one block per launch)" % path)
    for r in rows[2:]:
        print("kernel: %s" % r[ki])
        for w in WANT:
            if w in hdr:
                i = hdr.index(w)
                print("  %-88s %s %s" % (w, r[i], units[i]))
        print()


if __name__ == "__main__":
    main(sys.argv[1])
