"""Prints a handful of ncu raw-page metrics (DRAM bytes, tensor-pipe and issue activity) from a .ncu-rep."""
import csv, subprocess, sys
rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units, data = rows[0], rows[1], rows[2:]
want = ["Kernel Name", "gpu__time_duration.sum", "sm__cycles_elapsed.max", "launch__grid_size", "launch__block_size",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
        "sm__inst_executed_pipe_uniform.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_lsu.sum", "smsp__warp_issue_stalled_long_scoreboard_per_warp_active.pct",
        "gpc__cycles_elapsed.max", "sm__cycles_active.avg"]
for w in want:
    for i, h in enumerate(hdr):
        if h == w:
            print("%-85s %-10s %s" % (h, units[i], " | ".join(r[i] for r in data)))
