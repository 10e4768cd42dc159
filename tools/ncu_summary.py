"""Summarise one kernel of an .ncu-rep (needs only the ncu CLI, no GPU): python tools/ncu_summary.py report.ncu-rep [title]"""
import csv, subprocess, sys

rep = sys.argv[1]
out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr, vals = rows[0], rows[-1]
d = dict(zip(hdr, vals))
KEYS = ["Kernel Name", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "gpu__time_duration.sum", "sm__cycles_elapsed.avg.per_second",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_subpipe_imma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor_subpipe_dmma.avg.pct_of_peak_sustained_active",
        "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "lts__t_sector_hit_rate.pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__pipe_tma_cycles_active.avg.pct_of_peak_sustained_active"]
if len(sys.argv) > 2:
    print(sys.argv[2])
for k in KEYS:
    if k in d:
        print(f"{k:90s} {d[k]}")
# units row (second row) for the byte counters
units = dict(zip(hdr, rows[1])) if len(rows) > 2 else {}
for k in ("dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum"):
    if k in units:
        print(f"unit[{k}] = {units[k]}")
