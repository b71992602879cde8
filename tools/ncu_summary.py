"""Summarise an .ncu-rep (ncu --set full) into the handful of numbers DESIGN/profiles quote.
usage: python tools/ncu_summary.py <capture>.ncu-rep > <name>.txt"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor.sum",
        "sm__pipe_tensor_subpipe_hmma_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size",
        "sm__cycles_active.avg", "smsp__inst_executed_pipe_xu.sum", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
        "lts__t_bytes.sum", "l1tex__data_bank_conflicts_pipe_lsu.sum", "smsp__cycles_active.avg",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__pipe_xu_cycles_active.avg.pct_of_peak_sustained_active"]


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    if len(rows) < 3:
        print(out[:2000])
        return
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        print("== %s  grid=%s block=%s" % (d.get("Kernel Name", "?")[:70], d.get("Grid Size"), d.get("Block Size")))
        for k in hdr:
            if any(k == key or k.startswith(key) for key in KEYS) or "tensor" in k and "pct" in k:
                u = units[hdr.index(k)]
                print("   %-80s %s %s" % (k, d[k], u))


if __name__ == "__main__":
    main()
