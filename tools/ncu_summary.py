#!/usr/bin/env python3
"""Condense an .ncu-rep (ncu --set full) into the handful of numbers a kernel study quotes.
usage: python tools/ncu_summary.py x.ncu-rep [n_symbols_per_launch bytes_per_symbol]"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__bytes_read.sum.per_second",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_pipe_lsu_wavefronts.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_registers",
    "launch__occupancy_limit_shared_mem", "smsp__cycles_active.avg", "sm__cycles_elapsed.avg",
]
STALLS = "smsp__pcsamp_warps_issue_stalled_"


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        u = dict(zip(hdr, units))
        print(f"## {d.get('Kernel Name', '?')}  grid {d.get('Grid Size')} block {d.get('Block Size')}")
        for k in KEYS:
            if k in d:
                print(f"{k:75s} {d[k]:>18s} {u[k]}")
        st = sorted(((float(v), k[len(STALLS):]) for k, v in d.items() if k.startswith(STALLS) and not k.endswith("_not_issued") and v), reverse=True)
        tot = sum(v for v, _ in st) or 1.0
        print("stall samples (pc sampling): " + ", ".join(f"{n} {100 * v / tot:.0f}%" for v, n in st[:7]))
        if len(sys.argv) >= 4:
            n, b = float(sys.argv[2]), float(sys.argv[3])
            t = float(d["gpu__time_duration.sum"]) * {"us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1}[u["gpu__time_duration.sum"]]
            tr = float(d["dram__bytes_read.sum"]) * {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1}[u["dram__bytes_read.sum"]] + \
                float(d["dram__bytes_write.sum"]) * {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1}[u["dram__bytes_write.sum"]]
            print(f"algorithmic bytes/launch {n * b:.4g}  dram traffic/launch {tr:.4g}  ratio {tr / (n * b):.3f}  "
                  f"(under ncu, cold: {n * b / t / 1e9:.0f} GB/s algorithmic)")
            wf = d.get("l1tex__data_pipe_lsu_wavefronts.sum") or "nan"
            print(f"warp instructions per symbol {float(d['smsp__inst_executed.sum']) / n:.0f}; "
                  f"LSU wavefronts per symbol {float(wf) / n:.0f}; "
                  f"shared-memory wavefronts per symbol {float(d['l1tex__data_pipe_lsu_wavefronts_mem_shared.sum']) / n:.0f}")


if __name__ == "__main__":
    main()
