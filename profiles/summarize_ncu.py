#!/usr/bin/env python
"""Turn an .ncu-rep into a small text summary:  python profiles/summarize_ncu.py x.ncu-rep > x.txt"""
import csv
import io
import subprocess
import sys

WANT = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram__cycles_active.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
    "l1tex__throughput.avg.pct_of_peak_sustained_active",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
    "launch__shared_mem_per_block_dynamic", "launch__shared_mem_per_block_static",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    seen = {}
    for r in rows[2:]:
        name = r[idx["Kernel Name"]]
        seen.setdefault(name, []).append(r)
    print(f"# ncu summary of {path} (per kernel: launches captured, last launch shown)")
    for name, rs in seen.items():
        r = rs[-1]
        print(f"\n## {name}\nlaunches captured: {len(rs)}")
        for w in WANT:
            if w in idx:
                print(f"{w:90s} {r[idx[w]]} {units[idx[w]]}")
        try:
            t = float(r[idx["gpu__time_duration.sum"]])
            tu = units[idx["gpu__time_duration.sum"]]
            t_s = t * {"us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1.0}.get(tu.replace("second", "s").replace("usecond", "us"), 1e-6)
            rd = float(r[idx["dram__bytes_read.sum"]]); ru = units[idx["dram__bytes_read.sum"]]
            wr = float(r[idx["dram__bytes_write.sum"]]); wu = units[idx["dram__bytes_write.sum"]]
            sc = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0}
            traffic = rd * sc.get(ru, 1) + wr * sc.get(wu, 1)
            print(f"{'traffic = dram read + write':90s} {traffic:.4e} byte  ({traffic / t_s / 1e9:.0f} GB/s over the launch)")
        except Exception:
            pass


if __name__ == "__main__":
    main(sys.argv[1])
