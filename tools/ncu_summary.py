#!/usr/bin/env python
"""Summarise `ncu --set full` reports (read here, no GPU needed): per captured launch the duration, DRAM bytes, the pipe
utilisation that names the saturated pipe, issue activity, occupancy and the warp-stall breakdown.
usage: python tools/ncu_summary.py rep1.ncu-rep [rep2.ncu-rep ...] > summary.txt"""
import csv
import io
import re
import subprocess
import sys

KEYS = [
    ("gpu__time_duration.sum", "duration"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("launch__registers_per_thread", "registers/thread"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "achieved occupancy %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput %"),
    ("sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_elapsed", "pipe fmaheavy (IMAD/IMAD.WIDE) cycles active %"),
    ("sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "pipe fma cycles active %"),
    ("sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active", "pipe alu cycles active %"),
    ("sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "pipe fp64 cycles active %"),
    ("sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "pipe lsu inst %"),
    ("smsp__issue_active.avg.pct_of_peak_sustained_active", "issue slots active %"),
    ("smsp__inst_executed.sum", "warp instructions"),
    ("smsp__thread_inst_executed_per_inst_executed.ratio", "active threads / warp inst"),
    ("l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "shared-memory bank conflicts"),
    ("l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "shared-memory wavefronts"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram throughput %"),
    ("lts__t_sector_hit_rate.pct", "L2 hit rate %"),
]
STALL = re.compile(r"smsp__average_warps_issue_stalled_(\w+)_per_issue_active\.ratio")


def main():
    for path in sys.argv[1:]:
        raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(io.StringIO(raw)))
        hdr, units, data = rows[0], rows[1], rows[2:]
        col = {h: i for i, h in enumerate(hdr)}
        print("== %s" % path.split("/")[-1])
        for r in data:
            print("-- %s  grid %s block %s" % (r[col["Kernel Name"]][:90], r[col.get("Grid Size", 0)], r[col.get("Block Size", 0)]))
            for k, label in KEYS:
                if k in col:
                    print("   %-48s %s %s" % (label, r[col[k]], units[col[k]]))
            stalls = sorted(((float(r[i]), STALL.match(h).group(1)) for h, i in col.items() if STALL.match(h) and r[i] not in ("", "n/a")), reverse=True)
            print("   warp stalls per issue (top): " + ", ".join("%s %.2f" % (n, v) for v, n in stalls[:6]))
        print()


if __name__ == "__main__":
    main()
