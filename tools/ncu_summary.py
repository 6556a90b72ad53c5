#!/usr/bin/env python
"""Summarise an .ncu-rep (raw page) into a handful of DRAM / issue metrics.

    python tools/ncu_summary.py prof.ncu-rep [pattern ...]
"""
import csv
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput",
        "sm__throughput.avg.pct", "sm__warps_active.avg.pct_of_peak", "launch__registers_per_thread",
        "launch__occupancy_limit", "sm__pipe_tensor", "sm__inst_executed_pipe_tensor", "smsp__inst_executed.sum",
        "l1tex__t_requests_pipe_lsu_mem_global_op_st.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum",
        "l1tex__t_requests_pipe_lsu_mem_global_op_ld.sum", "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared", "smsp__warp_issue_stalled", "lts__t_sector_hit_rate",
        "sm__cycles_elapsed.max", "smsp__cycles_active.avg", "launch__shared_mem_per_block", "launch__grid_size",
        "smsp__issue_active.avg.pct", "sm__inst_executed_pipe_lsu", "dram__cycles_active", "l1tex__lsu_writeback",
        "smsp__average_warps_issue_stalled", "sm__inst_executed_pipe_fma", "sm__inst_executed_pipe_alu"]


def main():
    rep = sys.argv[1]
    pats = sys.argv[2:] or KEYS
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        print("==", r[hdr.index("Kernel Name")][:90], "grid", r[hdr.index("Grid Size")], "block", r[hdr.index("Block Size")])
        for i, h in enumerate(hdr):
            if any(p in h for p in pats):
                v = r[i]
                if v in ("", "0", "n/a"):
                    continue
                print(f"   {h.split('.', 2)[-1] if h.count('.') > 2 and h.split('.')[1].startswith('Triage') else h:90s} {v} {units[i]}")


if __name__ == "__main__":
    main()
