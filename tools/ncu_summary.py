#!/usr/bin/env python3
"""Condense an `ncu --set full` report into the metrics DESIGN.md quotes.

    ncu -i x.ncu-rep --page raw --csv > x.csv
    python tools/ncu_summary.py x.csv > ncu_summary.json
"""
import csv
import json
import sys

KEEP = {
    "gpu__time_duration.sum": "duration_us",
    "smsp__inst_executed.sum": "warp_instructions",
    "sm__inst_executed.avg.per_cycle_elapsed": "ipc_per_sm_elapsed",
    "sm__issue_active.avg.pct_of_peak_sustained_elapsed": "issue_active_pct_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active": "issue_active_pct_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active": "pipe_fma_pct",
    "sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active": "pipe_alu_pct",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active": "pipe_xu_pct",
    "dram__bytes_read.sum": "dram_read",
    "dram__bytes_write.sum": "dram_write",
    "dram__throughput.avg.pct_of_peak_sustained_elapsed": "dram_throughput_pct",
    "lts__t_sector_hit_rate.pct": "l2_hit_pct",
    "l1tex__t_sector_hit_rate.pct": "l1_hit_pct",
    "launch__registers_per_thread": "registers",
    "launch__grid_size": "grid",
    "launch__block_size": "block",
    "launch__shared_mem_per_block_dynamic": "smem_dynamic",
    "launch__occupancy_limit_registers": "occ_limit_regs_blocks",
    "launch__occupancy_limit_shared_mem": "occ_limit_smem_blocks",
    "sm__cycles_active.avg": "sm_cycles_active_avg",
    "sm__cycles_elapsed.avg": "sm_cycles_elapsed_avg",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio": "stall_wait",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio": "stall_not_selected",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio": "stall_math_pipe",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio": "stall_long_scoreboard",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio": "stall_short_scoreboard",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio": "stall_barrier",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio": "stall_mio_throttle",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio": "stall_lg_throttle",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum": "smem_bank_conflicts",
}


def main():
    rows = list(csv.reader(open(sys.argv[1])))
    hdr, units = rows[0], rows[1]
    out = []
    for vals in rows[2:]:
        rec = {"kernel": vals[hdr.index("Kernel Name")].split("(")[0].replace("grb::<unnamed>::", "")}
        for i, h in enumerate(hdr):
            if h in KEEP:
                try:
                    v = float(vals[i].replace(",", ""))
                except ValueError:
                    continue
                u = units[i]
                if u in ("Mbyte",):
                    v *= 1e6
                elif u in ("Kbyte", "Kbyte/block"):
                    v *= 1e3
                elif u in ("Gbyte",):
                    v *= 1e9
                elif u == "ms":
                    v *= 1e3
                elif u == "ns":
                    v /= 1e3
                rec[KEEP[h]] = round(v, 4)
        if "dram_read" in rec and "dram_write" in rec:
            rec["dram_bytes"] = rec["dram_read"] + rec["dram_write"]
        out.append(rec)
    json.dump(out, sys.stdout, indent=1)
    print()


if __name__ == "__main__":
    main()
