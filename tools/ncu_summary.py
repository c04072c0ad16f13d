"""Turns `ncu -i <rep> --page raw --csv` output into a short metric list.

    ncu -i profile_out/x.ncu-rep --page raw --csv > profile_out/x_raw.csv
    python tools/ncu_summary.py profile_out/x_raw.csv [kernel-name-substring] > profile_out/x_summary.txt
"""
import csv
import sys

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__occupancy_limit_shared_mem",
    "launch__occupancy_limit_registers", "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
    "smsp__inst_executed.sum", "sm__cycles_active.avg",
]
STALL = "smsp__average_warps_issue_stalled_"


def main():
    rows = list(csv.reader(open(sys.argv[1])))
    want = sys.argv[2] if len(sys.argv) > 2 else ""
    hdr = next(r for r in rows if r and r[0] == "ID")
    units = rows[rows.index(hdr) + 1]
    for r in rows[rows.index(hdr) + 2:]:
        d = dict(zip(hdr, r))
        if want and want not in d.get("Kernel Name", ""):
            continue
        u = dict(zip(hdr, units))
        print("# kernel:", d.get("Kernel Name", "?")[:120])
        for k in hdr:
            if k in KEEP or (k.startswith(STALL) and k.endswith("_per_issue_active.ratio")):
                print(k, d[k], u.get(k, ""))
        break


if __name__ == "__main__":
    main()
