"""Key metrics of every kernel in an ncu report.
    python tools/ncu_summary.py prof.ncu-rep > ncu_summary.txt
"""
import csv
import io
import subprocess
import sys

KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "smsp__thread_inst_executed_per_inst_executed.ratio", "sm__warps_active.avg.per_cycle_active",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "launch__shared_mem_per_block_static", "launch__occupancy_limit_shared_mem",
        "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor",
        "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "lts__t_sector_hit_rate.pct",
        "launch__grid_size", "launch__block_size"]


def main():
    rep = sys.argv[1]
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    head, units = rows[0], rows[1]
    col = {h: i for i, h in enumerate(head)}
    print("report: %s  (ncu --set full --clock-control none --import-source on, bench.py workload, steady state, 4096 bins)"
          % rep.split("/")[-1])
    for r in rows[2:]:
        print("  %-70s %s " % ("Kernel Name", r[col["Kernel Name"]]))
        for k in KEYS:
            if k in col:
                print("  %-70s %s %s" % (k, r[col[k]], units[col[k]]))
        print()


if __name__ == "__main__":
    main()
