"""Extract the roofline-relevant metrics of an ncu --set full report into a markdown table.

    ncu -i prof_X.ncu-rep --page raw --csv > x.csv ; python profiles/extract_ncu.py x.csv "title" > X.md
"""
import csv
import sys

KEEP = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__t_sector_hit_rate.pct", "lts__t_sectors_srcunit_tex_op_read.sum", "lts__t_sectors_srcunit_tex_op_write.sum",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size", "launch__block_size",
        "launch__cluster_size", "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
        "sm__cycles_elapsed.max", "smsp__inst_executed.sum", "sm__inst_executed_pipe_xu.sum", "smsp__inst_executed_pipe_xu.sum",
        "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_xu_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_fma.sum", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "smsp__cycles_active.avg",
        "sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active", "smsp__issue_active.avg.pct_of_peak_sustained_active"]


def main(path, title):
    rows = list(csv.reader(open(path)))
    hdr, units, data = rows[0], rows[1], rows[2:]
    print(f"# {title}\n")
    print("| metric | unit | " + " | ".join(f"launch {i}" for i in range(len(data))) + " |")
    print("|---|---|" + "---:|" * len(data))
    for i, k in enumerate(hdr):
        kk = k.split("TriageCompute.")[-1]
        if kk in KEEP:
            print(f"| {kk} | {units[i]} | " + " | ".join(r[i][:22] for r in data) + " |")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
