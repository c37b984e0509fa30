"""Compact text summary of an .ncu-rep (needs no GPU): python scripts/ncu_summary.py rep... > summary.txt"""
import csv
import subprocess
import sys

EXACT = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__cluster_size",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
    "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "l1tex__m_xbar2l1tex_read_bytes.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active",
    "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
    "sm__cycles_elapsed.avg", "sm__cycles_active.avg",
    "smsp__inst_executed.sum",
]


def main():
    for rep in sys.argv[1:]:
        out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
        rows = list(csv.reader(out.splitlines()))
        if len(rows) < 3:
            print(f"# {rep}: no data")
            continue
        hdr, units = rows[0], rows[1]
        col = {h: i for i, h in enumerate(hdr)}
        print(f"# {rep}  (ncu --set full --clock-control none; one replayed launch per row)")
        for r in rows[2:]:
            print(f"kernel: {r[col['Kernel Name']]}")
            for m in EXACT:
                if m in col and r[col[m]] != "":
                    print(f"  {m:95s} {r[col[m]]} {units[col[m]]}")
            # every tensor-op path that is actually used
            for h, i in col.items():
                if h.startswith("sm__ops_path_tensor_op_") and h.endswith(".avg.pct_of_peak_sustained_elapsed"):
                    try:
                        if float(r[i]) > 0:
                            print(f"  {h:95s} {r[i]} {units[i]}")
                    except ValueError:
                        pass
            print()


if __name__ == "__main__":
    main()
