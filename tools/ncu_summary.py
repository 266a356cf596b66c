"""Summarise an ncu report (needs no GPU):  python tools/ncu_summary.py x.ncu-rep > x.txt"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__shared_mem_per_block_dynamic", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_elapsed",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        u = dict(zip(hdr, units))
        print("=" * 100)
        print("kernel:", d.get("Kernel Name"), " id", d.get("ID"))
        for k in KEYS:
            if k in d and d[k] != "":
                print(f"  {k:75s} {d[k]} {u.get(k, '')}")
        stalls = sorted(((float(v), k) for k, v in d.items() if k.startswith("smsp__average_warps_issue_stalled_") and
                         k.endswith("_per_issue_active.ratio") and v not in ("", "n/a")), reverse=True)[:6]
        print("  top warp-stall reasons (warps stalled per issue-active cycle):")
        for v, k in stalls:
            print(f"    {k.replace('smsp__average_warps_issue_stalled_', '').replace('_per_issue_active.ratio', ''):28s} {v:.3f}")


if __name__ == "__main__":
    main(sys.argv[1])
