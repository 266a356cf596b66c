"""Aggregate an `ncu --metrics gpu__time_duration.sum --csv` launch list per kernel (needs no GPU):
  python tools/launch_summary.py launches.csv "header line" > launch_list_summary.txt"""
import csv
import re
import sys


def family(name):
    if "gemm" in name:
        return "gemm"
    if "attention" in name:
        return "attention"
    if "norm_kernel" in name:
        return "norm"
    return "other"


def main(path, header):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    hdr = rows[0]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg, fam, total = {}, {}, 0.0
    for r in rows[1:]:
        name = re.sub(r"\(.*", "", r[ki])
        us = float(r[vi].replace(",", "")) / (1e3 if r[ui] in ("ns", "nsecond") else 1.0)
        n, t = agg.get(name, (0, 0.0))
        agg[name] = (n + 1, t + us)
        fam[family(name)] = fam.get(family(name), 0.0) + us
        total += us
    print(header)
    for name, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{100 * t / total:6.2f}%  {n:5d} launches  {t:12.1f} us  avg {t / n:9.1f} us  {name}")
    print("family shares: " + ", ".join(f"{k} {100 * v / total:.1f}%" for k, v in sorted(fam.items(), key=lambda kv: -kv[1])))
    print(f"total {total / 1e3:.1f} ms over {sum(n for n, _ in agg.values())} launches")


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "")
