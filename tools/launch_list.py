"""Condense an `ncu --metrics gpu__time_duration.sum --csv --log-file X.csv` launch list into per-kernel count / total / share.

    python tools/launch_list.py launches.csv > launches_summary.txt
"""
import csv
import sys
from collections import OrderedDict


def main(path):
    rows = []
    with open(path, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    rd = csv.reader(lines)
    hdr = next(rd)
    ik, iv, iu, im = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit"), hdr.index("Metric Name")
    agg = OrderedDict()
    for r in rd:
        if len(r) <= iv or r[im] != "gpu__time_duration.sum":
            continue
        v = float(r[iv].replace(",", ""))
        u = r[iu]
        us = v * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(u, 1e-3)
        a = agg.setdefault(r[ik], [0, 0.0])
        a[0] += 1; a[1] += us
    tot = sum(a[1] for a in agg.values()) or 1.0
    print(f"# {path}: {sum(a[0] for a in agg.values())} launches, {tot:.1f} us of kernel time (cold-cache, serialised: compare SHARES, not absolutes)")
    for k, (n, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{k[:72]:72s} n={n:4d} total={t:9.1f}us avg={t / n:8.2f}us share={100 * t / tot:5.1f}%")


if __name__ == "__main__":
    main(sys.argv[1])
