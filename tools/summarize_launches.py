#!/usr/bin/env python
"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: per-kernel count, total
device time and share.  usage: tools/summarize_launches.py launches.csv"""
import collections
import csv
import re
import sys


def main(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    agg = collections.OrderedDict()
    for x in csv.DictReader(lines):
        name = re.sub(r"\(.*", "", x["Kernel Name"])[:90]
        v = float(x["Metric Value"].replace(",", ""))
        v *= {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "nsecond": 1e-3}.get(x["Metric Unit"], 1.0)
        a = agg.setdefault(name, [0, 0.0, x["Grid Size"], x["Block Size"]])
        a[0] += 1
        a[1] += v
    tot = sum(v[1] for v in agg.values())
    print(f"# {path}: {sum(v[0] for v in agg.values())} launches, {tot/1e3:.3f} ms total device time (cold-cache, serialised: compare SHARES)")
    print(f"# {'total_us':>12s} {'count':>5s} {'avg_us':>10s} {'share':>6s}  kernel (grid, block of last launch)")
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"{v[1]:14.1f} {v[0]:5d} {v[1]/v[0]:10.1f} {100*v[1]/tot:5.1f}%  {k}  grid={v[2]} block={v[3]}")


if __name__ == "__main__":
    main(sys.argv[1])
