#!/usr/bin/env python
"""Per-kernel totals and shares of an `ncu --metrics gpu__time_duration.sum --csv` launch list.
usage: launch_summary.py list.csv [first_kernel_of_a_step]   — with a step marker the last complete step is summarised as well."""
import csv
import sys
from collections import OrderedDict

rows = [r for r in csv.reader(open(sys.argv[1])) if len(r) > 5]
hdr = rows[0]
ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
seq = []
for r in rows[1:]:
    v = r[vi].replace(",", "")
    try:
        seq.append((r[ki].split("(")[0].replace("void ", "")[:70], float(v) / 1000.0))
    except ValueError:
        pass


def table(items, title):
    tot = sum(v for _, v in items)
    agg = OrderedDict()
    for k, v in items:
        a = agg.setdefault(k, [0, 0.0]); a[0] += 1; a[1] += v
    print(f"{title}: {len(items)} launches, {tot:.1f} us of kernel time (ncu: cold caches, serialised launches)")
    for k, (n, v) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print(f"  {v:9.1f} us  {100 * v / tot:5.1f} %  x{n:<4d} {k}")


table(seq, "whole capture")
if len(sys.argv) > 2:
    marks = [i for i, (k, _) in enumerate(seq) if sys.argv[2] in k]
    if len(marks) >= 2:
        table(seq[marks[-2]:marks[-1]], f"last complete step (from {sys.argv[2]} to the next)")
