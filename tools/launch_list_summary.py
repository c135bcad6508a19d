#!/usr/bin/env python
"""by-kernel summary of an `ncu --metrics gpu__time_duration.sum --csv` launch list:
   python tools/launch_list_summary.py out/x.csv "title" > x_by_kernel.txt"""
import collections
import csv
import sys

rows = list(csv.reader(open(sys.argv[1])))
hdr = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
H = rows[hdr]
ki, vi = H.index("Kernel Name"), H.index("Metric Value")
ui = H.index("Metric Unit")
agg = collections.OrderedDict()
tot = 0.0
n = 0
for r in rows[hdr + 2:]:
    if len(r) <= vi:
        continue
    t = float(r[vi].replace(",", ""))
    if r[ui] in ("ns", "nsecond"):
        t /= 1000.0
    elif r[ui] in ("ms", "msecond"):
        t *= 1000.0
    name = r[ki][:100]
    a = agg.setdefault(name, [0.0, 0])
    a[0] += t
    a[1] += 1
    tot += t
    n += 1
print(sys.argv[2] if len(sys.argv) > 2 else sys.argv[1])
for name, (t, c) in sorted(agg.items(), key=lambda kv: -kv[1][0]):
    print(f"{t:10.1f} us {c:5d}x {t / c:10.2f} us/launch {100 * t / tot:5.1f}%  {name}")
print(f"total {tot:.1f} us over {n} launches")
