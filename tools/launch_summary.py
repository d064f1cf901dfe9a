"""Summarises an `ncu --metrics gpu__time_duration.sum --csv` launch list: share of each kernel.
usage: python tools/launch_summary.py launches.csv "<header line>" """
import collections
import csv
import sys

rows = [r for r in csv.reader(open(sys.argv[1])) if len(r) > 5]
hdr = next(r for r in rows if "Kernel Name" in r)
kn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
tot, n = collections.Counter(), collections.Counter()
for r in rows:
    if r is hdr or r[kn] == "Kernel Name":
        continue
    try:
        v = float(r[mv].replace(",", ""))
    except ValueError:
        continue
    v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(r[mu], 1.0)
    name = r[kn].split("(")[0]
    tot[name] += v
    n[name] += 1
total = sum(tot.values())
if len(sys.argv) > 2:
    print(sys.argv[2])
for k, v in tot.most_common(24):
    print(f"{v / total * 100:6.2f}%  {v:11.1f} us  x{n[k]:3d}  {k[:110]}")
print(f"total {total / 1e3:.2f} ms over {sum(n.values())} launches")
