"""Opcode histogram per kernel of libsgb200.so from `cuobjdump -sass` (no GPU needed): which hardware paths each
kernel uses — bulk / tensor copies (UBLKCP, UTMALDG), cp.async (LDGSTS), mbarriers (SYNCS), warpgroup tensor-core
MMAs (HGMMA), legacy tensor path (HMMA).   usage: python tools/sass_summary.py [lib]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "semantic-gaussians_b200", "libsgb200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
KEY = ("FFMA", "FMUL", "FADD", "MUFU", "LDS", "STS", "LDG", "STG", "RED", "ATOM", "LDGSTS", "UBLKCP", "UTMALDG", "UTMASTG",
       "SYNCS", "BAR", "SHFL", "VOTE", "HGMMA", "WARPGROUP", "HMMA", "IMAD", "BRA")
kern, hist = None, {}
arch = None
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        kern = m.group(1)
        hist[kern] = collections.Counter()
        continue
    m = re.match(r"\s*arch = (\S+)", line)
    if m:
        arch = m.group(1)
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and kern:
        hist[kern][m.group(1)] += 1
print(f"# SASS opcode summary of {os.path.relpath(lib, ROOT)} ({arch}); static instruction counts per kernel")
demangle = subprocess.run(["c++filt"], input="\n".join(hist), capture_output=True, text=True).stdout.splitlines()
for name, pretty in zip(hist, demangle):
    h = hist[name]
    tot = sum(h.values())
    short = pretty.replace("(anonymous namespace)::", "").replace("void ", "")
    short = re.sub(r"\(.*", "", short).replace("sgb::", "")
    cols = " ".join(f"{k}={h[k]}" for k in KEY if h.get(k))
    print(f"{short[:70]:70s} total={tot:5d}  {cols}")
tot = collections.Counter()
for h in hist.values():
    tot.update(h)
print("\nwhole library:", " ".join(f"{k}={tot[k]}" for k in KEY if tot.get(k)))
