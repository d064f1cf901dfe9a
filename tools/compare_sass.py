#!/usr/bin/env python3
"""Compare the SASS of every kernel in two sets of object files, kernel by kernel (addresses and encodings included).

    tools/compare_sass.py --old old/a.o old/b.o --new new/c.o new/d.o [--rename old_kernel=new_kernel ...]

A kernel is identified by its mangled name without the anonymous-namespace tag (which embeds the file name), so a
kernel that moved to another translation unit is matched to itself.  Exit status 1 when a kernel of --old is missing
from --new or differs; kernels that only --new has are listed."""
import argparse
import re
import subprocess
import sys


def kernels(objs, renames):
    out = {}
    for obj in objs:
        text = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
        for part in re.split(r"^\s*Function : ", text, flags=re.M)[1:]:
            name, _, body = part.partition("\n")
            name = re.sub(r"(\d+)(_GLOBAL__N__\w+)", lambda m: m.group(2)[int(m.group(1)):], name.strip())
            for old, new in renames:
                name = name.replace(f"{len(old)}{old}", f"{len(new)}{new}")
            # cuobjdump pads its columns to the longest operand of the function's file: compare without the padding
            out[name] = re.sub(r"[ \t]+", " ", body.split("\nFatbin ")[0]).strip()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--old", nargs="+", required=True)
    ap.add_argument("--new", nargs="+", required=True)
    ap.add_argument("--rename", action="append", default=[], help="old=new, applied to the names of --old")
    a = ap.parse_args()
    old = kernels(a.old, [r.split("=") for r in a.rename])
    new = kernels(a.new, [])
    bad = 0
    for name in sorted(old):
        if name not in new:
            status = "MISSING"
        elif old[name] != new[name]:
            status = "DIFFERS"
        else:
            status = "identical"
        bad += status != "identical"
        print(f"{status:10s} {len(re.findall(r'^ ?/[*][0-9a-f]{4,}[*]/', old[name], flags=re.M)):6d} instr  {name}")
    for name in sorted(set(new) - set(old)):
        print(f"{'only new':10s} {'':6s}        {name}")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
