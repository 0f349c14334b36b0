#!/usr/bin/env python
"""Registers / shared memory / spills per kernel family of the built extensions (cuobjdump --dump-resource-usage; no GPU
needed).  `python tools/resource_usage.py`"""
import collections
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.split("\n")
    return dict(zip(names, out))


def main():
    for so in sorted(glob.glob(os.path.join(ROOT, "dear_pytorch_b200", "_*.so"))):
        txt = subprocess.run(["cuobjdump", "--dump-resource-usage", so], capture_output=True, text=True).stdout
        fams = collections.OrderedDict()
        names, rows = [], []
        cur = None
        for line in txt.split("\n"):
            m = re.match(r"\s*Function (\S+):", line)
            if m:
                cur = m.group(1)
                continue
            m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+) LOCAL:(\d+)", line)
            if m and cur:
                names.append(cur)
                rows.append((cur,) + tuple(int(x) for x in m.groups()))
                cur = None
        dm = demangle(names)
        for name, reg, stack, shared, local in rows:
            fam = re.sub(r"<.*", "", re.sub(r"\(.*", "", dm.get(name, name)).replace("void ", "")).strip()
            f = fams.setdefault(fam, {"n": 0, "reg": [], "stack": 0, "shared": set(), "local": 0})
            f["n"] += 1
            f["reg"].append(reg)
            f["stack"] = max(f["stack"], stack)
            f["local"] = max(f["local"], local)
            f["shared"].add(shared)
        print("== %s (sm_90a)" % os.path.basename(so))
        print("%-34s %5s %9s %14s %6s %6s" % ("kernel family", "inst.", "regs", "static smem B", "stack", "local"))
        for fam, f in fams.items():
            regs = "%d" % f["reg"][0] if min(f["reg"]) == max(f["reg"]) else "%d-%d" % (min(f["reg"]), max(f["reg"]))
            sh = ",".join(str(s) for s in sorted(f["shared"]))
            print("%-34s %5d %9s %14s %6d %6d" % (fam[:34], f["n"], regs, sh[:14], f["stack"], f["local"]))
        print()


if __name__ == "__main__":
    sys.exit(main())
