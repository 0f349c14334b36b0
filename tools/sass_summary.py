#!/usr/bin/env python
"""Instruction-mix evidence for the hand-written kernels: which SASS the peer / TMA / tensor-core paths compile to.

    python tools/sass_summary.py

Reads the in-tree extensions with ``cuobjdump -sass`` (works without a GPU).  Mnemonics that prove the Hopper paths:
``HGMMA`` = wgmma.mma_async, ``UTMALDG`` = cp.async.bulk.tensor, ``UBLKCP`` = cp.async.bulk, ``SYNCS`` = mbarrier,
``LDGMC`` / ``REDG``-style multimem = NVLS.
"""
import collections
import glob
import re
import subprocess
import sys

WANT = re.compile(r"^(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UBLKCP|SYNCS|LDGMC|LDG|STG|ATOMG|REDG|RED|MEMBAR|FENCE|ERRBAR|BAR|"
                  r"LDS|STS|NANOSLEEP|ELECT|R2UR|CCTL)")
KERNELS = ["rs_kernelIfLi8ELb0", "rs_kernelIfLi8ELb1", "rs_kernelI13__nv_bfloat16Li8ELb0", "rs_pipe_kernelIf",
           "rs_pipe_kernelI13__nv_bfloat16", "ag_kernelIfLi8ELb0ELb0", "ag_kernelIfLi8ELb1ELb0", "ffn_hw_kernelILi0ELb0",
           "ffn_hw_kernelILi1ELb0", "ffn_hw_kernelILi1ELb1"]


def main():
    for so in sorted(glob.glob("dear_pytorch_b200/_C*.so") + glob.glob("dear_pytorch_b200/_tc*.so")):
        sass = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
        fn, mix = None, collections.defaultdict(collections.Counter)
        for line in sass.splitlines():
            m = re.search(r"Function : (\S+)", line)
            if m:
                fn = m.group(1)
                continue
            m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]+)", line)
            if m and fn:
                op = m.group(1)
                if WANT.match(op):
                    mix[fn][op] += 1
        print("# %s" % so)
        for key in KERNELS:
            for fn in sorted(mix):
                if key in fn:
                    print("\n## %s" % fn)
                    for op, n in sorted(mix[fn].items(), key=lambda kv: (-kv[1], kv[0])):
                        print("%6d  %s" % (n, op))
        print()


if __name__ == "__main__":
    sys.exit(main())
