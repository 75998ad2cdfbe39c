#!/usr/bin/env python
"""Register / stack / spill table of every kernel in libb2b.so from the -Xptxas -v logs the Makefile keeps
(csrc/*.o.ptxas.log):  python tools/ptxas_table.py"""
import glob
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
rows = []
for log in sorted(glob.glob(os.path.join(ROOT, "bijectors.jl_b200", "csrc", "*.ptxas.log"))):
    name = None
    stack = st = ld = 0
    for line in open(log):
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            stack, st, ld = map(int, m.groups())
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            rows.append((name, int(m.group(1)), stack, st, ld))
            name = None
names = subprocess.run(["cu++filt"] + [r[0] for r in rows], capture_output=True, text=True).stdout.splitlines()
print("# -Xptxas -v of every kernel in libb2b.so registers / stack frame / spill stores / spill loads (bytes)")
out = []
for (mangled, regs, stack, st, ld), dn in zip(rows, names):
    dn = re.sub(r"\(.*$", "", dn.replace("void ", "").replace("b2b::", "").replace("(int)", "").replace("(bool)", ""))
    out.append(f"{dn:100s} regs {regs:3d}  stack {stack:4d}  spill_st {st:4d}  spill_ld {ld:4d}")
print("\n".join(sorted(out)))
