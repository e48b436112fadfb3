#!/usr/bin/env python
"""Per-kernel SASS opcode summary of the product library (cuobjdump -sass): total instructions and the counts of the
mnemonics that show which hardware path a kernel uses (UTMALDG / UBLKCP = TMA, SYNCS = mbarrier,
LDGSTS = cp.async, R2P = register-to-predicates).  usage: sass_summary.py lib.so > out.txt"""
import collections
import re
import subprocess
import sys

KEY = ["UTMALDG", "UBLKCP", "SYNCS", "LDGSTS", "R2P", "LDG", "STG", "LDS", "STS", "ATOMS", "ATOMG", "RED", "SHFL", "REDUX", "MUFU", "BAR", "UCGABAR"]
out = subprocess.run(["cuobjdump", "-sass", sys.argv[1]], capture_output=True, text=True).stdout
kern, cur = collections.OrderedDict(), None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = collections.Counter()
        kern[m.group(1)] = cur
        continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and cur is not None:
        cur["_total"] += 1
        cur[m.group(1)] += 1
dem = subprocess.run(["c++filt"], input="\n".join(kern), capture_output=True, text=True).stdout.splitlines()
print(f"{'kernel':70s} {'instr':>6s} " + " ".join(f"{k:>7s}" for k in KEY))
for (name, c), d in zip(kern.items(), dem):
    short = re.sub(r"\(.*", "", d).replace("void ", "")
    print(f"{short[:70]:70s} {c['_total']:6d} " + " ".join(f"{c[k]:7d}" for k in KEY))
