#!/usr/bin/env python
"""SASS opcode histogram per kernel of thor_b200/libthor_b200.so (cuobjdump -sass), written as markdown.
Usage: python tools/sass_hist.py [out.md]   (VERDICT r1 item 1e: evidence of which instructions the kernels are made of)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "thor_b200", "libthor_b200.so")
INTEREST = ["VABSDIFF4", "IDP.4A", "IDP.2A", "IDP", "IMAD", "LDG", "LDS", "STS", "STG", "SHFL", "BAR", "UTMALDG", "UBLKCP", "SYNCS", "HMMA", "IMMA", "DMUL", "DADD", "DFMA",
            "ATOM", "RED", "LDL", "STL", "I2IP", "VOTE", "MATCH"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    kernels, cur = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = cur.replace("(anonymous namespace)::", "")
            cur = re.sub(r"\(.*", "", cur)
            kernels[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    rows = []
    for k, c in kernels.items():
        total = sum(c.values())
        agg = collections.Counter()
        for op, n in c.items():
            for key in INTEREST:
                if op == key or op.startswith(key + "."):
                    agg[key] += n
                    break
        rows.append((total, k, agg))
    rows.sort(reverse=True)
    cols = ["VABSDIFF4", "IDP.4A", "IDP.2A", "IMAD", "LDG", "LDS", "STS", "SHFL", "BAR", "LDL", "STL", "DMUL", "DADD", "UTMALDG", "UBLKCP", "IMMA", "HMMA"]
    lines = ["# SASS opcode histogram per kernel (`cuobjdump -sass thor_b200/libthor_b200.so`, sm_90a)", "",
             "Static instruction counts (not executed counts).  LDL/STL = local-memory (spill or per-thread array) accesses; UTMALDG/UBLKCP = TMA bulk copies;",
             "IMMA/HMMA = mma.sync tensor-core ops.", "",
             "| kernel | SASS instrs | " + " | ".join(cols) + " |", "|---|---|" + "---|" * len(cols)]
    for total, k, agg in rows:
        if total < 50:
            continue
        lines.append("| `%s` | %d | " % (k[:90], total) + " | ".join(str(agg.get(c, 0)) for c in cols) + " |")
    text = "\n".join(lines) + "\n"
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(text)
    else:
        print(text)


if __name__ == "__main__":
    main()
