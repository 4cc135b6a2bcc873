#!/usr/bin/env python
"""Instruction counts of the device functions inside rdo_batch_kernel (nvdisasm of the sm_90a cubin of tb_rdo.cu), as markdown: the RD loop is bound by instruction
delivery, so the size of what each phase streams from L2 is the quantity to watch.  Usage: python tools/rdo_code_size.py [out.md]"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "thor_b200", "libthor_b200.so")


def main():
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run(["cuobjdump", "-xelf", "all", LIB], cwd=tmp, capture_output=True)
        cubin = [f for f in os.listdir(tmp) if f.startswith("tb_rdo") and f.endswith(".cubin")]
        assert cubin, "no tb_rdo cubin in %s" % LIB
        out = subprocess.run(["nvdisasm", "-c", os.path.join(tmp, cubin[0])], capture_output=True, text=True).stdout
    counts, name = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"^(\$?_Z\S*):$", line)
        if m:
            name = m.group(1)
            counts[name] = 0
        elif name and re.match(r"^\s+/\*[0-9a-f]+\*/", line):
            counts[name] += 1
    rows = {"unsigned char": [], "unsigned short": []}
    for sym, n in counts.items():  # the translation unit holds only the two instantiations of the RD kernel
        parts = sym.split("$")
        dem = subprocess.run(["c++filt", parts[-1] if parts[-1] else sym], capture_output=True, text=True).stdout.strip()
        dem = dem.replace("(anonymous namespace)::", "").replace("tb_rdo_tu::", "")
        kern = "unsigned short" if "kernelIt" in sym else "unsigned char"
        dem = re.sub(r"\(.*", "", dem)
        dem = re.sub(r"Rdo<unsigned (char|short), DevBackend<unsigned (char|short)> >", "Rdo", dem)
        rows[kern].append((n, dem))
    lines = ["# Device functions of rdo_batch_kernel by size (`nvdisasm` of tb_rdo.cu's sm_90a cubin; SASS instructions, 16 bytes each)", "",
             "An all-inlined build is several MB of SASS.  Every function of the control flow and of the backend exists",
             "once per kernel (`__noinline__`), the per-sample loops are rolled, the small transform chains are loops.", ""]
    for kern, r in rows.items():
        r.sort(reverse=True)
        tot = sum(n for n, _ in r)
        lines += ["## `rdo_batch_kernel<%s>`: %d instructions (%.0f KB) in %d functions" % (kern, tot, tot * 16 / 1024, len(r)), "", "| instructions | function |", "|---|---|"]
        lines += ["| %d | `%s` |" % (n, d[:110]) for n, d in r if n >= 150]
        lines.append("")
    text = "\n".join(lines)
    if len(sys.argv) > 1:
        open(sys.argv[1], "w").write(text)
    else:
        print(text)


if __name__ == "__main__":
    main()
