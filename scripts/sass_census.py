#!/usr/bin/env python
"""Per-kernel SASS census of the shipped library: `cuobjdump -sass` of momentum_b200/lib/libmomentum_b200.so reduced to the mnemonics
that say which hardware path a kernel uses (HMMA = mma.sync tensor cores, HGMMA = wgmma, UTMALDG / UBLKCP = TMA
tensor / bulk copies, STL / LDL = local-memory spills) plus registers and instruction count. Runs without a GPU.

    python scripts/sass_census.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "momentum_b200", "lib", "libmomentum_b200.so")
WATCH = ["HMMA", "HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "FFMA", "FMUL", "FADD", "MUFU", "LOP3", "IADD3", "IMAD", "SHFL", "LDS", "STS",
         "LDG", "STG", "LDL", "STL", "BAR", "LDSM", "REDUX", "ATOM", "RED", "DFMA", "DADD", "DMUL", "F2F", "F2FP"]


def demangle(names):
    try:
        out = subprocess.run(["c++filt"] + names, capture_output=True, text=True, check=True).stdout.splitlines()
        return dict(zip(names, out))
    except Exception:  # noqa: BLE001
        return {n: n for n in names}


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    regs = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = m.group(1)
        m = re.search(r"REG:(\d+).*?SHARED:(\d+)", line)
        if m and cur:
            regs[cur] = (int(m.group(1)), int(m.group(2)))
    kernels = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)(\.[A-Z0-9_.]+)?", line)
        if m and cur:
            kernels[cur][m.group(1)] += 1
            kernels[cur]["_total"] += 1
    names = demangle(list(kernels))
    print(f"SASS census of {os.path.relpath(LIB, ROOT)} (cuobjdump -sass; sm_90a). Static instruction counts per kernel.")
    print("HMMA = mma.sync; HGMMA = wgmma (warpgroup tensor path); UTMALDG = TMA tensor copy; UBLKCP = cp.async.bulk; STL/LDL = spills.\n")
    for k, c in kernels.items():
        short = re.sub(r"\(anonymous namespace\)::", "", names[k])
        short = re.sub(r"\(.*", "", short)
        r = regs.get(k, ("?", "?"))
        print(f"{short}\n    instructions {c['_total']:6d}   registers {r[0]}   static smem {r[1]} B")
        shown = [f"{w} {c[w]}" for w in WATCH if c[w]]
        print("    " + ", ".join(shown))
    return 0


if __name__ == "__main__":
    sys.exit(main())
