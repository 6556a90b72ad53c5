#!/usr/bin/env python
"""Per-kernel SASS opcode histogram of libmm_b200.so (cuobjdump -sass): which kernels use the Hopper
tensor path (HGMMA = wgmma, UTMALDG/UTMASTG/UBLKCP = TMA) and which the warp-level one (HMMA = mma.sync) or
cp.async (LDGSTS).

    python tools/sass_histogram.py
"""
import re
import subprocess
import sys
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
LIB = ROOT / "models_b200" / "_lib" / "libmm_b200.so"
KEY = ["HGMMA", "UTMALDG", "UTMASTG", "UBLKCP", "HMMA", "LDSM", "LDGSTS", "LDG", "STG", "LDS", "STS", "SHFL",
       "MUFU", "BAR", "SYNCS", "ATOM", "RED"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", str(LIB)], capture_output=True, text=True).stdout
    kernels = {}
    cur = None
    for ln in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            kernels[cur] = Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", ln)
        if m and cur:
            kernels[cur][m.group(1)] += 1
    demangle = subprocess.run(["c++filt"], input="\n".join(kernels), capture_output=True, text=True).stdout.splitlines()
    print(f"# SASS opcode counts per kernel of {LIB.name} (static instruction counts; cuobjdump -sass, sm_90a)")
    print("# columns:", " ".join(KEY), "| total")
    for raw, name in sorted(zip(kernels, demangle), key=lambda kv: kv[1]):
        c = kernels[raw]
        short = re.sub(r"\(.*", "", name)
        print(f"{short[:96]:96s} " + " ".join(f"{c.get(k, 0):5d}" for k in KEY) + f" | {sum(c.values()):6d}")


if __name__ == "__main__":
    main()
