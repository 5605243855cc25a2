"""Per-kernel SASS mnemonic counts of the in-tree engine library (evidence that the wgmma / TMA paths are the ones
compiled in).  No GPU needed:

    python tests/sass_summary.py
"""
from __future__ import annotations

import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "whisper_medusa_b200", "_lib", "libwm_b200.so")
WATCH = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UTMAPF", "UBLKCP", "SYNCS", "HMMA",
         "LDGSTS", "LDSM", "REDG", "ATOMG", "MEMBAR", "ERRBAR", "CCTL", "BAR", "UCGABAR", "MUFU", "LDG", "STG", "LDS", "STS"]


def demangle(name: str) -> str:
    try:
        return subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip() or name
    except Exception:  # noqa: BLE001
        return name


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    kernels = collections.OrderedDict()
    cur = None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m:
            op = m.group(1)
            kernels[cur]["_total"] += 1
            for w in WATCH:
                if op == w or op.startswith(w):
                    kernels[cur][w] += 1
                    break
    print(f"# cuobjdump -sass {os.path.relpath(LIB, ROOT)}: instruction counts per kernel (static), sm_90a")
    print("# wgmma = HGMMA (MMA) / WARPGROUP (arrive, depbar); TMA tensor copies = UTMALDG / UTMASTG;")
    print("# bulk (non-tensor) async copies = UBLKCP; mbarrier = SYNCS; legacy tensor-core MMA = HMMA; cp.async = LDGSTS")
    for k, c in kernels.items():
        name = demangle(k)
        name = re.sub(r"\(.*", "", name)
        cols = "  ".join(f"{w}={c[w]}" for w in WATCH if c[w])
        print(f"{name:<60} total={c['_total']:<6} {cols}")


if __name__ == "__main__":
    sys.exit(main())
