"""Per-kernel SASS instruction census of libb200whisper.so (cuobjdump -sass): which kernels are wgmma (HGMMA), which use TMA
(UTMALDG tensor loads, UBLKCP bulk copies, UBLKRED bulk reductions) and which are mma.sync (HMMA).  Needs no GPU.

    python tools/sass_census.py
"""
import os
import re
import subprocess
import sys
from collections import Counter, OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "faster_whisper_b200", "libb200whisper.so")
PATTERNS = OrderedDict([
    ("HGMMA (wgmma)", r"\bHGMMA"), ("UTMALDG (TMA tensor load)", r"\bUTMALDG"), ("UBLKCP (TMA bulk copy)", r"\bUBLKCP"),
    ("UBLKRED (TMA bulk reduce)", r"\bUBLKRED"), ("SYNCS (mbarrier)", r"\bSYNCS"), ("HMMA (mma.sync)", r"\bHMMA"), ("LDGSTS (cp.async)", r"\bLDGSTS"),
    ("RED/ATOM global", r"\b(RED|ATOMG|ATOM)\b"), ("total instructions", r"^\s+/\*[0-9a-f]{4,}\*/"),
])


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    kernels, cur = OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = Counter()
            continue
        if cur is None:
            continue
        for name, pat in PATTERNS.items():
            if re.search(pat, line):
                kernels[cur][name] += 1
    demangle = subprocess.run(["c++filt"], input="\n".join(kernels), capture_output=True, text=True).stdout.splitlines()
    print("SASS census of faster_whisper_b200/libb200whisper.so (sm_90a), one row per kernel; counts are static instruction counts\n")
    cols = list(PATTERNS)
    print("%-70s " % "kernel" + " ".join("%9s" % c.split(" ")[0][:9] for c in cols))
    for (mangled, cnt), name in zip(kernels.items(), demangle):
        short = re.sub(r"\(.*", "", name).replace("b2w::", "")[:70]
        print("%-70s " % short + " ".join("%9d" % cnt[c] for c in cols))
    print("\ncolumns: " + "; ".join(cols))


if __name__ == "__main__":
    sys.exit(main())
