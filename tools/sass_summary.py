#!/usr/bin/env python
"""Per-kernel SASS mnemonic counts of the built objects (gsplat_b200/build/*.o) -- which Hopper
features each kernel really uses: UBLKCP (1-D bulk TMA), SYNCS (mbarrier), REDG
(incl. the 128-bit REDG.E.ADD.F32x4 of the version-2 backward), MUFU, SHFL, VOTE, LDGMC / multimem (NVLS), ...

    python tools/sass_summary.py > out/sass_summary.txt
"""
import collections
import glob
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ["UBLKCP", "UTMALDG", "SYNCS", "REDG", "REDG.E.ADD.F32x4", "ATOMG", "ATOMS", "MUFU.EX2", "MUFU.RCP", "MUFU", "SHFL", "VOTE",
        "LDGMC", "STGMC", "REDUX", "CREDUX", "BAR.SYNC", "LDS", "STS", "LDG", "STG", "FFMA", "HMMA", "UTC", "LDL", "STL"]


def main():
    print("# SASS mnemonic counts per kernel (cuobjdump -sass of gsplat_b200/build/*.o, sm_90a); total = instructions")
    print("# kernel".ljust(72) + " total " + " ".join(k.rjust(7) for k in ("UBLKCP", "SYNCS", "REDG", "REDG.x4", "MUFU", "SHFL", "VOTE", "LDGMC", "LDL+STL")))
    for obj in sorted(glob.glob(os.path.join(ROOT, "gsplat_b200", "build", "*.o"))):
        txt = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
        cur, counts = None, collections.OrderedDict()
        for ln in txt.splitlines():
            m = re.search(r"Function : (\S+)", ln)
            if m:
                cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
                cur = re.sub(r"\(.*", "", cur)
                counts[cur] = collections.Counter()
                continue
            m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Za-z0-9_.]+)", ln)
            if m and cur:
                op = m.group(1)
                counts[cur]["total"] += 1
                for k in KEYS:
                    if op.startswith(k):
                        counts[cur][k] += 1
        print(f"## {os.path.basename(obj)}")
        for name, c in counts.items():
            if c["total"] < 40:
                continue
            row = [c["UBLKCP"], c["SYNCS"], c["REDG"], c["REDG.E.ADD.F32x4"], c["MUFU"], c["SHFL"], c["VOTE"], c["LDGMC"] + c["STGMC"], c["LDL"] + c["STL"]]
            print(name[:70].ljust(72) + f"{c['total']:6d} " + " ".join(str(v).rjust(7) for v in row))


if __name__ == "__main__":
    main()
