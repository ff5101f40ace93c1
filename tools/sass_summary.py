"""Opcode histogram per kernel of libcelebbasis_b200.so (cuobjdump -sass): which tensor-core and copy paths each kernel uses
(HGMMA = wgmma.mma_async, UTMALDG = TMA tensor load, UBLKCP = cp.async.bulk, SYNCS = mbarrier;
HMMA would be the legacy mma.sync path).  Writes profiles/sass_summary.txt.

    python tools/sass_summary.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "celebbasis_b200", "libcelebbasis_b200.so")
KEY = ["HGMMA", "WARPGROUP", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "UTCBAR", "UTCATOM",
       "HMMA", "IMMA", "MUFU", "REDG", "RED", "ATOMG", "ATOM", "LDG", "STG", "LDS", "STS", "BAR", "ACQBULK", "ELECT"]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    per = collections.OrderedDict()
    cur = None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            per[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)", line)
        if m and cur is not None:
            per[cur][m.group(1)] += 1
    demangle = subprocess.run(["c++filt"], input="\n".join(per.keys()), capture_output=True, text=True).stdout.splitlines()
    total = collections.Counter()
    lines = []
    for (name, cnt), dn in zip(per.items(), demangle):
        total.update(cnt)
        short = re.sub(r"\(.*", "", dn)
        short = short.replace("void ", "")
        hot = " ".join(f"{k}={cnt[k]}" for k in KEY if cnt.get(k))
        lines.append(f"{short[:110]:110s} instr={sum(cnt.values()):6d}  {hot}")
    hdr = [f"# cuobjdump -sass {os.path.relpath(LIB, ROOT)}  ({len(per)} kernels, sm_90a)",
           "# totals: " + " ".join(f"{k}={total[k]}" for k in KEY if total.get(k)),
           "# HGMMA (wgmma.mma_async), UTMALDG (cp.async.bulk.tensor), UBLKCP (cp.async.bulk), SYNCS (mbarrier); "
           "HMMA (legacy mma.sync) must be absent", ""]
    text = "\n".join(hdr + sorted(lines)) + "\n"
    dst = os.path.join(ROOT, "profiles", "sass_summary.txt")
    with open(dst, "w") as f:
        f.write(text)
    print("\n".join(hdr[:3]))
    print(f"wrote {dst}")


if __name__ == "__main__":
    sys.exit(main())
