"""CPU box: per-kernel SASS evidence of what each kernel is built from (cuobjdump of the objects in d3feat_b200/build):
wgmma (HGMMA), TMA (UBLKCP / UTMALDG), legacy mma.sync (HMMA), cp.async (LDGSTS), mbarrier (SYNCS), registers.
Writes profiles/sass_summary.txt."""
import glob
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pat = ["HGMMA", "UBLKCP", "UTMALDG", "HMMA", "LDGSTS", "SYNCS", "ATOMG", "RED", "MUFU", "LDG", "STG", "LDS", "STS"]
out = ["# SASS mnemonic counts per kernel (cuobjdump -sass of d3feat_b200/build/*.o, sm_90a)",
       "# wgmma.mma_async -> HGMMA, cp.async.bulk (TMA) -> UBLKCP / UTMALDG, mma.sync -> HMMA, cp.async -> LDGSTS",
       "%-64s %5s " % ("kernel", "regs") + " ".join("%7s" % p for p in pat)]
for obj in sorted(glob.glob(os.path.join(ROOT, "d3feat_b200", "build", "*.o"))):
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    res = subprocess.run(["cuobjdump", "-res-usage", obj], capture_output=True, text=True).stdout
    regs = dict(re.findall(r"Function (\S+):\s*\n\s*REG:(\d+)", res))
    cur, counts = None, {}
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = dict.fromkeys(pat, 0)
            continue
        if cur is None:
            continue
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m:
            op = m.group(1)
            for p in pat:
                if op.startswith(p):
                    counts[cur][p] += 1
    out.append("## " + os.path.basename(obj))
    for fn, c in counts.items():
        dem = subprocess.run(["cu++filt", fn], capture_output=True, text=True).stdout.strip() or fn
        dem = re.sub(r"\(.*", "", dem.replace("(int)", "").replace("(bool)", "")).replace("void ", "").replace("d3f::", "").replace("(anonymous namespace)::", "")
        out.append("%-64s %5s " % (dem[:64], regs.get(fn, "?")) + " ".join("%7d" % c[p] for p in pat))
os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
open(os.path.join(ROOT, "profiles", "sass_summary.txt"), "w").write("\n".join(out) + "\n")
print("\n".join(l for l in out if "HGMMA" in l or "fused" in l or "tc_gemm" in l or l.startswith("#"))[:3000])
