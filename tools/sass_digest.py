#!/usr/bin/env python
"""Per-kernel SASS digest of libb200seg.so: which tensor / copy paths each kernel really uses.

    python tools/sass_digest.py > sass_digest.txt

Counts the Hopper mnemonics: HGMMA = wgmma, UTMALDG/UTMASTG/UBLKCP = TMA, HMMA = mma.sync, LDGSTS = cp.async."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "pytorchdeeplearing_b200", "csrc", "libb200seg.so")
PAT = {"HGMMA(wgmma)": r"\bHGMMA\b",
       "UTMALDG(TMA load)": r"\bUTMALDG\b", "UTMASTG(TMA store)": r"\bUTMASTG\b", "UBLKCP(bulk copy)": r"\bUBLKCP\b",
       "HMMA(mma.sync)": r"\bHMMA\b", "LDGSTS(cp.async)": r"\bLDGSTS\b", "FFMA": r"\bFFMA\b", "DFMA/DADD": r"\bD(FMA|ADD|MUL)\b"}

out = subprocess.run(["cuobjdump", "-sass", LIB], stdout=subprocess.PIPE, text=True, check=True).stdout
kern, counts = None, collections.OrderedDict()
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        kern = m.group(1)
        counts[kern] = collections.Counter()
        continue
    if kern is None:
        continue
    for k, p in PAT.items():
        if re.search(p, line):
            counts[kern][k] += 1
dem = subprocess.run(["cu++filt"] + list(counts), stdout=subprocess.PIPE, text=True).stdout.splitlines() \
    if counts else []
names = {k: (d if d else k) for k, d in zip(counts, dem)}
print(f"SASS digest of {os.path.relpath(LIB, ROOT)} ({len(counts)} kernels, sm_90a)")
cols = list(PAT)
print(" | ".join(["kernel"] + cols))
tot = collections.Counter()
for k, c in counts.items():
    tot.update(c)
    nm = names[k].replace("(int)", "").replace("(bool)", "")
    nm = re.sub(r"\(.*$", "", nm).replace("b200seg::", "").replace("void ", "").replace("__nv_bfloat16", "bf16")
    print(" | ".join([nm[:70]] + [str(c.get(x, 0)) for x in cols]))
print(" | ".join(["TOTAL"] + [str(tot.get(x, 0)) for x in cols]))
