"""SASS evidence per kernel: counts of the Hopper tensor-core / TMA / legacy mnemonics in the shipped library.

    python profiles/sass_summary.py      (needs cuobjdump + c++filt; no GPU)

HGMMA = wgmma, WARPGROUP = wgmma fence / arrive, UTMALDG = TMA tensor load, HMMA = legacy
mma.sync, LDGSTS = cp.async, SYNCS = mbarrier ops, ELECT = elect.sync (single-lane issue from a converged warp)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "propainter_b200", "libpropainter_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
cols = ["HGMMA", "WARPGROUP", "UTMALDG", "HMMA", "LDGSTS", "SYNCS", "ELECT"]
rows = []
for f in re.split(r"\n\s*Function : ", txt)[1:]:
    cnt = collections.Counter(m.group(1) for m in re.finditer(r"\b(" + "|".join(cols) + r")\b", f))
    rows.append((f.split("\n", 1)[0].strip(), cnt))
names = subprocess.run(["c++filt"] + [r[0] for r in rows], capture_output=True, text=True).stdout.split("\n")
print(f"# {os.path.relpath(lib, ROOT)}: SASS mnemonic counts per kernel (profiles/sass_summary.py)")
print(f"{'kernel':44s} " + " ".join(f"{k:>8s}" for k in cols))
for (n, c), dn in zip(rows, names):
    if sum(c.values()):
        print(f"{re.sub(r'[(].*', '', dn)[:44]:44s} " + " ".join(f"{c.get(k, 0):8d}" for k in cols))
