#!/usr/bin/env python
"""profiles/sass.txt: per-kernel opcode counts of the shipped libovb200.so (cuobjdump -sass) — the SASS evidence of the
FP64 tensor-core path (DMMA), cp.async (LDGSTS), the hardware-seeded pivot rsqrt (MUFU.RSQ64H) and of the absence of
wgmma / tensor-map TMA opcodes (wgmma has no FP64 kind). Runs without a GPU."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "open_vins_b200", "libovb200.so")
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
WATCH = ["DMMA.8x8x4", "DMMA.16x8x4", "DMMA.16x8x8", "DMMA.16x8x16", "DFMA", "DMUL", "DADD", "MUFU.RSQ64H", "MUFU.RCP64H", "LDGSTS", "UBLKCP", "SYNCS", "SHFL", "BAR", "LDS", "STS", "UTMALDG", "HGMMA", "IGMMA", "QGMMA"]
counts = collections.OrderedDict()
fn = None
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = m.group(1)
        counts[fn] = collections.Counter()
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)", line)
    if m and fn:
        op = m.group(1)
        for w in WATCH:
            if op == w or op.startswith(w + "."):
                counts[fn][w] += 1
                break
demangle = subprocess.run(["c++filt"], input="\n".join(counts.keys()), capture_output=True, text=True).stdout.splitlines()
with open(os.path.join(ROOT, "profiles", "sass.txt"), "w") as f:
    f.write("# SASS opcode counts per kernel of open_vins_b200/libovb200.so (cuobjdump -sass, sm_90a); regenerate: python tools/sass_listing.py\n")
    f.write("# DMMA.8x8x4 / .16x8x4 / .16x8x8 / .16x8x16 = mma.sync.m8n8k4 / m16n8k4 / m16n8k8 / m16n8k16 .f64 (FP64 tensor-core path); LDGSTS = cp.async; MUFU.RSQ64H = rsqrt.approx.f64 pivot seed.\n")
    f.write("# UBLKCP = cp.async.bulk (TMA engine, 1-D) + SYNCS = mbarrier ops: the packed Cholesky factor of k_cq_trsm. wgmma / tensor-map TMA opcodes\n# (HGMMA, IGMMA, QGMMA, UTMALDG): none — wgmma has no FP64 kind, and every other operand tile here is\n")
    f.write("# either register-resident or a few KB staged by cp.async (DESIGN.md §4).\n")
    for (fn, c), dm in zip(counts.items(), demangle):
        name = dm.split("(")[0]
        f.write(f"{name:60s} " + " ".join(f"{k}={c[k]}" for k in WATCH if c[k]) + "\n")
    tot = collections.Counter()
    for c in counts.values():
        tot.update(c)
    f.write("TOTAL " + " ".join(f"{k}={tot[k]}" for k in WATCH) + "\n")
print(open(os.path.join(ROOT, "profiles", "sass.txt")).read()[:3000])
