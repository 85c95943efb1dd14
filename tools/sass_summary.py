#!/usr/bin/env python3
"""Per-kernel counts of the SASS mnemonics that show what a kernel is built on (TMA, wgmma, FP64 tensor cores,
integer dot products, SWAR byte ops, population counts) from `cuobjdump -sass alvaar_b200/libalva_b200.so`.
usage: python tools/sass_summary.py > profiles/sass_summary.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "alvaar_b200", "libalva_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
PAT = [("UTMALDG", r"UTMALDG"), ("UBLKCP", r"UBLKCP"), ("GMMA", r"[A-Z]*GMMA"),
       ("SYNCS(mbarrier)", r"SYNCS"), ("DMMA", r"DMMA"), ("IMMA", r"\bIMMA"), ("HMMA", r"HMMA"), ("IDP", r"\bIDP"), ("VABSDIFF4", r"VABSDIFF4"),
       ("VIMNMX*", r"VIMNMX"), ("POPC", r"\bPOPC"), ("LOP3", r"\bLOP3"), ("SHFL", r"\bSHFL"), ("REDUX", r"REDUX"), ("MATCH", r"\bMATCH"),
       ("DFMA", r"\bDFMA"), ("FFMA", r"\bFFMA")]
kern, rows, name = None, [], None
counts, total = collections.Counter(), 0
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        if name:
            rows.append((name, total, dict(counts)))
        name = subprocess.run(["c++filt", "-p", m.group(1)], capture_output=True, text=True).stdout.strip() or m.group(1)
        name = re.sub(r"\(anonymous namespace\)::", "", name)
        counts, total = collections.Counter(), 0
        continue
    if re.match(r"\s+/\*[0-9a-f]{4,6}\*/", line):
        total += 1
        for k, p in PAT:
            if re.search(p, line):
                counts[k] += 1
if name:
    rows.append((name, total, dict(counts)))
print("# static SASS of", os.path.relpath(so, ROOT), "(sm_90a): instructions per kernel and the mnemonics that matter")
print("# UTMALDG / UBLKCP = TMA (tensor / bulk copies); IGMMA / QGMMA = wgmma (int8 / fp8) with register accumulators; DMMA = FP64 tensor cores")
cols = [k for k, _ in PAT]
print("kernel".ljust(58), "instr".rjust(6), " ".join(c.rjust(9) for c in cols))
for name, total, c in sorted(rows, key=lambda r: -r[1]):
    print(name[:58].ljust(58), str(total).rjust(6), " ".join(str(c.get(k, 0) or "").rjust(9) for k in cols))
agg = collections.Counter()
for _, _, c in rows:
    agg.update(c)
print("TOTAL".ljust(58), str(sum(r[1] for r in rows)).rjust(6), " ".join(str(agg.get(k, 0)).rjust(9) for k in cols))
