#!/usr/bin/env python
"""SASS evidence per kernel of libetl_decode.so: instruction-class counts (byte loads, local memory, bulk copies,
mbarrier ops, votes / shuffles) and the lines around every UBLKCP / SYNCS.  Usage: sass_excerpt.py [rNN]"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.normpath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
rnd = sys.argv[1] if len(sys.argv) > 1 else "r02"
lib = os.path.join(ROOT, "etl_b200", "libetl_decode.so")
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
kernels = collections.OrderedDict()
cur = None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        kernels[cur] = []
        continue
    if cur is not None and re.search(r"/\*[0-9a-f]{4}\*/", line):
        kernels[cur].append(line.rstrip())
res = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True).stdout
usage = {}
fn = None
for line in res.splitlines():
    m = re.search(r"Function (\S+):", line)
    if m:
        fn = m.group(1)
    elif fn and "REG:" in line:
        usage[fn] = line.strip()
        fn = None
CLASSES = [("LDG.E.U8 (byte loads from global)", r"\bLDG\.E\.U8"), ("LDG (all global loads)", r"\bLDG\b"), ("LDL/STL (local memory)", r"\b(LDL|STL)\b"),
           ("UBLKCP (1-D bulk async copy)", r"\bUBLKCP"), ("SYNCS (mbarrier)", r"\bSYNCS"), ("LDS (shared loads)", r"\bLDS\b"),
           ("SHFL", r"\bSHFL\b"), ("VOTE / MATCH", r"\b(VOTE|MATCH|VOTEU)\b"), ("MEMBAR", r"\bMEMBAR"), ("ATOM/RED (global atomics)", r"\b(ATOMG|ATOM|RED)\b")]
want = ["k_rows", "k_heavy", "k_records", "k_chase", "k_utf8_dead", "k_long_cells", "k_copy_rows", "k_perm", "k_fix"]
out = os.path.join(ROOT, "profiles", f"{rnd}_sass.txt")
os.makedirs(os.path.dirname(out), exist_ok=True)
with open(out, "w") as f:
    f.write("cuobjdump -sass / -res-usage etl_b200/libetl_decode.so (sm_90a), per kernel: resources, instruction-class counts,\n"
            "and the SASS around every bulk copy / mbarrier operation (tools/sass_excerpt.py)\n\n")
    for name, lines in kernels.items():
        short = next((w for w in want if w in name), None)
        if not short:
            continue
        f.write(f"== {name}   ({len(lines)} instructions)\n   {usage.get(name, '')}\n")
        for label, pat in CLASSES:
            n = sum(1 for l in lines if re.search(pat, l))
            f.write(f"   {label:38s} {n}\n")
        hits = [i for i, l in enumerate(lines) if "UBLKCP" in l] + [i for i, l in enumerate(lines) if "SYNCS" in l][:4]
        shown = set()
        for i in sorted(set(hits)):
            block = [j for j in range(max(0, i - 3), min(len(lines), i + 4)) if j not in shown]
            if not block:
                continue
            if shown and block[0] - 1 not in shown:
                f.write("      ...\n")
            for j in block:
                shown.add(j)
                f.write("      " + re.sub(r"\s+", " ", lines[j]).strip()[:150] + "\n")
        f.write("\n")
print("wrote", out)
