#!/usr/bin/env python
"""cuobjdump -sass of the built library, condensed: per kernel the code size, the count of the mnemonics that show what the
kernel is made of (bulk / tensor-map copies, tensor-core MMAs, FP64, cache-hinted accesses, warp reductions, PDL) and the
first occurrence of each.  Usage: python tools/sass_excerpts.py > sass_excerpts.txt"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gr-baz_b200", "csrc", "libmusic_b200.so")
KEYS = ["UBLKCP", "UTMALDG", "LDGSTS", "HMMA", "DMMA", "DFMA", "DMUL", "F2F", "MUFU", "CREDUX", "REDUX", "SHFL", "ATOMS", "SYNCS", "ACQBULK",
        "PREEXIT", "NANOSLEEP", "MEMBAR", "RED", "UTCHMMA", "UTCQMMA", "LDTM", "STTM"]
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
print("# cuobjdump -sass %s (sm_90a), condensed by tools/sass_excerpts.py" % os.path.relpath(LIB, ROOT))
print("# UBLKCP = cp.async.bulk (1-D TMA), UTMALDG = cp.async.bulk.tensor (tensor-map TMA), LDGSTS = cp.async, HMMA.1688.F32.TF32 = mma.sync tf32,")
print("# CREDUX = redux.sync, PREEXIT / ACQBULK = griddepcontrol.launch_dependents / .wait (programmatic dependent launch), `desc[UR..]` on UBLKCP / UTMALDG / LDG = L2 cache-hint operand (evict_first stream, evict_last tables).")
print("# No tcgen05 (UTC*MMA / LDTM / STTM) by design: the one tensor-core contraction is a 6 %-utilised screen, see DESIGN.md section 5.\n")
cur, body = None, []
funcs = []
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        if cur:
            funcs.append((cur, body))
        cur, body = m.group(1), []
    elif cur:
        body.append(line)
if cur:
    funcs.append((cur, body))
for name, body in funcs:
    dem = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip().split("(")[0]
    if not re.search(r"fused|covN|cov4_tma|eig_coop|scan_peak1|prep_table_tc|gather", dem):
        continue
    cnt, first, last_addr, hinted = collections.Counter(), {}, 0, collections.Counter()
    for l in body:
        m = re.match(r"\s*/\*([0-9a-f]{4,6})\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)(.*?);", l)
        if not m:
            continue
        last_addr = int(m.group(1), 16)
        op = m.group(2)
        base = op.split(".")[0]
        if base in KEYS:
            cnt[base] += 1
            first.setdefault(base, (m.group(1), (op + m.group(3)).strip()))
            if base in ("UBLKCP", "UTMALDG") and "desc[" in m.group(3):
                hinted[base] += 1
    print("== %s   (%d bytes of SASS)" % (dem, last_addr + 16))
    print("   " + "  ".join("%s=%d" % (k, cnt[k]) for k in KEYS if cnt[k]) + ("   [with L2 cache hint: %s]" % dict(hinted) if hinted else ""))
    for k in ("UBLKCP", "UTMALDG", "LDGSTS", "HMMA", "CREDUX", "PREEXIT", "ACQBULK"):
        if k in first:
            print("   first %-8s /*%s*/ %s" % (k, first[k][0], first[k][1]))
    print()
