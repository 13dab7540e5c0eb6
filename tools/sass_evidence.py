#!/usr/bin/env python3
"""Instruction counts per kernel from `cuobjdump -sass fei_b200/libfeiscan.so` for the mnemonics that show how the kernels are built
(tools/sass_evidence.py > profiles/rN_sass_evidence.txt).  Runs without a GPU."""
import collections, os, re, subprocess, sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = sys.argv[1] if len(sys.argv) > 1 else os.path.join(REPO, "fei_b200", "libfeiscan.so")
WANT = ("UBLKCP", "SYNCS", "ELECT", "VOTE", "MATCH", "SHFL", "LDS", "STS", "LDG", "STG", "ATOM", "RED", "SHF.R.W", "SHF.L.W", "IADD3", "LOP3", "PRMT",
        "BAR", "MEMBAR", "NANOSLEEP", "DADD", "DMUL", "DFMA")
SKIP = ("IADD3.X",)
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
arch = sorted(set(re.findall(r"arch = (sm_\w+)", txt)))
cur, counts, total = None, {}, {}
for line in txt.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1); counts[cur] = collections.Counter(); total[cur] = 0
        continue
    m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
    if m and cur:
        op = m.group(1); total[cur] += 1
        if op.startswith(WANT) and op not in SKIP:
            counts[cur][op] += 1
demangle = subprocess.run(["c++filt"] + list(counts), capture_output=True, text=True).stdout.split("\n") if counts else []
print(f"# SASS evidence: cuobjdump -sass {os.path.relpath(so, REPO)} (cubins: {', '.join(arch)}); regenerate with tools/sass_evidence.py")
print("""
Counts per kernel of the mnemonics that show the design: UBLKCP.S.G = cp.async.bulk (TMA bulk copy into shared memory), SYNCS.* = mbarrier
arrive / expect_tx / try_wait, ELECT = elected issuing lane, VOTE* = warp ballots, SHFL = warp shuffles, LDS.U16 = one automaton lookup
per byte, LDS.128 = ring read-back, LDG.E.NA.128.CONSTANT = ld.global.nc.L1::no_allocate.v4 streaming loads, LDG/STG.E.128 = 16-byte
rows, ATOMG / REDG = global atomics (work counters, window completion counters, hit counts), SHF.R.W = 32-bit rotates (SHA-256),
NANOSLEEP = the back-off of the ordered-list look-back and help_tail waits, D* = FP64 (only the shortest-repr float formatter's checks), no MATCH anywhere.
""")
for (name, c), dm in sorted(zip(counts.items(), demangle), key=lambda t: t[1]):
    short = re.sub(r"\(.*", "", dm)
    print(f"## {short}  ({total[name]} instructions)   [{name}]")
    print("   " + "  ".join(f"{k}={v}" for k, v in sorted(c.items())))
