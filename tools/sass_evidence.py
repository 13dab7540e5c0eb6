#!/usr/bin/env python3
"""Instruction counts per kernel from `cuobjdump -sass fei_b200/libfeiscan.so` for the mnemonics that show how the kernels are built
(tools/sass_evidence.py > profiles/rN_sass_evidence.txt); with --row-loop 'k_body<true, 2, false>' [LIB], the instructions
per 16-byte row of that kernel's row loop by pipe.  Runs without a GPU."""
import collections, os, re, subprocess, sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
argv = sys.argv[1:]
row_loop = None                      # --row-loop 'k_body<true, 2, false>': the per-pipe count of that kernel's full-row loop
if "--row-loop" in argv:
    i = argv.index("--row-loop"); row_loop = argv[i + 1]; del argv[i:i + 2]
so = argv[0] if argv else os.path.join(REPO, "fei_b200", "libfeiscan.so")

# Which pipe of an H100 SM sub-partition an instruction occupies.  ALU and FMA (IMAD runs on the FMA pipe) take 16 lanes
# per clock each, so a warp-wide instruction holds its pipe for 2 clocks; that is what makes the ALU count a floor.
ALU = ("PRMT", "SHF", "LOP3", "PLOP3", "IADD3", "VIADD", "IABS", "ISETP", "SEL", "POPC", "FLO", "LEA", "VIMNMX", "IMNMX", "MOV", "SGXT", "BMSK")
FMA = ("IMAD", "FFMA", "FMUL", "FADD")
LSU = ("LDS", "STS", "LDG", "STG", "LDL", "STL", "ATOM", "RED", "LD.", "ST.")


def pipe_of(op):
    return "ALU" if op.startswith(ALU) else "FMA" if op.startswith(FMA) else "LSU" if op.startswith(LSU) else "other"


def row_loop_table(body):
    """body: [(address, predicate, opcode, operands)] of one kernel.  The row loop is the innermost loop (a backward branch
    with no other inside) whose fullest pass executes the most LDS.U16, one per byte; of the passes through it with that
    many lookups the shortest is the full-row path (a partial row branches around every byte)."""
    idx = {a: i for i, (a, _, _, _) in enumerate(body)}
    back = [(idx[int(m.group(1), 16)], i) for i, (a, _, op, args) in enumerate(body)
            if op.startswith("BRA") and (m := re.search(r"0x([0-9a-f]+)", args)) and int(m.group(1), 16) in idx and int(m.group(1), 16) <= a]
    best = None
    for head, tail in back:
        if any((h, t) != (head, tail) and head <= t <= tail and h >= head for h, t in back):
            continue                                           # not innermost
        score = {}                                             # i -> (lookups, -instructions, path) from i to the back edge
        for i in range(tail, head - 1, -1):
            _, pred, op, args = body[i]
            here = (1 if op.startswith("LDS.U16") else 0, -1)
            if i == tail:
                score[i] = (*here, (i,)); continue
            succ = [i + 1]
            if op.startswith("BRA"):
                t = idx.get(int(re.search(r"0x([0-9a-f]+)", args).group(1), 16), -1)
                succ = ([i + 1] if pred else []) + ([t] if i < t <= tail else [])
            elif op.startswith(("EXIT", "RET")) and not pred:
                succ = []
            cand = [score[j] for j in succ if j in score]
            if cand:
                c = max(cand, key=lambda t: t[:2])
                score[i] = (c[0] + here[0], c[1] + here[1], (i,) + c[2])
        if head in score and (best is None or score[head][:2] > best[:2]):
            best = score[head]
    if not best or best[0] < 16:
        sys.exit("no loop with 16 LDS.U16 per pass in this kernel")
    rows = best[0] // 16
    per_pipe, ops = collections.Counter(), collections.Counter()
    for i in best[2]:
        per_pipe[pipe_of(body[i][2])] += 1; ops[(pipe_of(body[i][2]), body[i][2].split(".")[0])] += 1
    print(f"   full-row loop 0x{body[best[2][0]][0]:04x}..0x{body[best[2][-1]][0]:04x}: {len(best[2])} instructions for {rows} row(s) of 16 bytes")
    for pipe in ("ALU", "FMA", "LSU", "other"):
        detail = "  ".join(f"{o}={n}" for (pp, o), n in sorted(ops.items()) if pp == pipe)
        print(f"   {pipe:5s} {per_pipe[pipe] / rows:6.1f} per row  {per_pipe[pipe] / rows / 16:5.2f} per byte   ({detail})")
WANT = ("UBLKCP", "SYNCS", "ELECT", "VOTE", "MATCH", "SHFL", "LDS", "STS", "LDG", "STG", "ATOM", "RED", "SHF.R.W", "SHF.L.W", "IADD3", "LOP3", "PRMT",
        "BAR", "MEMBAR", "NANOSLEEP", "DADD", "DMUL", "DFMA")
SKIP = ("IADD3.X",)
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
arch = sorted(set(re.findall(r"arch = (sm_\w+)", txt)))
cur, counts, total, bodies = None, {}, {}, {}
for line in txt.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1); counts[cur] = collections.Counter(); total[cur] = 0; bodies[cur] = []
        continue
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)([^;]*)", line)
    if m and cur:
        op = m.group(3); total[cur] += 1
        bodies[cur].append((int(m.group(1), 16), m.group(2), op, m.group(4)))
        if op.startswith(WANT) and op not in SKIP:
            counts[cur][op] += 1
demangle = subprocess.run(["c++filt"] + list(counts), capture_output=True, text=True).stdout.split("\n") if counts else []
if row_loop:
    want = re.sub(r"\s", "", row_loop)
    for name, dm in zip(counts, demangle):
        if want in re.sub(r"\s", "", dm):
            print(f"## {re.sub(r'[(].*', '', dm)}  ({total[name]} instructions)   [{name}]")
            row_loop_table(bodies[name])
    sys.exit(0)
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
