#!/usr/bin/env python3
"""Time of the head kernels on `Subject` regexes the DFA holds and regexes that take the head position automaton, on the
synthetic bench corpus:

    tools/bench_head_nfa.py [--entries 10000000] [--steps 10] [--warmup 3] [--sample 20000]

Workloads, each one program over the whole corpus: a DFA-sized regex, two proximity regexes the DFA refuses, and a filter
set of 32 `Subject` rules (30 words and the two proximity regexes: only those move to the automaton).  After a warm-up of
every workload, the steps alternate the workloads; each step is one scan_count call, and the median head_ms / total_ms of
the steps is reported with the hit counts and the words per position vector of the program's Subject automaton.  The hit
counts are checked against CPython re on the first `--sample` records, fetched back from the device.  The card's name and
power limit are printed with the numbers.  Exits non-zero without a GPU."""
import argparse, json, os, re, statistics, struct, subprocess, sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
os.environ.setdefault("TZ", "UTC")

import numpy as np  # noqa: E402

DFA = r"recommendation.*dashboard"
PROXIMITY = [r"(project|feature).{0,40}(tracker|dashboard)", r"(reflections|notes).{0,50}(node|rust|python)"]
WORDS = ["python", "rust", "docker", "kubernetes", "react", "angular", "node", "dashboard", "tracker", "system", "feature",
         "project", "idea", "request", "reflections", "learning", "notes", "meeting", "review", "design", "api", "data", "cloud",
         "security", "testing", "mobile", "web", "ai", "model", "deploy"]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--entries", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=20000)
    args = ap.parse_args()
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        sys.exit("tools/bench_head_nfa.py measures on a GPU and found none")
    import bench
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    from fei_b200.program import C_SLOT, Cond, ProgramBuilder
    from fei_b200.regexc import Pattern
    _abi.init(0)
    work = {"dfa " + DFA: [DFA]}
    for p in PROXIMITY:
        work["nfa " + p] = [p]
    work["32 rules, 2 proximity"] = WORDS + PROXIMITY

    def program(pats):
        pb = ProgramBuilder()
        for p in pats:
            pb.add_query([Cond(C_SLOT, pattern=Pattern("regex", p, re.IGNORECASE), field="Subject")])
        return pb.build()

    def words(prog):                                     # W of slot 0's position automaton (0: the DFA holds every pattern)
        off = struct.unpack_from("<I", prog, struct.unpack_from("<I", prog, 32)[0] + 12)[0]
        return struct.unpack_from("<I", prog, off)[0] if off else 0

    progs = {k: program(v) for k, v in work.items()}
    c = Corpus().synth(bench.SEED, 0, args.entries)
    for _ in range(args.warmup):
        for k, prog in progs.items():
            c.scan_count(prog, len(work[k]))
    steps = {k: [] for k in work}
    counts = {}
    for _ in range(args.steps):
        for k, prog in progs.items():
            counts[k] = c.scan_count(prog, len(work[k]))
            steps[k].append(c.timing())
    # hit counts of the sample against CPython re on the Subject values
    n = min(args.sample, args.entries)
    f = c.fetch(0, n)
    off = f["hdr_off"].astype(np.int64)
    subjects = []
    for i in range(n):
        lines = bytes(f["hdr"][off[i]:off[i + 1]]).decode("utf-8").split("\n")
        subjects.append(next((ln.split(":", 1)[1].strip() for ln in lines if ln.split(":", 1)[0].strip().lower() == "subject"), None))
    sample = Corpus().synth(bench.SEED, 0, n)
    sample_ok = {}
    for k, prog in progs.items():
        got = sample.scan_count(prog, len(work[k]))
        want = [sum(1 for s in subjects if s is not None and re.search(p, s, re.IGNORECASE)) for p in work[k]]
        sample_ok[k] = [int(x) for x in got] == want
    for k in work:
        tms = steps[k]
        row = {"workload": k, "head_ms": round(statistics.median(t["head_ms"] for t in tms), 3),
               "total_ms": round(statistics.median(t["total_ms"] for t in tms), 3), "nfa_words": words(progs[k]),
               "hits": [int(x) for x in counts[k]] if len(work[k]) <= 2 else int(np.sum(counts[k])), "sample_equals_re": sample_ok[k]}
        print(json.dumps(row), flush=True)
    print("GPU (name, power limit, max SM clock):", gpu)
    if not all(sample_ok.values()):
        sys.exit("hit counts differ from CPython re on the sample")


if __name__ == "__main__":
    main()
