#!/usr/bin/env python3
"""Throughput of the content position automaton (k_body_nfa) next to the DFA kernels, on the synthetic bench corpus:

    tools/bench_nfa.py [--entries 10000000] [--steps 10] [--warmup 3] [--sample 20000]

Workloads, each one program over the whole corpus: `kubernetes.*docker` (a DFA), three proximity patterns the DFA refuses
(position vectors of 4 and 8 words), the longest gap the plain position automaton holds (`kubernetes.{0,238}docker`, 8 words)
and three it refuses, which run with one counter (`{0,239}`, `{0,1000}`, `{0,5000}`), the first 31 patterns of the 32-pattern bench batch plus one proximity pattern (the
DFA and the position automaton in one kernel) and the plain 32-pattern batch.  After a warm-up of every workload, the steps
alternate the workloads; each step is one scan_count call, and the median body_ms / total_ms of the steps is reported with
the content GB/s (body bytes of the corpus over body_ms), the kernel the scan ran (fei_scan_timing.body_kernel), the
words per position vector and its counters.  The hit counts are checked against CPython re on the first `--sample` records, fetched back from
the device.  The card's name and power limit are printed with the numbers.  Exits non-zero without a GPU."""
import argparse, json, os, re, statistics, subprocess, sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
os.environ.setdefault("TZ", "UTC")

import numpy as np  # noqa: E402

PROXIMITY = [r"kubernetes.{0,60}docker", r"kubernetes.{0,200}docker", r"\bpython\b.{0,60}\b(rust|django)\b"]
LONG_GAPS = [r"kubernetes.{0,238}docker", r"kubernetes.{0,239}docker", r"kubernetes.{0,1000}docker", r"kubernetes.{0,5000}docker"]


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
        sys.exit("tools/bench_nfa.py measures on a GPU and found none")
    import bench
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    from fei_b200.program import content_batch_program
    from fei_b200.regexc import Pattern
    _abi.init(0)
    rx = lambda p: Pattern("regex", p, re.IGNORECASE)                     # noqa: E731
    work = {"dfa kubernetes.*docker": [r"kubernetes.*docker"]}
    for p in PROXIMITY + LONG_GAPS:
        work["nfa " + p] = [p]
    work["batch31 + " + PROXIMITY[0]] = bench.BATCH32[:31] + [PROXIMITY[0]]
    work["batch32"] = list(bench.BATCH32)
    progs = {k: content_batch_program([rx(p) for p in v]) for k, v in work.items()}
    c = Corpus().synth(bench.SEED, 0, args.entries)
    body_bytes = c.stats()["body_bytes"]
    for _ in range(args.warmup):
        for k, prog in progs.items():
            c.scan_count(prog, len(work[k]))
    steps = {k: [] for k in work}
    counts = {}
    for _ in range(args.steps):
        for k, prog in progs.items():
            counts[k] = c.scan_count(prog, len(work[k]))
            steps[k].append(c.timing())
    # hit counts of the sample against CPython re
    n = min(args.sample, args.entries)
    f = c.fetch(0, n)
    off = f["body_off"].astype(np.int64)
    texts = [bytes(f["body"][off[i]:off[i + 1]]).decode("utf-8") for i in range(n)]
    sample_ok = {}
    sample = Corpus().synth(bench.SEED, 0, n)
    for k, prog in progs.items():
        got = sample.scan_count(prog, len(work[k]))
        want = [sum(1 for t in texts if re.search(p, t, re.IGNORECASE)) for p in work[k]]
        sample_ok[k] = [int(x) for x in got] == want
    out = []
    for k in work:
        tms = steps[k]
        body_ms = statistics.median(t["body_ms"] for t in tms)
        row = {"workload": k, "body_ms": round(body_ms, 3), "total_ms": round(statistics.median(t["total_ms"] for t in tms), 3),
               "body_kernel": int(tms[-1]["body_kernel"]), "body_nfa_words": int(tms[-1]["body_nfa_words"]),
               "body_nfa_counters": int(tms[-1]["body_nfa_counters"]),
               "body_GB_per_s": round(body_bytes / body_ms / 1e6, 1),
               "hits": int(np.sum(counts[k])), "sample_equals_re": sample_ok[k]}
        out.append(row)
        print(json.dumps(row), flush=True)
    print("GPU (name, power limit, max SM clock):", gpu)
    if not all(sample_ok.values()):
        sys.exit("hit counts differ from CPython re on the sample")


if __name__ == "__main__":
    main()
