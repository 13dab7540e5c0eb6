#!/usr/bin/env python3
"""Where the time of the 32-pattern batch goes after the scan: tools/scan_tail.py [entries] [calls].

Synthesizes the bench corpus (bench.SEED, 10 M entries by default), runs fei_scan_count with the 32 content patterns of
bench.py a few times to warm up, then `calls` timed calls, and prints one JSON line: medians of the per-call CUDA-event
timings (total_ms, body_ms = the body kernel including the ordered lists it builds, compact_ms = what is left after the
body kernel), the kernel launches per call, the host wall time per call (scan_count returns after the totals are on the
host), and the GPU it ran on (name, power limit, max SM clock from nvidia-smi)."""
import json, os, re, statistics, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("TZ", "UTC")
from fei_b200.corpus import Corpus
from fei_b200.program import content_batch_program
from fei_b200.regexc import Pattern
import bench


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    c = Corpus().synth(bench.SEED, 0, n)
    prog, nq = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in bench.BATCH32]), 32
    for _ in range(3):
        c.scan_count(prog, nq)
    rows, wall = [], []
    for _ in range(calls):
        t0 = time.perf_counter()
        c.scan_count(prog, nq)
        wall.append((time.perf_counter() - t0) * 1e3)
        rows.append(c.timing())
    med = lambda k: round(statistics.median(r[k] for r in rows), 4)
    print(json.dumps({"entries": n, "calls": calls, "total_ms": med("total_ms"), "body_ms": med("body_ms"),
                      "compact_ms": med("compact_ms"), "kernel_launches": int(rows[-1]["kernel_launches"]),
                      "wall_ms_per_call": round(statistics.median(wall), 4), "gpu": gpu_info()}))
    c.close()


if __name__ == "__main__":
    main()
