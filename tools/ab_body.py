#!/usr/bin/env python3
"""A/B of the multi-pattern body kernel between two (or more) builds of libfeiscan.so, alternated in one session:

    tools/ab_body.py A.so B.so [--rounds 5] [--calls 20] [--entries 10000000]

A round is one process per library (A, then B): it builds the synthetic bench corpus (two corpora of 10 M entries do not
fit one 80 GB card, so the libraries take turns) and runs `--calls` scan_count calls of the 32-pattern bench batch and of
a batch of 32 words that occur nowhere (every byte goes through the automaton, no record is ever decided), printing the
median body_ms / total_ms of each from Corpus.timing().  Every scan_count call is followed by a scan_masks call of the same
batch (the same kernel without the ordered lists): the difference of their body_ms medians is what building the lists costs.  The card's name, power limit and SM clock are printed last: they
belong to every number above.  Exits non-zero without a GPU."""
import argparse, json, os, re, statistics, subprocess, sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
os.environ.setdefault("TZ", "UTC")

# 32 patterns of words the synthetic text never uses; three alternations, like the bench batch, so that the automaton
# has 35 accepting states and runs the kernel instance the bench batch runs
ABSENT32 = ["quagga", "zebra|okapi", "narwhal", "axolotl", "wombat", "ocelot", "tapir", "pangolin", "capybara", "lemur",
            "meerkat", "platypus", "aardvark", "manatee", "ibex|kakapo|numbat", "quokka", "dugong", "gharial", "saiga",
            "tarsier", "caracal", "echidna", "bonobo", "marmot", "gibbon", "jackal", "walrus", "heron", "osprey", "dingo",
            "stoat", "civet"]


def worker(lib_path, entries, calls):
    from fei_b200 import _abi
    _abi.LIB_PATH = os.path.abspath(lib_path)
    _abi.init(0)
    import bench
    from fei_b200.corpus import Corpus
    from fei_b200.program import content_batch_program
    from fei_b200.regexc import Pattern
    c = Corpus().synth(bench.SEED, 0, entries)
    out = {}
    for name, pats in (("batch32", bench.BATCH32), ("absent32", ABSENT32)):
        prog = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in pats])
        for _ in range(3):
            cnt = c.scan_count(prog, 32)
            c.scan_masks(prog)
        body, total, masks_body = [], [], []
        for _ in range(calls):
            cnt = c.scan_count(prog, 32)
            tm = c.timing()
            body.append(tm["body_ms"]); total.append(tm["total_ms"])
            c.scan_masks(prog)
            masks_body.append(c.timing()["body_ms"])
        out[name] = {"body_ms": statistics.median(body), "total_ms": statistics.median(total), "hits": int(cnt.sum()),
                     "masks_body_ms": statistics.median(masks_body),
                     "body_bytes_read": int(tm["body_bytes_read"]),
                     "kernel": [int(tm["body_kernel"]), int(tm["body_direct"]), int(tm["body_acc_mode"])]}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("libs", nargs="+", metavar="LIB")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--entries", type=int, default=10_000_000)
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args.worker, args.entries, args.calls)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        gpu = ""
    if not gpu:
        sys.exit("tools/ab_body.py measures on a GPU and found none")
    res = {lib: {"batch32": [], "absent32": []} for lib in args.libs}
    for r in range(args.rounds):
        for lib in args.libs:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), *args.libs, "--worker", lib, "--entries", str(args.entries),
                                "--calls", str(args.calls)], capture_output=True, text=True)
            if p.returncode != 0:
                sys.exit(f"worker for {lib} failed:\n{p.stdout}\n{p.stderr}")
            out = json.loads(p.stdout.strip().splitlines()[-1])
            for name, o in out.items():
                res[lib][name].append(o)
                print(f"round {r} {lib:40s} {name:9s} body_ms {o['body_ms']:7.3f}  masks-only body_ms {o['masks_body_ms']:7.3f}  "
                      f"total_ms {o['total_ms']:7.3f}  hits {o['hits']}  "
                      f"body_bytes_read {o['body_bytes_read']}  kernel/direct/acc {o['kernel']}", flush=True)
    print()
    for name in ("batch32", "absent32"):
        for lib in args.libs:
            b = [o["body_ms"] for o in res[lib][name]]; t = [o["total_ms"] for o in res[lib][name]]
            mb = [o["masks_body_ms"] for o in res[lib][name]]; share = [o["body_ms"] - o["masks_body_ms"] for o in res[lib][name]]
            print(f"{name:9s} {lib:40s} body_ms median {statistics.median(b):7.3f} (range {min(b):.3f}-{max(b):.3f})  "
                  f"total_ms median {statistics.median(t):7.3f} (range {min(t):.3f}-{max(t):.3f})  "
                  f"masks-only body_ms median {statistics.median(mb):7.3f}  lists share median {statistics.median(share):6.3f} "
                  f"(range {min(share):.3f}-{max(share):.3f})")
        same = len({(o["hits"], o["body_bytes_read"]) for lib in args.libs for o in res[lib][name]}) == 1
        print(f"{name:9s} hits and body_bytes_read equal in every run: {same}")
    print("GPU (name, power limit, SM clock now, SM clock max):", gpu.splitlines()[0])


if __name__ == "__main__":
    main()
