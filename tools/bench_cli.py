#!/usr/bin/env python3
"""The Memdir command line (fei_b200.memdir_tools.cli) on a synthetic on-disk Memdir:

    tools/bench_cli.py [--files 1000000] [--repeats 3] [--tree-dir DIR]

The tree is synth.write_memdir_native's.  Commands: `list --json` and `list -c --json` of the Inbox `cur` directory, `view <id>`,
`flag <id> --add F`, and `search "#python" --format json|csv|compact` with and without --with-content.  For each: the median
CUDA-event time of fei_corpus_format_records summed over the command's device calls, and the median wall time of the command
with stdout sent to /dev/null.  In the same run the current route: search_memories + json.dumps of its dicts for the searches,
utils.list_memories (+ json.dumps) for the listings.  The card's name and power limit are printed with the numbers.  Exits
non-zero without a GPU."""
import argparse, contextlib, io, json, os, statistics, subprocess, sys, tempfile, time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
os.environ.setdefault("TZ", "UTC")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        sys.exit("tools/bench_cli.py measures on a GPU and found none")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--tree-dir", default=None)
    args = ap.parse_args()
    card = gpu_info()
    from fei_b200 import corpus, packer, synth
    from fei_b200.memdir_tools import cli, search, utils as U
    tmp = tempfile.mkdtemp(dir=args.tree_dir)
    base = os.path.join(tmp, "Memdir")
    t0 = time.perf_counter()
    synth.write_memdir_native(base, 0xC11, 0, args.files)
    U.set_memdir_base(base)
    U.ensure_memdir_structure()
    t1 = time.perf_counter()
    pm = packer.packed(base)
    t2 = time.perf_counter()
    seg = pm.segments[("", "cur")]
    uid = pm.materialize([seg[0] + (seg[1] - seg[0]) // 2], False)[0]["metadata"]["unique_id"]
    print(f"# {card}; {args.files} files written in {t1 - t0:.1f} s, packed in {t2 - t1:.1f} s; Inbox/cur {seg[1] - seg[0]} records",
          flush=True)

    dev_ms = []
    real = corpus.Corpus.format_records

    def timed(self, *a, **k):
        r = real(self, *a, **k)
        dev_ms.append(self.last_format_ms)
        return r
    corpus.Corpus.format_records = timed

    def run(argv):
        old = sys.argv
        sys.argv = argv
        try:
            with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
                cli.main()
        finally:
            sys.argv = old

    def measure(argv):
        walls, devs = [], []
        for _ in range(args.repeats + 1):
            dev_ms.clear()
            t = time.perf_counter()
            run(argv)
            walls.append(time.perf_counter() - t)
            devs.append(sum(dev_ms))
        return statistics.median(walls[1:]), statistics.median(devs[1:])      # the first run warms up

    def current(fn):
        ts = []
        for _ in range(args.repeats):
            t = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                fn()
            ts.append(time.perf_counter() - t)
        return statistics.median(ts)

    def list_route(content):
        mems = U.list_memories("", "cur", include_content=content)
        for m in mems:
            m["metadata"]["date"] = m["metadata"]["date"].isoformat()
        json.dumps(mems, indent=2)

    def search_route(content):
        q = search.parse_search_args("#python")
        q.with_content(content)
        res = search.search_memories(q)
        for m in res:
            m["metadata"]["date"] = m["metadata"]["date"].isoformat()
        json.dumps(res, indent=2)

    rows = []
    for name, argv, route in [
            ("list --json", ["cli", "list", "--json"], lambda: list_route(False)),
            ("list -c --json", ["cli", "list", "-c", "--json"], lambda: list_route(True)),
            ("view <id>", ["cli", "view", uid], None),
            ("search json", ["cli", "search", "#python", "--format", "json"], lambda: search_route(False)),
            ("search csv", ["cli", "search", "#python", "--format", "csv"], None),
            ("search compact", ["cli", "search", "#python", "--format", "compact"], None),
            ("search json --with-content", ["cli", "search", "#python", "--format", "json", "--with-content"], lambda: search_route(True)),
            ("search csv --with-content", ["cli", "search", "#python", "--format", "csv", "--with-content"], None),
            ("search compact --with-content", ["cli", "search", "#python", "--format", "compact", "--with-content"], None)]:
        wall, dev = measure(argv)
        cur = current(route) if route else None
        rows.append({"command": name, "format_records_ms": round(dev, 2), "wall_s": round(wall, 3),
                     "current_route_s": None if cur is None else round(cur, 3)})
        print(json.dumps(rows[-1]), flush=True)
    t = time.perf_counter()
    run(["cli", "flag", uid, "--add", "F"])
    rows.append({"command": "flag <id> --add F", "format_records_ms": 0.0, "wall_s": round(time.perf_counter() - t, 3), "current_route_s": None})
    print(json.dumps(rows[-1]), flush=True)
    print(json.dumps({"card": card, "files": args.files, "rows": rows}))
    packer.drop()
    import shutil
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
