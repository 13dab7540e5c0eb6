#!/usr/bin/env python3
"""MemoryArchiver.run_maintenance(dry_run=True) on a synthetic on-disk Memdir, stage by stage:

    tools/bench_maintenance.py [--files 1000000] [--repeats 3] [--tree-dir DIR] [--oracle-files 20000]

The tree is synth.write_memdir_native's (the bench corpus as files).  `now` is frozen at the median record's date plus the
archive age, so the age cut falls at the median record.  Two archiver settings run: the defaults, and one with a tag rule and
two retention policies (importance and age).  For each, every stage runs `--repeats` times after one warm-up; the
median wall time per stage, the scan programs each stage ran and the records it selected are printed.  The first sync (the
cold pack of the tree) is timed on its own.  The oracle's per-file rate (list, read and parse every file of one directory, as
each reference stage does for the whole tree) is measured on a sub-tree of `--oracle-files` files, and the time the reference
would need for one run is estimated from it: the five stages list the tree about five times.

The card's name and power limit are printed with the numbers.  Exits non-zero without a GPU."""
import argparse, contextlib, io, json, os, shutil, statistics, subprocess, sys, tempfile, time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
os.environ.setdefault("TZ", "UTC")


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        sys.exit("tools/bench_maintenance.py measures on a GPU and found none")


def configure(arch, name, n_inbox):
    if name == "tags+retention":
        arch.add_tag_based_archive_rule("python", ".Archive/Tagged")
        arch.set_retention_policy("", n_inbox // 2, "importance")
        arch.set_retention_policy(".Projects/AI", 1000, "age")


def maintenance(args):
    gpu = gpu_info()
    from datetime import datetime, timedelta
    from fei_b200 import _abi, packer, synth
    from fei_b200.memdir_tools import archiver as A, utils as U
    from oracle import memdir_oracle as mo
    _abi.init(0)
    root = args.tree_dir or ("/dev/shm" if shutil.disk_usage("/dev/shm").free > 8 << 30 else None)
    scratch = tempfile.mkdtemp(prefix="fei_maint_", dir=root)
    try:
        base = os.path.join(scratch, "Memdir")
        t0 = time.perf_counter()
        synth.write_memdir_native(base, 0xB200, 0, args.files)
        write_s = time.perf_counter() - t0
        U.set_memdir_base(base)
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            pm = packer.packed()
        pack_s = time.perf_counter() - t0
        ts_sorted = sorted(pm.arrays["ts"].tolist())
        now = datetime.fromtimestamp(ts_sorted[len(ts_sorted) // 2]) + timedelta(days=90)
        Frozen = type("Frozen", (datetime,), {"now": classmethod(lambda cls, tz=None: cls.fromtimestamp(now.timestamp()))})
        A.datetime = Frozen
        n_inbox = pm.segments.get(("", "cur"), (0, 0))[1] - pm.segments.get(("", "cur"), (0, 0))[0]
        stages = ("archive_old_memories", "cleanup_memories", "empty_trash", "apply_retention_policies", "update_memory_statuses")
        result = {"files": args.files, "write_tree_s": round(write_s, 2), "first_sync_cold_pack_s": round(pack_s, 2),
                  "now": now.isoformat(), "configs": {}}
        for name in ("default", "tags+retention"):
            times = {s: [] for s in stages}
            passes, selected = {}, {}
            for rep in range(args.repeats + 1):
                arch = A.MemoryArchiver()
                configure(arch, name, n_inbox)
                for s in stages:
                    before = arch.scan_passes
                    t0 = time.perf_counter()
                    with contextlib.redirect_stdout(io.StringIO()):
                        st = arch.empty_trash(dry_run=True) if s == "empty_trash" else getattr(arch, s)(True)
                    dt = time.perf_counter() - t0
                    if rep:
                        times[s].append(dt)
                    passes[s] = arch.scan_passes - before
                    selected[s] = len(st["details"])
            arch = A.MemoryArchiver()
            configure(arch, name, n_inbox)
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                arch.run_maintenance(dry_run=True)
            whole = time.perf_counter() - t0
            result["configs"][name] = {
                "stages": {s: {"median_s": round(statistics.median(times[s]), 4), "runs_s": [round(x, 4) for x in times[s]],
                               "scan_programs": passes[s], "selected": selected[s]} for s in stages},
                "run_maintenance_dry_run_s": round(whole, 3)}
        # the oracle's per-file rate: one directory listed, read and parsed the way every reference stage does
        folder = max(((f, s) for f, s in pm.segments if s == "cur"), key=lambda k: pm.segments[k][1] - pm.segments[k][0])
        sub = os.path.join(scratch, "sub")
        src = os.path.join(base, folder[0], "cur")
        os.makedirs(os.path.join(sub, "cur"))
        for fn in sorted(os.listdir(src))[:args.oracle_files]:
            shutil.copy(os.path.join(src, fn), os.path.join(sub, "cur", fn))
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            k = len(mo.read_folder(sub, "", "cur", True))
        rate = k / (time.perf_counter() - t0)
        result["oracle"] = {"files": k, "files_per_s": round(rate, 1), "reference_run_estimate_s": round(5 * args.files / rate, 1),
                            "note": "one host core lists, reads and parses each file; the reference's five stages list the whole tree about five times"}
        result["gpu"] = gpu
        for name, row in result.pop("configs").items():
            print(json.dumps({"config": name, **row}), flush=True)
        print(json.dumps(result), flush=True)
    finally:
        packer.drop()
        shutil.rmtree(scratch, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--tree-dir")
    ap.add_argument("--oracle-files", type=int, default=20000)
    maintenance(ap.parse_args())


if __name__ == "__main__":
    main()
