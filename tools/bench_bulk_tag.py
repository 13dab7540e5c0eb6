#!/usr/bin/env python3
"""MemdirFolderManager.bulk_tag_folder on a synthetic on-disk Memdir:

    tools/bench_bulk_tag.py [--files 1000000] [--repeats 5] [--tree-dir DIR] [--oracle-files 20000]

The tree is synth.write_memdir_native's (the bench corpus as files).  Three edits of the Inbox run one after the other:
  remove-rare      remove the Inbox's rarest tag (few files change);
  add-most         add a new tag to `cur` (it rewrites most files of the Inbox);
  add-satisfied    add the same tag to `cur` and `new` (most records already carry it: only `new` is rewritten).
For each, the device call alone (fei_corpus_tag_edit on every packed corpus, no file written) is timed `--repeats` times first:
the median of its CUDA-event time (selection scan, measure and write kernels, copies) and of its wall time.  Then the edit runs
for real once: its wall time, the part spent in the device call, the files rewritten, and the sync before it (which reads the
files the previous edit rewrote).  The oracle's rate (list, read and parse every file of one directory, as the reference does
before its first write) is measured on a sub-tree of `--oracle-files` files.

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
        sys.exit("tools/bench_bulk_tag.py measures on a GPU and found none")


def per_edit(values, k):
    """Median over edits of the sum over the k corpora (base, delta) each edit calls."""
    return statistics.median([sum(values[i:i + k]) for i in range(0, len(values), k)])


def bench(args):
    gpu = gpu_info()
    from fei_b200 import _abi, packer, synth
    from fei_b200.corpus import Corpus
    from fei_b200.memdir_tools import folders as F, utils as U
    from oracle import memdir_oracle as mo
    _abi.init(0)
    calls = []                                                  # (wall s, CUDA-event ms) of every device call
    plain_tag_edit = Corpus.tag_edit

    def timed_tag_edit(self, prog, operation, tags):
        t0 = time.perf_counter()
        out = plain_tag_edit(self, prog, operation, tags)       # ends in a stream synchronise
        calls.append((time.perf_counter() - t0, self.timing()["total_ms"]))
        return out
    Corpus.tag_edit = timed_tag_edit
    root = args.tree_dir or ("/dev/shm" if shutil.disk_usage("/dev/shm").free > 8 << 30 else None)
    scratch = tempfile.mkdtemp(prefix="fei_bulktag_", dir=root)
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
        mgr = F.MemdirFolderManager()
        with contextlib.redirect_stdout(io.StringIO()):
            tags = mgr.get_folder_stats("")["tags"]
        rare = min(tags, key=lambda t: (tags[t], t))
        inbox = {st: pm.segments.get(("", st), (0, 0))[1] - pm.segments.get(("", st), (0, 0))[0] for st in U.STANDARD_FOLDERS}
        result = {"files": args.files, "inbox": inbox, "write_tree_s": round(write_s, 2), "first_sync_cold_pack_s": round(pack_s, 2),
                  "rare_tag": rare, "rare_tag_records": tags[rare], "edits": {}}
        for name, tag_list, statuses, op in (("remove-rare", [rare], ["cur"], "remove"), ("add-most", ["bench-new"], ["cur"], "add"),
                                             ("add-satisfied", ["bench-new"], ["cur", "new"], "add")):
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                pm = packer.packed()
            sync_s = time.perf_counter() - t0
            with pm.lock:
                del calls[:]
                for _ in range(args.repeats):
                    F.MemdirFolderManager._tag_edit(pm, "", statuses, op, [t.encode() for t in tag_list])
                walls, events = [c[0] for c in calls], [c[1] for c in calls]
                k = len(pm._corpora())
            del calls[:]
            t0 = time.perf_counter()
            with contextlib.redirect_stdout(io.StringIO()):
                count, _details = mgr.bulk_tag_folder("", tag_list, statuses, op)
            whole = time.perf_counter() - t0
            device = sum(c[0] for c in calls)
            result["edits"][name] = {
                "operation": op, "tags": tag_list, "statuses": statuses, "files_rewritten": count, "corpora": k,
                "device_call_event_ms_median": round(per_edit(events, k), 3),
                "device_call_wall_ms_median": round(1000 * per_edit(walls, k), 3),
                "sync_before_s": round(sync_s, 3), "bulk_tag_folder_s": round(whole, 3), "device_call_s": round(device, 3),
                "host_rest_s": round(whole - device, 3),
                "note": "host_rest_s: sync, listing bookkeeping and the rewrite of the affected files on the host"}
        sub = os.path.join(scratch, "sub")
        src = os.path.join(base, "cur")
        os.makedirs(os.path.join(sub, "cur"))
        for fn in sorted(os.listdir(src))[:args.oracle_files]:
            shutil.copy(os.path.join(src, fn), os.path.join(sub, "cur", fn))
        t0 = time.perf_counter()
        with contextlib.redirect_stdout(io.StringIO()):
            n_listed = len(mo.read_folder(sub, "", "cur", False))
        rate = n_listed / (time.perf_counter() - t0)
        result["oracle"] = {"files": n_listed, "files_per_s": round(rate, 1), "reference_listing_estimate_s": round(inbox["cur"] / rate, 1),
                            "note": "one host core lists, reads and parses each file of the Inbox's cur before the reference's first write"}
        result["gpu"] = gpu
        for name, row in result.pop("edits").items():
            print(json.dumps({"edit": name, **row}), flush=True)
        print(json.dumps(result), flush=True)
    finally:
        Corpus.tag_edit = plain_tag_edit
        packer.drop()
        shutil.rmtree(scratch, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--files", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--tree-dir")
    ap.add_argument("--oracle-files", type=int, default=20000)
    bench(ap.parse_args())


if __name__ == "__main__":
    main()
