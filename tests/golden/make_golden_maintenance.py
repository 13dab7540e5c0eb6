"""Write tests/golden/maintenance_golden.json from the reference's MemoryArchiver (memdir_tools/archiver.py).

Run on a machine that has the reference project:  python tests/golden/make_golden_maintenance.py /path/to/reference

The tree is tests/maintenance_tree.py's seeded tree; `memdir_tools.archiver.datetime.now` is frozen at its NOW.  For each of
maintenance_tree.CASES the golden records the statistics and the digest of the tree the run leaves (a dry run creates archive
folders too).  Each case starts from a fresh copy of the tree.  It also records the reference's signatures of the maintenance
methods.  One case per line."""
import contextlib
import inspect
import io
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
os.environ["TZ"] = "UTC"
time.tzset()

from tests import maintenance_tree as T          # noqa: E402


def main(reference: str) -> None:
    sys.path.insert(0, reference)
    import memdir_tools.archiver as ra
    import memdir_tools.utils as ru
    ra.datetime = T.frozen_datetime(ra.datetime)
    head = {"seed": T.SEED, "now": T.NOW.isoformat(), "signatures": {m: str(inspect.signature(getattr(ra.MemoryArchiver, m))) for m in T.METHODS}}
    cases = []
    with tempfile.TemporaryDirectory() as tmp:
        for k, (config, stage, dry_run) in enumerate(T.CASES):
            base = os.path.join(tmp, f"case{k}", "Memdir")
            T.build_tree(base)
            ru.MEMDIR_BASE = ra.MEMDIR_BASE = base
            arch = ra.MemoryArchiver()
            T.configure(arch, config)
            with contextlib.redirect_stdout(io.StringIO()):
                stats = T.run_stage(arch, stage, dry_run)
            cases.append({"config": config, "stage": stage, "dry_run": dry_run, "stats": stats, "tree": T.tree_digest(base)})
    with open(os.path.join(HERE, "maintenance_golden.json"), "w") as f:
        f.write(json.dumps(head)[:-1] + ', "cases": [\n' + ",\n".join(json.dumps(c) for c in cases) + "\n]}\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_maintenance.py <directory holding the reference's memdir_tools package>")
    main(sys.argv[1])
