"""MemoryArchiver's maintenance stages (archive_old_memories, cleanup_memories, empty_trash, apply_retention_policies,
update_memory_statuses, run_maintenance) on the GPU against the reference-generated goldens (tests/golden/maintenance_golden.json):
the same statistics with the same details, and the same tree afterwards: files, bytes and directories (a dry run creates some).  Each case runs on a fresh
copy of the seeded tree (tests/maintenance_tree.py) with `datetime.now()` frozen as the goldens froze it.

The order of details is compared per listed directory and kind of rule, with records shown by timestamp: the reference lists a
directory newest first with ties in the order the file system enumerates it, and walks the folders in os.walk order, both of
which differ between machines.  The tie order the packed listing gives is checked on the machine itself against the oracle's
listing."""
import contextlib
import io
import json
import re
import sys

import pytest

from tests import maintenance_tree as T
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return load_golden("maintenance_golden.json")


@pytest.fixture
def fresh(gpu, tmp_path, monkeypatch):
    """A fresh copy of the golden tree as the Memdir base, with now() frozen; the packed corpora are dropped afterwards."""
    from fei_b200 import packer
    from fei_b200.memdir_tools import archiver as A, utils as U
    monkeypatch.setattr(A, "datetime", T.frozen_datetime(A.datetime))
    bases = []

    def make(name):
        base = str(tmp_path / name / "Memdir")
        T.build_tree(base)
        monkeypatch.setattr(U, "MEMDIR_BASE", base)
        bases.append(base)
        return base
    yield make
    for b in bases:
        packer.drop(b)


def _same_stats(got, want, recs, where, moved):
    assert {k: v for k, v in got.items() if k != "details"} == {k: v for k, v in want.items() if k != "details"}, where
    dump = lambda ds: sorted(json.dumps(d, sort_keys=True) for d in ds)                       # noqa: E731
    assert dump(got["details"]) == dump(want["details"]), where

    def per_dir(ds, moved_to):
        """Per listed directory and kind of rule: the details in order, by timestamp; records that share one may come in either
        order.  A record a real run moved is listed from its new folder by the rules and stages after the move (moved_to)."""
        out = {}
        for d in ds:
            folder, status, ts = recs[d["memory_id"]]
            key = (moved_to.get(d["memory_id"], folder), status, d.get("tag"), "age" in d)
            out.setdefault(key, []).append((ts, sorted((k, v) for k, v in d.items() if k not in ("memory_id", "subject"))))
            m = re.match(r"(?:Archived|Moved) to (\S+)", d["action"])
            if m:
                moved_to[d["memory_id"]] = m.group(1)
        for key, seq in out.items():
            runs = [[seq[0]]] if seq else []
            for item in seq[1:]:
                if item[0] == runs[-1][-1][0]:
                    runs[-1].append(item)
                else:
                    runs.append([item])
            out[key] = [sorted(run) for run in runs]
        return out
    assert per_dir(got["details"], moved[0]) == per_dir(want["details"], moved[1]), where


def _check_case(case, got, recs, base):
    where = (case["config"], case["stage"], case["dry_run"])
    if case["stage"] == "run_maintenance":
        assert list(got) == list(case["stats"]), where
        moved = ({}, {})                                        # the stages run one after the other on one tree
        for k in got:
            _same_stats(got[k], case["stats"][k], recs, where + (k,), moved)
    else:
        _same_stats(got, case["stats"], recs, where, ({}, {}))
    assert T.tree_digest(base) == case["tree"], where          # moves, renames, deletions, rewritten bytes, directories created


@pytest.mark.parametrize("k", range(len(T.CASES)))
def test_maintenance_matches_reference_goldens(golden, fresh, k):
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    case = golden["cases"][k]
    base = fresh("tree")
    recs = T.records(base)
    arch = MemoryArchiver()
    T.configure(arch, case["config"])
    with contextlib.redirect_stdout(io.StringIO()):
        got = T.run_stage(arch, case["stage"], case["dry_run"])
    _check_case(case, got, recs, base)


def test_stages_scan_once_per_32_queries(golden, fresh):
    """A dry run selects each stage with one scan program; the retention policies' importance buckets are one program too."""
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    fresh("passes")
    arch = MemoryArchiver()
    T.configure(arch, "configured")
    with contextlib.redirect_stdout(io.StringIO()):
        for stage in ("archive_old_memories", "empty_trash", "apply_retention_policies", "update_memory_statuses"):
            before = arch.scan_passes
            T.run_stage(arch, stage, True)
            assert arch.scan_passes - before == 1, stage


def test_retention_by_age_reverses_runs_of_equal_timestamps(fresh):
    """Mode `age` is Python's stable sort by timestamp over the listing: on this machine's own listing order (the oracle's), the
    records that share a timestamp keep their listing order inside their run."""
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    from oracle import memdir_oracle as mo
    base = fresh("ties")
    folder = ".Projects/Alpha"                                  # the golden tree lets records of this folder share timestamps
    with contextlib.redirect_stdout(io.StringIO()):
        mems = mo.read_folder(base, folder, "cur", False)
    ts = [m["metadata"]["timestamp"] for m in mems]
    assert len(set(ts)) < len(ts)                               # the folder does hold ties
    want = sorted(mems, key=lambda m: m["metadata"]["timestamp"])[:len(mems) - 3]
    arch = MemoryArchiver()
    arch.set_retention_policy(folder, 3, "age")
    with contextlib.redirect_stdout(io.StringIO()):
        got = arch.apply_retention_policies(dry_run=True)
    assert [d["memory_id"] for d in got["details"]] == [m["metadata"]["unique_id"] for m in want]


def test_dropin_routes_the_reference_class_to_the_gpu(golden, fresh, tmp_path):
    """install() rebinds the maintenance methods of a package laid out like the reference's; they then run on the GPU with
    that object's settings and give the golden results."""
    import fei_b200.dropin as D
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    stages = T.STAGES + ("run_maintenance",)
    pkg = tmp_path / "standin" / "memdir_tools"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "utils.py").write_text("MEMDIR_BASE = ''\ndef search_memories(): pass\n")
    (pkg / "search.py").write_text("def search_memories(): pass\n")
    (pkg / "filter.py").write_text("class MemoryFilter: pass\nclass FilterManager: pass\ndef run_filters(): pass\n")
    (pkg / "archiver.py").write_text("class MemoryArchiver:\n" + "".join(f"    def {m}(self, *a, **k): raise AssertionError\n" for m in stages))
    saved = {k: v for k, v in sys.modules.items() if k == "memdir_tools" or k.startswith("memdir_tools.")}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, str(pkg.parent))
    try:
        import memdir_tools.archiver as RA
        import memdir_tools.utils as RU
        D.install()
        assert all(getattr(RA.MemoryArchiver, m).__module__ == "fei_b200.dropin" for m in stages)
        for k, case in enumerate(golden["cases"][-3:]):          # run_maintenance and retention, real runs
            RU.MEMDIR_BASE = base = fresh(f"dropin{k}")
            recs = T.records(base)
            settings = MemoryArchiver()
            T.configure(settings, case["config"])
            arch = RA.MemoryArchiver()                              # a reference object carrying those settings
            arch.__dict__.update(settings.__dict__)
            with contextlib.redirect_stdout(io.StringIO()):
                got = T.run_stage(arch, case["stage"], case["dry_run"])
            _check_case(case, got, recs, base)
    finally:
        sys.path.remove(str(pkg.parent))
        for k in [k for k in sys.modules if k == "memdir_tools" or k.startswith("memdir_tools.")]:
            del sys.modules[k]
        sys.modules.update(saved)
