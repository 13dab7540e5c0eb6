"""MemdirFolderManager.bulk_tag_folder and list_folders on the GPU (fei_corpus_tag_edit) against the reference-generated goldens
(tests/golden/bulk_tag_golden.json) and the oracle: the same return value or exception, the same printed lines and the same
tree afterwards.  Every golden case runs on a fresh copy of the seeded tree (tests/bulk_tag_tree.py), once with the header
directory and once with every header parsed from its text (FEI_HDIR=0).  Further cases cover a packed base with a delta, seeded
random operand sets on a synthetic tree of 20 k records, a search right after an edit without inotify, and the drop-in."""
import contextlib
import io
import os
import random
import sys

import pytest

from tests import bulk_tag_tree as T
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return load_golden("bulk_tag_golden.json")


@pytest.fixture
def fresh(gpu, tmp_path, monkeypatch):
    """make(name, build) -> a new tree as the Memdir base; the packed corpora are dropped afterwards."""
    from fei_b200 import packer
    from fei_b200.memdir_tools import utils as U
    bases = []

    def make(name, build=T.build_tree):
        base = str(tmp_path / name / "Memdir")
        build(base)
        monkeypatch.setattr(U, "MEMDIR_BASE", base)
        bases.append(base)
        return base
    yield make
    for b in bases:
        packer.drop(b)


def _manager():
    from fei_b200.memdir_tools.folders import MemdirFolderManager
    return MemdirFolderManager()                              # creates the special folders, as the reference's constructor does


def _run(mgr, case):
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        got = T.run_case(mgr, case)
    return got, out.getvalue()


@pytest.mark.parametrize("hdir", ["1", "0"])
@pytest.mark.parametrize("k", range(len(T.CASES)))
def test_bulk_tag_matches_reference_goldens(golden, fresh, monkeypatch, k, hdir):
    monkeypatch.setenv("FEI_HDIR", hdir)
    case = golden["cases"][k]
    base = fresh(f"case{k}")
    got, out = _run(_manager(), T.CASES[k])
    assert got["error"] == case["error"]
    assert got["result"] == case["result"]                   # every timestamp of the tree is distinct: the order is the listing's
    assert out == case["stdout"]
    assert T.tree_digest(base) == case["tree"]


def test_list_folders_matches_reference_goldens(golden, fresh):
    fresh("lists")
    mgr = _manager()
    for want in golden["list_folders"]:
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            got = mgr.list_folders(want["parent"], want["recursive"])
        assert got == want["folders"], (want["parent"], want["recursive"])
        assert out.getvalue() == want["stdout"]


class _Oracle:
    def __init__(self, base):
        self.base = base

    def bulk_tag_folder(self, *args):
        from tests import bulk_tag_oracle as bo
        return bo.bulk_tag_folder(self.base, *args)


def _oracle_pair(fresh, name, build):
    """The same tree twice: one for the GPU (the Memdir base), one for the oracle; both with the directories the folder
    manager's constructor creates."""
    oracle_base = fresh(name + "_oracle", build)
    for folder in ("", ".Trash", ".ToDoLater", ".Projects", ".Archive"):
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(oracle_base, folder, st), exist_ok=True)
    return fresh(name, build), oracle_base


def _same_details(got, want, base):
    """Equal results, with details compared per directory modulo the order of records that share a timestamp."""
    assert got[0] == want[0]
    ts = {}
    for root, _d, files in os.walk(base):
        for f in files:
            ts[f.split(".")[1]] = int(f.split(".")[0])
    key = lambda d: (ts.get(d["id"], 0), sorted(d.items()))          # noqa: E731
    assert sorted(got[1], key=key) == sorted(want[1], key=key)
    assert [ts.get(d["id"]) for d in got[1]] == [ts.get(d["id"]) for d in want[1]]


def _add_files(base, k0, n):
    for k in range(n):
        name = f"{T.NOW_TS + 1000 + k0 + k}.{0xD0000000 + k0 + k:08x}.late:2,"
        tags = ["python, late", "", "late", None][k % 4]
        head = f"Subject: late {k}\n" + (f"Tags: {tags}\n" if tags is not None else "")
        with open(os.path.join(base, "cur", name), "w") as f:
            f.write(head + "---\nlate body\n")


def test_bulk_tag_on_base_and_delta(fresh):
    """Files added after the first pack go to the delta corpus; both corpora take part, in listing order."""
    from fei_b200 import packer
    base, obase = _oracle_pair(fresh, "delta", T.build_tree)
    mgr = _manager()
    with contextlib.redirect_stdout(io.StringIO()):
        packer.packed()
    for b in (base, obase):
        _add_files(b, 0, 12)
        os.remove(os.path.join(b, "cur", sorted(os.listdir(os.path.join(b, "cur")))[3]))      # a tombstone in the base
    pm = packer.packed()
    assert pm.delta is not None and pm.n_delta > 0
    for case in [("", ["late", "python"], ["cur", "new"], "add"), ("", ["python"], None, "remove"), ("", ["z"], None, "replace")]:
        got, out = _run(mgr, case)
        want, wout = _run(_Oracle(obase), case)
        assert got == want and out == wout, case
        assert T.tree_digest(base) == T.tree_digest(obase), case


def test_random_operands_on_synthetic_tree(fresh):
    """Seeded operand sets for add, remove and replace on a 20 k record synthetic tree, one after the other on the same tree
    (each edit is re-synced before the next), against the oracle on a copy."""
    from fei_b200 import synth
    from oracle import memdir_oracle as mo
    base, obase = _oracle_pair(fresh, "synth", lambda b: synth.write_memdir_native(b, 0xB7A6, 0, 20000))
    mgr = _manager()
    with contextlib.redirect_stdout(io.StringIO()):
        vocab = sorted(mo.folder_stats(obase, "", True)["tags"])
    rng = random.Random(20261018)
    for step in range(9):
        op = ("add", "remove", "replace")[step % 3]
        folder = rng.choice(synth.FOLDERS)
        statuses = rng.sample(["cur", "new", "tmp"], rng.randint(1, 3))
        tags = rng.sample(vocab, rng.randint(0, 4)) + (["brand-new"] if rng.random() < 0.5 else [])
        if rng.random() < 0.3 and tags:
            tags.append(tags[0])                              # a repeated operand
        case = (folder, tags, statuses, op)
        got, out = _run(mgr, case)
        want, wout = _run(_Oracle(obase), case)
        assert got["error"] is None and want["error"] is None and out == wout, case
        _same_details(got["result"], want["result"], obase)
        assert T.tree_digest(base) == T.tree_digest(obase), case


def test_search_sees_the_edit_without_inotify(fresh, monkeypatch):
    """An in-place rewrite leaves the directory's mtime alone: the edit marks its directories, so the next search reads the
    rewritten files even without inotify and long before the periodic full check."""
    from fei_b200.memdir_tools.search import SearchQuery, search_memories
    from oracle import memdir_oracle as mo
    monkeypatch.setenv("FEI_INOTIFY", "0")
    monkeypatch.setenv("FEI_REVALIDATE_S", "3600")
    base = fresh("inotify")
    mgr = _manager()
    q = SearchQuery().add_condition("Tags", "has_tag", "brand-new")
    with contextlib.redirect_stdout(io.StringIO()):
        assert search_memories(q) == []
        count, _ = mgr.bulk_tag_folder("", ["brand-new"], ["cur", "new"], "add")
        got = search_memories(q)
        mems = mo.listing(base, None, None, False)
    want = [mems[i] for i in mo.run_search(mems, q.conditions)]
    assert 0 < len(want) <= count                             # a file without `---` is counted but written back unchanged
    assert got == want


def test_operand_limits_raise_not_implemented(fresh):
    fresh("limits")
    mgr = _manager()
    with contextlib.redirect_stdout(io.StringIO()):
        with pytest.raises(NotImplementedError):
            mgr.bulk_tag_folder("", [f"t{k}" for k in range(65)], None, "add")
        with pytest.raises(NotImplementedError):
            mgr.bulk_tag_folder("", ["x" * 4097], None, "add")
        with pytest.raises(NotImplementedError):
            mgr.bulk_tag_folder("", "ab", None, "remove")


def test_dropin_routes_the_reference_folder_manager_to_the_gpu(golden, fresh, tmp_path):
    """install() rebinds get_folder_stats, list_folders and bulk_tag_folder of a package laid out like the reference's; they
    then give the golden results."""
    import fei_b200.dropin as D
    from oracle import memdir_oracle as mo
    pkg = tmp_path / "standin" / "memdir_tools"
    pkg.mkdir(parents=True)
    (pkg / "__init__.py").write_text("")
    (pkg / "utils.py").write_text("MEMDIR_BASE = ''\ndef search_memories(): pass\n")
    (pkg / "search.py").write_text("def search_memories(): pass\n")
    (pkg / "filter.py").write_text("class MemoryFilter: pass\nclass FilterManager: pass\ndef run_filters(): pass\n")
    (pkg / "folders.py").write_text("class MemdirFolderManager:\n" + "".join(f"    def {m}(self, *a, **k): raise AssertionError\n" for m in T.METHODS))
    saved = {k: v for k, v in sys.modules.items() if k == "memdir_tools" or k.startswith("memdir_tools.")}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, str(pkg.parent))
    try:
        import memdir_tools.folders as RF
        import memdir_tools.utils as RU
        D.install()
        assert all(getattr(RF.MemdirFolderManager, m).__module__ == "fei_b200.dropin" for m in T.METHODS)
        RU.MEMDIR_BASE = base = fresh("dropin")
        _manager()
        ref = RF.MemdirFolderManager()
        for want in golden["list_folders"]:
            with contextlib.redirect_stdout(io.StringIO()):
                assert ref.list_folders(want["parent"], want["recursive"]) == want["folders"]
        with contextlib.redirect_stdout(io.StringIO()):
            assert ref.get_folder_stats(".Projects", True)["total_memories"] == mo.folder_stats(base, ".Projects", True)["total_memories"]
        case = golden["cases"][0]
        got, out = _run(ref, T.CASES[0])
        assert got["result"] == case["result"] and out == case["stdout"]
        assert T.tree_digest(base) == case["tree"]
    finally:
        sys.path.remove(str(pkg.parent))
        for k in [k for k in sys.modules if k == "memdir_tools" or k.startswith("memdir_tools.")]:
            del sys.modules[k]
        sys.modules.update(saved)
