"""Folder predicates past 64 folders: `folder:` conditions of search_memories and get_folder_stats on a tree of about 80 folders,
after folders were created and removed so that the packed folder ids (handed out once, never reused) run well past 64.  Those
sets travel as a bitmap in the program head (fei_prog_cond.off_set_words).  Checked against the oracle on the same tree."""
import contextlib
import io
import os
import random
import shutil

import pytest

from oracle import memdir_oracle as mo
from tests.memdir_util import key_of

pytestmark = pytest.mark.gpu

_TAGS = ["python", "ai, python", "work", "", "misc,ai"]


def _write_folder(base, folder, rng, n):
    for st in ("cur", "new", "tmp"):
        os.makedirs(os.path.join(base, folder, st), exist_ok=True)
    for k in range(n):
        ts = 1700000000 + rng.randint(0, 40_000_000)
        flags = rng.choice(["", "S", "F", "SP", "R"])
        st = "cur" if k % 4 else "new"
        text = f"Subject: note {k} of {folder or 'Inbox'}\nTags: {rng.choice(_TAGS)}\n---\nbody {rng.random():.6f}\n"
        with open(os.path.join(base, folder, st, f"{ts}.{rng.getrandbits(32):08x}.box:2,{flags}"), "w") as f:
            f.write(text)


@pytest.fixture(scope="module")
def tree(gpu, tmp_path_factory):
    from fei_b200 import packer
    from fei_b200.memdir_tools import utils as U
    base = str(tmp_path_factory.mktemp("folder_sets") / "Memdir")
    rng = random.Random(64)
    folders = [""] + [f".F{k:02d}" for k in range(60)] + [f".F{k:02d}/sub{j}" for k in range(0, 20, 2) for j in range(2)]
    for f in folders:
        _write_folder(base, f, rng, 4)
    old = U.MEMDIR_BASE
    U.set_memdir_base(base)
    with contextlib.redirect_stdout(io.StringIO()):
        packer.packed()                                          # ids 0 .. 80 handed out
        for k in range(40, 50):                                  # folders go away, new ones arrive: ids past 80
            shutil.rmtree(os.path.join(base, f".F{k:02d}"))
        for k in range(12):
            _write_folder(base, f".New{k:02d}" + ("/deep" if k % 3 == 0 else ""), rng, 3)
        pm = packer.packed()
    assert max(pm.folder_ids[f] for f in pm.folders) >= 90
    yield base
    packer.drop(base)
    U.set_memdir_base(old)


def _search(conds):
    from fei_b200.memdir_tools.search import SearchQuery, search_memories
    q = SearchQuery()
    for f, op, v in conds:
        q.add_condition(f, op, v)
    return search_memories(q)


@pytest.mark.parametrize("conds", [
    [("folder", "=", ".New07")],
    [("folder", "=", ".F05")],
    [("folder", "contains", "new")],
    [("folder", "contains", "sub1")],
    [("folder", "matches", r"^\.(F5[0-9]|New0[0-5])")],
    [("folder", "matches", r"deep$"), ("flags", "has_flag", "S")],
    [("folder", "!=", ".F03")],
    [("folder", "startswith", ".F1")],
])
def test_folder_conditions_past_64_folders(tree, conds):
    with contextlib.redirect_stdout(io.StringIO()):
        got = _search(conds)
        mems = mo.listing(tree, None, None, False)
    want = [mems[i] for i in mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in conds])]
    assert [key_of(m) for m in got] == [key_of(m) for m in want]
    assert want


@pytest.mark.parametrize("folder_path", ["", ".New03", ".F1", ".F04"])
def test_folder_stats_past_64_folders(tree, folder_path):
    from fei_b200.memdir_tools.folders import MemdirFolderManager
    with contextlib.redirect_stdout(io.StringIO()):
        got = MemdirFolderManager().get_folder_stats(folder_path, include_subfolders=True)
        want = mo.folder_stats(tree, folder_path, include_subfolders=True)
    assert got == want
    assert list(got["tags"]) == list(want["tags"])
