"""The oracle's bulk_tag_folder and list_folders against the reference-generated goldens (tests/golden/bulk_tag_golden.json), and
the folder manager's signatures against the reference's, without a GPU."""
import contextlib
import inspect
import io
import os

import pytest

from tests import bulk_tag_tree as T
from tests.conftest import load_golden

_SPECIAL = (".Trash", ".ToDoLater", ".Projects", ".Archive")


@pytest.fixture(scope="module")
def golden():
    return load_golden("bulk_tag_golden.json")


def _fresh(path, digest=None):
    """The golden tree (checked against `digest`, if given) plus the directories the reference's MemdirFolderManager() creates
    (ensure_memdir_structure)."""
    base = str(path / "Memdir")
    T.build_tree(base)
    assert digest is None or T.tree_digest(base) == digest
    for folder in ("",) + _SPECIAL:
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(base, folder, st), exist_ok=True)
    return base


def test_signatures_match_reference(golden):
    from fei_b200.memdir_tools.folders import MemdirFolderManager
    assert set(golden["signatures"]) == set(T.METHODS)
    for name, sig in golden["signatures"].items():
        assert str(inspect.signature(getattr(MemdirFolderManager, name), eval_str=True)) == sig, name


def test_golden_covers_every_case(golden):
    assert [(c["folder"], c["tags"], c["statuses"], c["operation"]) for c in golden["cases"]] == list(T.CASES)
    assert [(x["parent"], x["recursive"]) for x in golden["list_folders"]] == T.LIST_ARGS


@pytest.mark.parametrize("k", range(len(T.CASES)))
def test_oracle_bulk_tag_matches_reference(golden, tmp_path, k):
    from tests import bulk_tag_oracle as bo
    case = golden["cases"][k]
    base = _fresh(tmp_path)

    class Oracle:
        def bulk_tag_folder(self, folder, tags, statuses, op):
            return bo.bulk_tag_folder(base, folder, tags, statuses, op)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        got = T.run_case(Oracle(), T.CASES[k])
    assert got["error"] == case["error"]
    assert got["result"] == case["result"]
    assert out.getvalue() == case["stdout"]
    assert T.tree_digest(base) == case["tree"]


def test_oracle_list_folders_matches_reference(golden, tmp_path):
    from tests import bulk_tag_oracle as bo
    base = _fresh(tmp_path, golden["tree"])
    for want in golden["list_folders"]:
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            got = bo.list_folders(base, want["parent"], want["recursive"])
        assert got == want["folders"], (want["parent"], want["recursive"])
        assert out.getvalue() == want["stdout"]
