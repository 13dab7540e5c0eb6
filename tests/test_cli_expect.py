"""CPU checks of the command-line layer: tests/cli_expect.py reproduces the reference goldens of `list` and `view`
(tests/golden/cli_golden.json) from the oracle's dicts, libfeiscan exports the formatter, and dropin.install() rebinds the
reference command line's functions."""
import ctypes
import os
import subprocess
import sys

import pytest

from tests import cli_expect as X
from tests.conftest import load_golden
from tests.memdir_util import build_tree

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    return load_golden("cli_golden.json")


def test_expected_output_reproduces_the_reference_goldens(golden, tmp_path):
    """Every golden `list` / `view` case, over the golden tree with the reference's order of equal timestamps."""
    base = str(tmp_path / "Memdir")
    build_tree(base)
    from fei_b200.memdir_tools import utils as U
    U.set_memdir_base(base)
    U.ensure_memdir_structure()
    n = 0
    for case in golden["cases"]:
        argv = case["argv"]
        if case["kind"] != "cli" or argv[0] not in ("list", "view"):
            continue
        fn = X.list_cmd if argv[0] == "list" else X.view_cmd
        assert X.digest(fn(base, argv, golden["ties"]))["sha256"] == case["sha256"], argv
        n += 1
    assert n >= 18


def test_json_items_join_to_json_dumps():
    from datetime import datetime
    m = {"filename": "1.a.h:2,", "folder": "", "status": "cur", "headers": {}, "metadata": {"timestamp": 1, "unique_id": "a",
         "hostname": "h\udcff", "flags": [], "date": datetime(2024, 1, 2, 3, 4, 5)}}
    m2 = dict(m, headers={"K": "v\U0001F409"}, metadata=dict(m["metadata"], flags=["F", "S"]), content="c\x01")
    assert b"[\n" + b",\n".join(X.json_items([m, m2])) + b"\n]\n" == X.json_list([m, m2])


def test_library_exports_the_formatter():
    lib = ctypes.CDLL(os.path.join(REPO, "fei_b200", "libfeiscan.so"))
    assert hasattr(lib, "fei_corpus_format_records")


_STANDIN = {
    "__init__.py": "",
    "utils.py": "import os\nMEMDIR_BASE = os.path.join(os.getcwd(), 'Memdir')\n"
                "def search_memories(query, folders=None, statuses=None, headers_only=False): raise AssertionError('unpatched')\n",
    "search.py": "def search_memories(query, folders=None, statuses=None, debug=False): raise AssertionError('unpatched')\n"
                 "def main(): raise AssertionError('unpatched')\n",
    "filter.py": "class MemoryFilter:\n    def matches(self, memory): raise AssertionError('unpatched')\n"
                 "class FilterManager:\n    def process_memories(self, folders=None, statuses=None, dry_run=False): raise AssertionError('unpatched')\n"
                 "def run_filters(dry_run=False): raise AssertionError('unpatched')\n",
    "cli.py": "".join(f"def {n}(args): raise AssertionError('unpatched')\n" for n in
                      ("list_memories_cmd", "view_memory", "move_memory_cmd", "search_memories_cmd", "flag_memory", "create_memory", "mkdir_cmd")),
    "__main__.py": "from memdir_tools.cli import view_memory\n",
}


def test_dropin_install_patches_the_reference_cli(tmp_path):
    """install() rebinds the five command functions of the reference cli and search.main, names imported before install()
    included; create and mkdir stay the reference's."""
    pkg = tmp_path / "pkg" / "memdir_tools"
    pkg.mkdir(parents=True)
    for name, src in _STANDIN.items():
        (pkg / name).write_text(src)
    code = (
        "import sys, os; os.chdir(%r); sys.path.insert(0, %r); sys.path.insert(0, %r); sys.dont_write_bytecode = True;"
        "import memdir_tools.__main__ as MM, memdir_tools.cli as C, memdir_tools.search as S;"
        "from memdir_tools.search import main as early_main;"
        "import fei_b200.dropin as D; D.install();"
        "names = ('list_memories_cmd', 'view_memory', 'move_memory_cmd', 'search_memories_cmd', 'flag_memory');"
        "assert all(getattr(C, n).__module__ == 'fei_b200.dropin' and getattr(C, n).__name__ == n for n in names);"
        "assert C.create_memory.__module__ == 'memdir_tools.cli' and C.mkdir_cmd.__module__ == 'memdir_tools.cli';"
        "assert S.main.__module__ == 'fei_b200.dropin' and MM.view_memory is C.view_memory;"
        "assert sys.modules['__main__'].__dict__.get('early_main', S.main) is S.main; print('patched')"
    ) % (str(tmp_path), str(tmp_path / "pkg"), REPO)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "patched" in out.stdout, out.stderr[-2000:]
