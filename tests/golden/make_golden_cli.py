"""Write tests/golden/cli_golden.json from the reference's command lines (memdir_tools/cli.py main, memdir_tools/search.py main).

Run on a machine that has the reference project:  TZ=UTC python tests/golden/make_golden_cli.py /path/to/reference

Every case runs on a fresh copy of the golden Memdir tree (the synthetic records plus make_golden_memdir.ADVERSARIAL): the
recorded argv goes through the unmodified reference, and the golden keeps the digest of its stdout (cli_expect.digest: length,
SHA-256, SHA-256 of the sorted lines), the stdout itself (base64) when it is short, the exception it raised if any and, for
`move` / `flag`, the files of the tree they removed and added (cli_expect.tree_change).  `ties` lists, per directory, the records with equal timestamps in the order
they were listed in: os.listdir decides it, and it depends on the file system."""
import base64
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.dont_write_bytecode = True
os.environ["TZ"] = "UTC"
time.tzset()

from tests.cli_expect import digest, tie_groups, tree_change, tree_files   # noqa: E402
from tests.golden.make_golden_memdir import build_corpus   # noqa: E402

SHORT = 600                                              # stdout of at most this many bytes is kept whole

CLI = [
    ["list"], ["list", "-s", "new"], ["list", "-s", "tmp"], ["list", "--json"], ["list", "-s", "new", "-c"], ["list", "-s", "new", "-c", "--json"],
    ["list", "-f", ".Projects/AI"], ["list", "-f", ".Projects/AI", "-s", "new", "--json", "-c"], ["list", "-f", "no-such-folder"],
    ["list", "-f", ".Trash"],
    ["view", "adv00001"], ["view", "1700000504.adv00006.hostA:2,F"], ["view", "ADV00001"], ["view", "adv00003"],
    ["view", "adv00004", "-f", ".Projects/AI", "-s", "tmp"], ["view", "adv00009"], ["view", "adv00014"], ["view", "nope"],
    ["move", "adv00002", "", ".Archive", "--flags", "SR"], ["move", "adv00003", "", ".Projects/AI", "-s", "new"],
    ["move", "adv00404", "", ".Archive"],
    ["flag", "adv00001", "--add", "RP"], ["flag", "adv00006", "--remove", "F"], ["flag", "adv00012", "--set", "S"], ["flag", "adv00010"],
    ["flag", "adv00004", "-f", ".Projects/AI", "--add", "F"], ["flag", "missing", "--add", "F"],
    ["search", "#python"], ["search", "#python", "--format", "json"], ["search", "#python", "--format", "csv"],
    ["search", "#python", "--format", "compact"], ["search", "#python", "--format", "csv", "--sort", "subject"],
    ["search", "#python", "--format", "compact", "--sort", "date", "--reverse"], ["search", "+F", "--format", "compact", "--limit", "3", "--offset", "2"],
    ["search", "+F", "--format", "compact", "--offset", "2"], ["search", "python", "--with-content"],
    ["search", "python", "--with-content", "--headers-only"], ["search", "#python", "--json"],
    ["search", "dup", "--format", "json", "--with-content"], ["search", "nothing-matches-xyz"],
    ["search", "#python", "-f", ".Projects/AI", "--format", "json"], ["search", "+S", "-s", "new", "--format", "csv", "--with-content"],
    ["search", "#python", "--format", "compact", "--sort", "due"],
]
SEARCH_MAIN = [
    ["--tags", "python"], ["--flags", "F", "--format", "compact"], ["--priority", "high", "--format", "csv"],
    ["sort:-date", "limit:3", "python", "--format", "compact"], ["#python", "--format", "json", "--limit", "2"],
    ["zzz-nothing"], ["python", "--with-content"], ["--tags", "python,learning", "--format", "json", "--with-content"],
]


def run(fn, argv):
    buf = io.BytesIO()
    out = io.TextIOWrapper(buf, encoding="utf-8", errors="surrogateescape", newline="\n", write_through=True)
    old = sys.argv
    sys.argv = argv
    exc = None
    try:
        with contextlib.redirect_stdout(out):
            fn()
    except Exception as e:
        exc = type(e).__name__
    finally:
        sys.argv = old
    out.flush()
    return buf.getvalue(), exc


def main(reference: str) -> None:
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        sys.path.insert(0, reference)
        import memdir_tools.cli as rc
        import memdir_tools.search as rs
        import memdir_tools.utils as ru
        base = os.path.join(tmp, "Memdir")
        assert ru.MEMDIR_BASE == base
        cases = []

        def fresh():
            shutil.rmtree(base, ignore_errors=True)
            build_corpus(base)
            ru.ensure_memdir_structure()                   # what main() does first: the special folders exist in every case

        fresh()
        ties = tie_groups(base)
        for kind, argvs, fn in (("cli", CLI, rc.main), ("search", SEARCH_MAIN, rs.main)):
            for argv in argvs:
                fresh()
                before = tree_files(base)
                out, exc = run(fn, [kind] + argv)
                case = {"kind": kind, "argv": argv, "exception": exc, **digest(out)}
                if len(out) <= SHORT:
                    case["stdout"] = base64.b64encode(out).decode()
                if argv[0] in ("move", "flag"):
                    case["tree"] = tree_change(before, tree_files(base))
                cases.append(case)
    with open(os.path.join(HERE, "cli_golden.json"), "w") as f:
        f.write('{"generator": "tests/golden/make_golden_cli.py", "ties": ' + json.dumps(ties, sort_keys=True) + ',\n"cases": [\n')
        f.write(",\n".join(json.dumps(c) for c in cases))
        f.write("\n]}\n")
    print("wrote cli_golden.json:", len(cases), "cases")


if __name__ == "__main__":
    main(sys.argv[1])
