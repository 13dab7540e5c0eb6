"""Write tests/golden/bulk_tag_golden.json from the reference's MemdirFolderManager (memdir_tools/folders.py).

Run on a machine that has the reference project:  python tests/golden/make_golden_bulk_tag.py /path/to/reference

The tree is tests/bulk_tag_tree.py's seeded tree.  For each of bulk_tag_tree.CASES, on a fresh copy of the tree, the golden
records bulk_tag_folder's return value or exception (type and message), what it printed and the digest of the tree it leaves.
It also records list_folders for bulk_tag_tree.LIST_ARGS on the fresh tree, with what each call printed, and the reference's
signatures of the folder manager methods this project implements.  One case per line."""
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

from tests import bulk_tag_tree as T          # noqa: E402


def main(reference: str) -> None:
    sys.path.insert(0, reference)
    import memdir_tools.folders as rf
    import memdir_tools.utils as ru

    def manager(base):
        ru.MEMDIR_BASE = rf.MEMDIR_BASE = base
        return rf.MemdirFolderManager()

    head = {"seed": T.SEED, "signatures": {m: str(inspect.signature(getattr(rf.MemdirFolderManager, m))) for m in T.METHODS}}
    cases, lists = [], []
    with tempfile.TemporaryDirectory() as tmp:
        base = os.path.join(tmp, "fresh", "Memdir")
        T.build_tree(base)
        head["tree"] = T.tree_digest(base)
        mgr = manager(base)
        for parent, recursive in T.LIST_ARGS:
            out = io.StringIO()
            with contextlib.redirect_stdout(out):
                got = mgr.list_folders(parent, recursive)
            lists.append({"parent": parent, "recursive": recursive, "folders": got, "stdout": out.getvalue()})
        for k, case in enumerate(T.CASES):
            base = os.path.join(tmp, f"case{k}", "Memdir")
            T.build_tree(base)
            mgr = manager(base)
            out = io.StringIO()
            with contextlib.redirect_stdout(out):
                got = T.run_case(mgr, case)
            folder, tags, statuses, op = case
            cases.append({"folder": folder, "tags": tags, "statuses": statuses, "operation": op, **got, "stdout": out.getvalue(),
                          "tree": T.tree_digest(base)})
    with open(os.path.join(HERE, "bulk_tag_golden.json"), "w") as f:
        f.write(json.dumps(head)[:-1] + ', "list_folders": [\n' + ",\n".join(json.dumps(x, ensure_ascii=False) for x in lists)
                + '\n], "cases": [\n' + ",\n".join(json.dumps(c, ensure_ascii=False) for c in cases) + "\n]}\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_bulk_tag.py <directory holding the reference's memdir_tools package>")
    main(sys.argv[1])
