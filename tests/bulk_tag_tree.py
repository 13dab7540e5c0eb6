"""The seeded Memdir tree of the bulk tag goldens (tests/golden/make_golden_bulk_tag.py, bulk_tag_golden.json), the cases they
run and a runner shared by the golden maker, the oracle test and the GPU test.

Besides seeded ordinary records, the tree holds the records whose tag edit is easy to get wrong: `Tags:` with an empty value,
no `---` at all, CRLF line ends, a repeated `Tags` key (the last line wins, and every line is rewritten), an `Old-Tags:` header
and a `Tags:` line inside the body (both rewritten too), a lower-case `tags:` key and a ` Tags :` key (neither contains
"Tags:", so a `Tags` line is inserted before `---`), Unicode whitespace around pieces, non-ASCII tags, `a,,b`, `a, a`, an
invalid UTF-8 file (printed and skipped by every listing) and, in `.Projects/Alpha`, a tag holding a backslash escape on an old
record, so that the edit fails in `re.sub` after the newer records were rewritten.  Every timestamp is distinct, so the listing
order does not depend on the file system."""
import os
import random

from tests.maintenance_tree import tree_digest          # noqa: F401  (re-exported for the golden maker and the tests)

SEED = 20261018
NOW_TS = 1781524800                                      # 2026-06-15 12:00:00 UTC
LAYOUT = {"": (30, 6), ".Projects": (18, 4), ".Projects/Alpha": (10, 2), ".Trash": (6, 0), ".ToDoLater/Later": (5, 2)}
EMPTY_FOLDERS = [".Empty"]
_TAGS = [None, "python", "Python, work", "misc", "work,urgent", "python, ai", "notes", "ai, python, misc", "x, y", "a"]

# (folder, statuses, header lines or None for no `---`, body, line end)
SPECIAL = [
    ("", "cur", ["Subject: empty tags", "Tags:"], "body", "\n"),
    ("", "cur", None, "no separator here\nTags in prose only", "\n"),
    ("", "cur", ["Subject: crlf", "Tags: python, crlf"], "crlf body", "\r\n"),
    ("", "cur", ["Subject: twice", "Tags: first", "Priority: high", "Tags: python, second"], "body", "\n"),
    ("", "cur", ["Subject: old tags", "Old-Tags: q", "Tags: misc"], "body", "\n"),
    ("", "cur", ["Subject: body tags", "Tags: ai"], "text\nTags: in the body\nmore", "\n"),
    ("", "cur", ["Subject: lower key", "tags: python"], "body", "\n"),
    ("", "cur", ["Subject: spaced key", " Tags : python, spaced"], "body", "\n"),
    ("", "cur", ["Subject: unicode space", "Tags:  python ,　café , x"], "body", "\n"),
    ("", "cur", ["Subject: non-ascii", "Tags: café, 日本, python"], "body", "\n"),
    ("", "cur", ["Subject: empty piece", "Tags: a,,b"], "body", "\n"),
    ("", "cur", ["Subject: doubled", "Tags: a, a"], "body", "\n"),
    ("", "cur", ["Tags: python, no subject"], "body", "\n"),
    ("", "new", ["Subject: new one", "Tags: ai, work"], "body", "\n"),
    (".Projects", "cur", ["Subject: group ref", "tags: g"], "body", "\n"),
    (".Projects/Alpha", "cur", ["Subject: escape", "Tags: old, \\d"], "body", "\n"),
]
INVALID_UTF8 = ("", "cur")


def _write(path: str, text: str, eol: str) -> None:
    with open(path, "wb") as f:
        f.write(text.replace("\n", eol).encode("utf-8"))


def build_tree(base: str) -> None:
    rng = random.Random(SEED)
    used = set()

    def stamp(old: bool = False) -> int:
        while True:
            ts = NOW_TS - (rng.randint(2000, 3000) * 86400 if old else rng.randint(0, 1500 * 86400))
            if ts not in used:
                used.add(ts)
                return ts

    i = 0
    for folder, (n_cur, n_new) in LAYOUT.items():
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(base, folder, st), exist_ok=True)
        for st, n in (("cur", n_cur), ("new", n_new)):
            for _ in range(n):
                lines = [f"Subject: Memory {i} in {folder or 'Inbox'}", "Date: 2026-01-01T00:00:00"]
                tags = rng.choice(_TAGS)
                if tags is not None:
                    lines.append(f"Tags: {tags}")
                name = f"{stamp()}.{rng.getrandbits(32):08x}.host{i % 3}:2,{rng.choice(['', 'S', 'F', 'RS'])}"
                _write(os.path.join(base, folder, st, name), "\n".join(lines) + "\n---\nbody of memory %d\n" % i, "\n")
                i += 1
    for k, (folder, st, lines, body, eol) in enumerate(SPECIAL):
        name = f"{stamp(old=folder == '.Projects/Alpha')}.{0xA0000000 + k:08x}.special:2,"
        text = body + "\n" if lines is None else "\n".join(lines) + "\n---\n" + body + "\n"
        _write(os.path.join(base, folder, st, name), text, eol)
    folder, st = INVALID_UTF8
    with open(os.path.join(base, folder, st, f"{stamp()}.badbad00.special:2,"), "wb") as f:
        f.write(b"Subject: broken \xff\xfe\nTags: python\n---\nbody\n")
    for folder in EMPTY_FOLDERS:
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(base, folder, st), exist_ok=True)


# (folder_path, tags, statuses, operation): every case runs on a fresh copy of the tree
CASES = [
    ("", ["python"], None, "add"),
    ("", ["work", "fresh", "work"], ["cur", "new"], "add"),
    ("", ["python", "a", ""], None, "remove"),
    ("", [5, "misc"], ["cur", "new"], "remove"),
    ("", ["x", "y"], None, "replace"),
    ("", [], None, "replace"),
    ("", ["a", "a"], None, "replace"),
    ("", "ab", None, "add"),
    ("", [5], None, "add"),
    ("", ["a", 5], None, "replace"),
    ("", ["python"], ["cur", "tmp"], "merge"),
    ("", ["python"], ["cur", "bogus"], "add"),
    (".Nope", ["python"], None, "add"),
    (".Projects/Alpha", ["z"], None, "add"),
    (".Projects", ["\\1"], None, "add"),
    ("", ["python"], ["cur", "cur"], "remove"),
    ("", ["café", "日本"], None, "remove"),
    ("", ["python", "ai"], ["new", "cur"], "replace"),
    ("/.Projects/", ["misc"], None, "add"),
    ("\\.ToDoLater\\Later", ["later"], ["cur", "new", "tmp"], "add"),
    (".Trash", ["python"], None, "remove"),
]
LIST_ARGS = [("", False), ("", True), (".Projects", False), (".Projects", True), (".ToDoLater", False), (".Nope", True)]
METHODS = ("get_folder_stats", "list_folders", "bulk_tag_folder")


def run_case(manager, case):
    """{"result", "error"} of one bulk_tag_folder call; stdout is captured by the caller."""
    folder, tags, statuses, op = case
    try:
        count, details = manager.bulk_tag_folder(folder, tags, statuses, op)
        return {"result": [count, details], "error": None}
    except Exception as e:                               # noqa: BLE001  (the reference's exceptions are part of its behaviour)
        return {"result": None, "error": [type(e).__name__, str(e)]}
