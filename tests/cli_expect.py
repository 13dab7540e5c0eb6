"""Expected command-line output from list_memories-shaped dicts (the oracle's, oracle/memdir_oracle.py), written the way the
reference writes it: json.dumps(indent=2) and f-strings (memdir_tools/cli.py:41-67, :103-144, search.py:521-594).  Everything is
bytes as print() would send them to a UTF-8 stream with surrogate escapes.  The GPU tests compare fei_b200.memdir_tools.cli and
Corpus.format_records against these; tests/test_cli_expect.py shows they reproduce the reference goldens."""
import hashlib
import json
import os

from oracle import memdir_oracle as mo

COLORS = {"reset": "\033[0m", "bold": "\033[1m", "green": "\033[32m", "yellow": "\033[33m", "red": "\033[31m"}
FLAGS = {"S": "Seen", "R": "Replied", "F": "Flagged", "P": "Priority"}
SEPARATOR = "-" * 34


def colorize(text, color):
    return f"{COLORS.get(color, '')}{text}{COLORS['reset']}"


def enc(text: str) -> bytes:
    return text.encode("utf-8", "surrogateescape")


def _iso(m):
    m = dict(m)
    m["metadata"] = dict(m["metadata"], date=m["metadata"]["date"].isoformat())
    return m


def json_items(mems) -> list:
    """The element of json.dumps(mems, indent=2) for every memory, as format_records writes it (indent of a list element)."""
    return [enc("\n".join("  " + line for line in json.dumps(_iso(m), indent=2).split("\n"))) for m in mems]


def json_list(mems) -> bytes:
    return enc(json.dumps([_iso(m) for m in mems], indent=2) + "\n")


def csv_row(m) -> bytes:
    h, md = m["headers"], m["metadata"]
    row = [md["unique_id"], h.get("Subject", "").replace('"', '""'), md["date"].isoformat(), m["folder"] or "Inbox",
           h.get("Tags", "").replace('"', '""'), h.get("Priority", ""), h.get("Status", ""), "".join(md["flags"])]
    return enc(",".join(f'"{r}"' for r in row) + "\n")


def compact_line(m) -> bytes:
    md = m["metadata"]
    return enc(f"{md['unique_id']} - {md['date'].strftime('%Y-%m-%d')} - {m['headers'].get('Subject', 'No subject')} "
               f"({m['folder'] or 'Inbox'}) {''.join(md['flags'])}\n")


def text_block(m, show_content=True, separator=False) -> bytes:
    md = m["metadata"]
    lines = [colorize(f"Memory ID: {md['unique_id']}", "bold"), f"File: {m['filename']}", f"Date: {md['date'].isoformat()}",
             f"Folder: {m['folder'] or 'Inbox'}", f"Status: {m['status']}",
             f"Flags: {', '.join([FLAGS.get(f, f) for f in md['flags']])}" if md["flags"] else "Flags: None",
             colorize("\nHeaders:", "yellow")]
    lines += [f"  {k}: {v}" for k, v in m["headers"].items()]
    if show_content and "content" in m:
        lines += [colorize("\nContent:", "green"), m["content"]]
    lines.append("")
    if separator:
        lines.append(SEPARATOR)
    return enc("\n".join(lines) + "\n")


def record(m, fmt: str, content: bool, separator: bool = False) -> bytes:
    """One record as Corpus.format_records writes it (fmt: json / csv / compact / text)."""
    if fmt == "json":
        return json_items([m])[0]
    if fmt == "csv":
        return csv_row(m)
    if fmt == "compact":
        return compact_line(m)
    return text_block(m, content, separator)


# ----------------------------------------------------------------------------- golden records
def digest(out: bytes) -> dict:
    """What a golden keeps of a command's stdout: its length, its SHA-256, and the SHA-256 of its lines sorted (equal when only
    the order of records with equal timestamps differs)."""
    return {"bytes": len(out), "sha256": hashlib.sha256(out).hexdigest(),
            "sha256_lines": hashlib.sha256(b"\n".join(sorted(out.split(b"\n")))).hexdigest()}


def tie_groups(base) -> dict:
    """Per directory of the tree ("folder/status"), the file names whose timestamp another file there shares, in listing order:
    os.listdir decides their order, and it depends on the file system."""
    import contextlib
    import io
    out = {}
    with contextlib.redirect_stdout(io.StringIO()):
        for f in mo.memdir_folders(base):
            for st in mo.STATUS_DIRS:
                names = [m["filename"] for m in mo.read_folder(base, f, st, False)]
                ts = [n.split(".")[0] for n in names]
                tied = [n for n, t in zip(names, ts) if ts.count(t) > 1]
                if tied:
                    out[f"{f}/{st}"] = tied
    return out


# ----------------------------------------------------------------------------- commands over the oracle's listing
def _listing(base, folder, status, include_content, ties=None):
    mems = mo.read_folder(base, folder, status, include_content)
    if ties is not None:                        # the order of equal timestamps the golden was recorded with
        rank = {n: k for k, n in enumerate(ties.get(f"{folder}/{status}", []))}
        mems.sort(key=lambda m: (-m["metadata"]["timestamp"], rank.get(m["filename"], 0)))
    return mems


def list_cmd(base, argv, ties=None) -> bytes:
    """`cli list` (cli.py:103-124) on the tree at base."""
    folder, status, content, as_json = "", "cur", False, False
    it = iter(argv[1:])
    for a in it:
        if a in ("-f", "--folder"):
            folder = next(it)
        elif a in ("-s", "--status"):
            status = next(it)
        elif a in ("-c", "--content"):
            content = True
        elif a == "--json":
            as_json = True
    import contextlib, io
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        mems = _listing(base, folder, status, content, ties)
    out = enc(buf.getvalue())
    if not mems:
        return out + enc(colorize(f"No memories found in {folder or 'Inbox'}/{status}", "yellow") + "\n")
    out += enc(colorize(f"Found {len(mems)} memories in {folder or 'Inbox'}/{status}", "bold") + "\n")
    return out + (json_list(mems) if as_json else b"".join(text_block(m, content) for m in mems))


def view_cmd(base, argv, ties=None) -> bytes:
    """`cli view` (cli.py:126-144)."""
    mid, folder = argv[1], ""
    if "-f" in argv:
        folder = argv[argv.index("-f") + 1]
    import contextlib, io
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        mems = [m for st in mo.STATUS_DIRS for m in _listing(base, folder, st, True, ties)]
    out = enc(buf.getvalue())
    for m in mems:
        if mid in (m["filename"], m["metadata"]["unique_id"]):
            return out + text_block(m, True)
    return out + enc(colorize(f"Memory not found: {mid}", "red") + "\n")


def tree_files(base):
    out = []
    for root, _dirs, files in os.walk(base):
        rel = os.path.relpath(root, base)
        out.extend(["" if rel == "." else rel, f] for f in files)
    return sorted(out)


def tree_change(before, after) -> dict:
    """The [folder, file] entries a command removed from the tree and added to it."""
    b, a = set(map(tuple, before)), set(map(tuple, after))
    return {"removed": sorted(map(list, b - a)), "added": sorted(map(list, a - b))}
