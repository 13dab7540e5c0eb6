"""memdir_tools.cli on the GPU: the reference's command line (memdir_tools/cli.py) with its names, arguments and output.

`list`, `view`, `move`, `flag` and `search` run on the packed corpus.  A memory is found by id with one scan (file name or
unique id equal to the argument, cli.py:133-138) instead of reading all three status directories, and every listing or result
is printed from bytes the GPU writes (Corpus.format_records) instead of from per-record dicts.  `create` and `mkdir` are the
reference's file operations.
"""
from __future__ import annotations

import argparse
import os
import sys
from typing import Optional, Sequence

import numpy as np

from .. import _abi, packer
from ..program import C_FOLDER_SET, C_NAME, NAME_FILENAME, NAME_ID, Cond, ProgramBuilder
from ..regexc import Pattern
from . import search as S
from . import utils as U

STANDARD_FOLDERS = U.STANDARD_FOLDERS
FLAGS = U.FLAGS
COLORS = {"reset": "\033[0m", "bold": "\033[1m", "green": "\033[32m", "yellow": "\033[33m", "blue": "\033[34m", "magenta": "\033[35m",
          "cyan": "\033[36m", "red": "\033[31m"}
_FORMATS = {"json": _abi.FEI_FMT_JSON, "csv": _abi.FEI_FMT_CSV, "compact": _abi.FEI_FMT_COMPACT, "text": _abi.FEI_FMT_TEXT}


def colorize(text: str, color: str) -> str:
    return f"{COLORS.get(color, '')}{text}{COLORS['reset']}"


# ----------------------------------------------------------------------------- output
def _write(data: bytes) -> None:
    """Bytes the GPU wrote, to sys.stdout as print() would write the same text under any stdout encoding.  A record whose name is
    not UTF-8 reaches the stream as str with surrogate escapes; those go line by line, so that a strict stream raises at the line
    print() raises at, after the same output."""
    try:
        sys.stdout.write(data.decode("utf-8"))
    except UnicodeDecodeError:
        for line in data.decode("utf-8", "surrogateescape").splitlines(keepends=True):
            sys.stdout.write(line)


def write_records(pm: "packer.PackedMemdir", positions: Sequence[int], fmt: str, content: bool, separator: bool = False) -> None:
    """The records at these listing positions in one output format: the text of print_memory (cli.py:41-67, with the search
    commands' separator line when `separator`), the JSON list of json.dumps(results, indent=2), or the csv / compact lines of
    print_search_results (search.py:554-582) without their header line.  `content`: the memories carry their content."""
    opts = (_abi.FEI_FMT_CONTENT if content else 0) | (_abi.FEI_FMT_SEPARATOR if separator else 0)
    if fmt != "json":
        for data, _ in pm.format_records(positions, _FORMATS[fmt], opts):
            _write(data)
        return
    first = True
    sys.stdout.write("[\n")
    for data, off in pm.format_records(positions, _FORMATS[fmt], opts):
        o = off.tolist()
        parts = [data[o[k]:o[k + 1]] for k in range(len(o) - 1)]
        _write((b"" if first else b",\n") + b",\n".join(parts))
        first = False
    sys.stdout.write("\n]\n")


def print_results(pm: "packer.PackedMemdir", positions: Sequence[int], output_format: str, content: bool) -> None:
    """print_search_results (search.py:521-594) for search hits given as listing positions."""
    if not len(positions):
        print("No matching memories found.")
        return
    if output_format == "csv":
        print(",".join(f'"{h}"' for h in ["ID", "Subject", "Date", "Folder", "Tags", "Priority", "Status", "Flags"]))
    elif output_format not in ("json", "compact"):
        output_format = "text"
        print(colorize(f"Found {len(positions)} matching memories", "bold"))
        print("")
    write_records(pm, positions, output_format, content, separator=output_format == "text")


# ----------------------------------------------------------------------------- lookup
def _check_folder(pm: "packer.PackedMemdir", folder: str) -> bool:
    """Is `folder` a folder of the packed tree?  A directory the tree walk lists under another spelling raises."""
    if folder in pm.folder_ids and folder in pm.folders:
        return True
    if any(os.path.isdir(U.get_memory_path(folder, st)) for st in STANDARD_FOLDERS):
        raise NotImplementedError(f"folder {folder!r} is not spelled the way the tree walk lists it")
    return False


def listing(pm: "packer.PackedMemdir", folder: str, status: str) -> np.ndarray:
    """Listing positions of list_memories(folder, status) (utils.py:202-253), after its `Error processing` lines."""
    U.get_memory_path(folder, status)                          # the reference's ValueError for a status that is not cur / new / tmp
    pm.report_skipped([folder], [status])
    if not _check_folder(pm, folder):
        return np.zeros(0, dtype=np.int64)
    a, b = pm.segments[(folder, status)]
    return np.arange(a, b, dtype=np.int64)


def find_memory(pm: "packer.PackedMemdir", folder: str, memory_id: str) -> Optional[int]:
    """Listing position of the first memory of `folder` over cur, new, tmp whose filename or unique_id equals memory_id (the loop
    of cli.py:132-141), or None; prints the `Error processing` lines of the three listings first.  One scan, two queries."""
    pm.report_skipped([folder], STANDARD_FOLDERS)
    if not _check_folder(pm, folder):
        return None
    ranges = pm.ranges([folder], STANDARD_FOLDERS)
    if not ranges:
        return None
    in_folder = Cond(C_FOLDER_SET, set64=1 << pm.folder_ids[folder])
    pb = ProgramBuilder()
    for which in (NAME_FILENAME, NAME_ID):
        pb.add_query([in_folder, Cond(C_NAME, pattern=Pattern("exact_equals", memory_id), which=which)])
    hits = np.union1d(*pm.scan_hits(pb.build(), 2))
    for a, b in ranges:
        k = int(np.searchsorted(hits, a))
        if k < len(hits) and hits[k] < b:
            return int(hits[k])
    return None


def _find(folder: str, memory_id: str) -> Optional[dict]:
    """The dict (without content) of the memory find_memory finds, or None."""
    pm = packer.packed()
    with pm.lock:
        pos = find_memory(pm, folder, memory_id)
        return pm.materialize([pos], False)[0] if pos is not None else None


# ----------------------------------------------------------------------------- commands
def create_memory(args: argparse.Namespace) -> None:
    headers = {}
    if args.subject:
        headers["Subject"] = args.subject
    if args.tags:
        headers["Tags"] = args.tags
    if args.priority:
        headers["Priority"] = args.priority
    if args.file:
        with open(args.file, "r") as f:
            content = f.read()
    elif args.content:
        content = args.content
    else:
        print(colorize("Enter memory content (Ctrl+D to finish):", "yellow"))
        lines = []
        try:
            while True:
                lines.append(input())
        except EOFError:
            content = "\n".join(lines)
    folder = args.folder if args.folder else ""
    filename = U.save_memory(folder, content, headers, args.flags)
    print(colorize(f"Memory created: {filename}", "green"))
    print(f"In folder: {folder or 'Inbox'}")


def list_memories_cmd(args: argparse.Namespace) -> None:
    folder = args.folder if args.folder else ""
    status = args.status if args.status else "cur"
    pm = packer.packed()
    with pm.lock:
        positions = listing(pm, folder, status)
        if not len(positions):
            print(colorize(f"No memories found in {folder or 'Inbox'}/{status}", "yellow"))
            return
        print(colorize(f"Found {len(positions)} memories in {folder or 'Inbox'}/{status}", "bold"))
        write_records(pm, positions, "json" if args.json else "text", args.content)


def view_memory(args: argparse.Namespace) -> None:
    folder = args.folder if args.folder else ""
    pm = packer.packed()
    with pm.lock:
        pos = find_memory(pm, folder, args.id)                 # --status is not consulted (cli.py:126-144)
        if pos is None:
            print(colorize(f"Memory not found: {args.id}", "red"))
            return
        write_records(pm, [pos], "text", True)


def move_memory_cmd(args: argparse.Namespace) -> None:
    memory = _find(args.source_folder, args.id)
    if memory is None:
        print(colorize(f"Memory not found: {args.id}", "red"))
        return
    source_status = memory["status"]
    if U.move_memory(memory["filename"], args.source_folder, args.target_folder, source_status, args.target_status, args.flags):
        print(colorize(f"Memory {args.id} moved from {args.source_folder or 'Inbox'}/{source_status} to "
                       f"{args.target_folder or 'Inbox'}/{args.target_status}", "green"))
    else:
        print(colorize(f"Failed to move memory {args.id}", "red"))


def search_memories_cmd(args: argparse.Namespace) -> None:
    folders = [args.folder] if args.folder else None
    statuses = [args.status] if args.status else None
    query = S.parse_search_args(args.query)
    if getattr(args, "sort", None):
        query.set_sort(args.sort, getattr(args, "reverse", False))
    if getattr(args, "limit", None):
        query.set_pagination(limit=args.limit, offset=getattr(args, "offset", 0))
    if getattr(args, "with_content", False):
        query.with_content(True)
    output_format = args.format if hasattr(args, "format") else "json" if getattr(args, "json", False) else "text"
    pm = packer.packed()
    with pm.lock:
        positions, _ = S.search_positions(pm, query, folders, statuses)
        if not len(positions):
            print(colorize(f"No memories found matching query: {args.query}", "yellow"))
            return
        print(colorize(f"Found {len(positions)} memories matching query: {args.query}", "bold"))
        if output_format == "text":
            write_records(pm, positions, "text", query.include_content and not args.headers_only, separator=True)
        else:
            print_results(pm, positions, output_format, query.include_content)


def flag_memory(args: argparse.Namespace) -> None:
    folder = args.folder if args.folder else ""
    memory = _find(folder, args.id)
    if memory is None:
        print(colorize(f"Memory not found: {args.id}", "red"))
        return
    current = "".join(memory["metadata"]["flags"])
    if args.add:
        new_flags = "".join(sorted(set(current + args.add)))
    elif args.remove:
        new_flags = "".join(f for f in current if f not in args.remove)
    elif args.set:
        new_flags = args.set
    else:
        print(colorize(f"Current flags: {current}", "green"))
        return
    if U.update_memory_flags(memory["filename"], folder, memory["status"], new_flags):
        print(colorize(f"Memory {args.id} flags updated from '{current}' to '{new_flags}'", "green"))
    else:
        print(colorize(f"Failed to update flags for memory {args.id}", "red"))


def mkdir_cmd(args: argparse.Namespace) -> None:
    path = os.path.join(U.MEMDIR_BASE, args.folder)
    try:
        for st in STANDARD_FOLDERS:
            os.makedirs(os.path.join(path, st), exist_ok=True)
        print(colorize(f"Created memory directory: {args.folder}", "green"))
    except Exception as e:
        print(colorize(f"Error creating directory {args.folder}: {e}", "red"))


def parse_args() -> argparse.Namespace:
    parser = argparse.ArgumentParser(description="Memdir memory management on the GPU")
    sub = parser.add_subparsers(dest="command", help="Command")
    p = sub.add_parser("create", help="Create a memory")
    p.add_argument("-s", "--subject", help="Subject header")
    p.add_argument("-t", "--tags", help="Tags header (comma-separated)")
    p.add_argument("-p", "--priority", choices=["high", "medium", "low"], help="Priority header")
    p.add_argument("-f", "--folder", help="Folder (default: Inbox)")
    p.add_argument("--flags", default="", help="Flag letters")
    p.add_argument("--file", help="Read the content from this file")
    p.add_argument("--content", help="Content")
    p = sub.add_parser("list", help="List the memories of a folder")
    p.add_argument("-f", "--folder", help="Folder (default: Inbox)")
    p.add_argument("-s", "--status", choices=STANDARD_FOLDERS, default="cur", help="Status directory")
    p.add_argument("-c", "--content", action="store_true", help="Include the content")
    p.add_argument("--json", action="store_true", help="JSON output")
    p = sub.add_parser("view", help="Show one memory")
    p.add_argument("id", help="Unique id or file name")
    p.add_argument("-f", "--folder", help="Folder (default: Inbox)")
    p.add_argument("-s", "--status", choices=STANDARD_FOLDERS, help="Status directory (not consulted)")
    p = sub.add_parser("move", help="Move a memory to another folder")
    p.add_argument("id", help="Unique id or file name")
    p.add_argument("source_folder", help="Source folder ('' for Inbox)")
    p.add_argument("target_folder", help="Target folder ('' for Inbox)")
    p.add_argument("-s", "--target-status", choices=STANDARD_FOLDERS, default="cur", help="Target status directory")
    p.add_argument("--flags", help="New flag letters")
    p = sub.add_parser("search", help="Search memories", description="Search memories with the query syntax of memdir_tools.search")
    p.add_argument("query", help="Query string")
    p.add_argument("-f", "--folder", help="Folder (default: all)")
    p.add_argument("-s", "--status", choices=STANDARD_FOLDERS, help="Status directory (default: all)")
    p.add_argument("--headers-only", action="store_true", help="Leave the content out of the text output")
    p.add_argument("--format", choices=["text", "json", "csv", "compact"], default="text", help="Output format")
    p.add_argument("--with-content", action="store_true", help="Include the content")
    p.add_argument("--sort", help="Sort field")
    p.add_argument("--reverse", action="store_true", help="Reverse the sort")
    p.add_argument("--limit", type=int, help="At most this many results")
    p.add_argument("--offset", type=int, default=0, help="Skip this many results (with --limit)")
    p.add_argument("--json", action="store_true", help="Kept for compatibility; --format decides")
    p = sub.add_parser("flag", help="Change the flags of a memory")
    p.add_argument("id", help="Unique id or file name")
    p.add_argument("-f", "--folder", help="Folder (default: Inbox)")
    p.add_argument("--add", help="Flags to add")
    p.add_argument("--remove", help="Flags to remove")
    p.add_argument("--set", help="Flags to set")
    p = sub.add_parser("mkdir", help="Create a folder")
    p.add_argument("folder", help="Folder name")
    args = parser.parse_args()
    if not args.command:
        parser.print_help()
        sys.exit(1)
    return args


def main() -> None:
    U.ensure_memdir_structure()
    args = parse_args()
    commands = {"create": create_memory, "list": list_memories_cmd, "view": view_memory, "move": move_memory_cmd,
                "search": search_memories_cmd, "flag": flag_memory, "mkdir": mkdir_cmd}
    commands[args.command](args)


if __name__ == "__main__":
    main()
