"""The reference's MemdirFolderManager (memdir_tools/folders.py) over the packed corpus: the methods that read every record of
a folder.

`get_folder_stats` (folders.py:216-318, SURVEY.md section 8(f) row 4): memory counts come from the packed segments, flag counts
from one GPU pass with four flag queries, newest / oldest from the packed wall-clock column, and the tag statistics from
fei_corpus_token_histogram (the `Tags` values tokenised and counted on the GPU).  `list_folders` (:320-380) reads its memory
counts from the packed segments.  `bulk_tag_folder` (:483-587) decides on the GPU which records an add / remove / replace of
tags changes (fei_corpus_tag_edit) and gets back only their Subject and old and new tag strings; the host rewrites those files
with the reference's code.  Folder creation, moving, copying and symlinks are file-system work and stay with the reference."""
from __future__ import annotations

import os
import re
from typing import Any, Dict, List, Tuple

import numpy as np

from .. import packer
from ..program import C_FLAGS, C_FOLDER_SET, C_SLOT, C_STATUS_SET, Cond, ProgramBuilder
from ..regexc import Pattern
from . import utils as U


class MemdirFolderManager:
    def __init__(self):
        U.ensure_memdir_structure()

    def get_folder_stats(self, folder_path: str, include_subfolders: bool = False) -> Dict[str, Any]:
        folder_path = folder_path.replace("\\", "/").strip("/")
        all_folders = U.get_memdir_folders()
        folders_to_process: List[str] = []
        if include_subfolders:
            for folder in all_folders:
                if folder == folder_path or (folder.startswith(folder_path) and folder != folder_path):
                    folders_to_process.append(folder)
        elif folder_path in all_folders or folder_path == "":
            folders_to_process = [folder_path]
        stats: Dict[str, Any] = {
            "folder": folder_path or "Inbox", "total_memories": 0, "memory_counts": {"cur": 0, "new": 0, "tmp": 0},
            "flag_counts": {"S": 0, "R": 0, "F": 0, "P": 0}, "tags": {}, "subfolders": [], "newest_memory": None, "oldest_memory": None,
        }
        pm = packer.packed()
        with pm.lock:
            pm.compact()                                            # whole-corpus statistics run on one corpus in listing order
            pm.report_skipped(folders_to_process, None)
            segs = []                                               # (folder, status, lo, hi) in the reference's iteration order
            for folder in folders_to_process:
                sub = {"folder": folder or "Inbox", "memory_counts": {"cur": 0, "new": 0, "tmp": 0}, "total_memories": 0}
                for status in U.STANDARD_FOLDERS:
                    lo, hi = pm.segments.get((folder, status), (0, 0))
                    k = hi - lo
                    sub["memory_counts"][status] = k; sub["total_memories"] += k
                    stats["total_memories"] += k; stats["memory_counts"][status] += k
                    if k:
                        segs.append((folder, status, lo, hi))
                if include_subfolders and folder != folder_path:
                    stats["subfolders"].append(sub)
            if not segs:
                return stats
            # which packed folder ids are in play (one bit per folder id, as search does for folder restrictions; ids of 64 and
            # above go into the program as a bitmap)
            folder_ids = sorted({int(pm.arrays["fsb"][lo]) & 0xFFFF for _f, _s, lo, _hi in segs})
            fset = 0
            for fid in folder_ids:
                fset |= 1 << fid
            in_folders = Cond(C_FOLDER_SET, set64=fset)
            # flags: one pass, four queries (folders.py:282-284)
            pb = ProgramBuilder()
            for letter in "SRFP":
                pb.add_query([in_folders, Cond(C_FLAGS, pattern=Pattern("exact_contains", letter))])
            counts = pm.corpus.scan_count(pb.build(), 4)
            for letter, cnt in zip("SRFP", counts):
                stats["flag_counts"][letter] = int(cnt)
            # tags: exact key "Tags", value split at "," and stripped piece by piece (folders.py:286-292)
            pb = ProgramBuilder()
            pb.add_query([in_folders, Cond(C_SLOT, pattern=Pattern("regex", "", 0), field="Tags", mode=1)])
            order = {(f, s): k for k, (f, s, _lo, _hi) in enumerate(segs)}
            toks = pm.corpus.token_histogram(pb.build(), ",")
            # dict order = first occurrence in the reference's loop = segment order here, then pack order inside a segment
            seg_of = lambda i: next(k for k, (_f, _s, lo, hi) in enumerate(segs) if lo <= i < hi)
            toks.sort(key=lambda t: (seg_of(t[2] - pm.corpus.global_base), t[2]))
            for raw, cnt, _first in toks:
                stats["tags"][raw.decode("utf-8")] = cnt
            # newest / oldest: strict comparisons, so the first extreme in iteration order wins (folders.py:294-309)
            wall = pm.arrays["wall"]
            best_new = best_old = None
            for _f, _s, lo, hi in segs:
                w = wall[lo:hi]
                i_new, i_old = lo + int(np.argmax(w)), lo + int(np.argmin(w))
                if best_new is None or wall[i_new] > wall[best_new]:
                    best_new = i_new
                if best_old is None or wall[i_old] < wall[best_old]:
                    best_old = i_old
            for key, i in (("newest_memory", best_new), ("oldest_memory", best_old)):
                m = pm.materialize([i], False)[0]
                stats[key] = {"id": m["metadata"]["unique_id"], "subject": m["headers"].get("Subject", "No subject"), "date": m["metadata"]["date"]}
        return stats

    def list_folders(self, parent_folder: str = "", recursive: bool = False) -> List[Dict[str, Any]]:
        """folders.py:320-380: the reference's folder filter, entries and sort; each folder's memory counts are its packed segments'
        sizes (the reference runs get_folder_stats per folder for them), and its unreadable files are printed as those listings do."""
        parent_folder = parent_folder.replace("\\", "/").strip("/")
        all_folders = U.get_memdir_folders()
        if parent_folder:
            if recursive:
                folders = [f for f in all_folders if f.startswith(parent_folder) and f != parent_folder]
            else:
                folders = [f for f in all_folders if f.startswith(parent_folder + "/") and f.count("/") == parent_folder.count("/") + 1]
        else:
            folders = all_folders if recursive else [f for f in all_folders if "/" not in f and f]
        if not parent_folder and not recursive:
            folders = [""] + folders
        pm = packer.packed()
        folder_info = []
        with pm.lock:
            for folder in folders:
                pm.report_skipped([folder], None)
                counts = {}
                for status in U.STANDARD_FOLDERS:
                    lo, hi = pm.segments.get((folder, status), (0, 0))
                    counts[status] = hi - lo
                folder_info.append({"path": folder or "Inbox", "name": os.path.basename(folder) or "Inbox", "is_special": folder in U.SPECIAL_FOLDERS,
                                    "memory_counts": counts, "total_memories": sum(counts.values())})
        folder_info.sort(key=lambda x: (0 if x["is_special"] else 1, x["name"]))
        return folder_info

    def bulk_tag_folder(self, folder_path: str, tags: List[str], statuses: List[str] = None,
                        operation: str = "add") -> Tuple[int, List[Dict[str, Any]]]:
        """folders.py:483-587.  One device call per packed corpus selects the records of the requested directories, decides for
        each whether the operation changes the multiset of its `Tags` pieces, and returns the affected records' Subject and
        ", "-joined old and new tags; no record dict is built.  The affected files are then rewritten in listing order with the
        reference's code (its re.sub template rules included), directory by directory in the order of `statuses`."""
        folder_path = folder_path.replace("\\", "/").strip("/")
        if statuses is None:
            statuses = ["cur"]
        pm = packer.packed()
        with pm.lock:
            listed: List[Tuple[str, Tuple[int, int]]] = []       # (status, listing range) of each listing the reference makes
            for status in statuses:
                pm.ranges([folder_path], [status])               # ValueError for a status the reference's get_memory_path refuses
                pm.report_skipped([folder_path], [status])
                r = pm.segments.get((folder_path, status))
                if r is None and os.path.isdir(U.get_memory_path(folder_path, status)):
                    raise NotImplementedError(f"folder {folder_path!r} is not spelled the way the tree walk lists it")
                listed.append((status, r or (0, 0)))
            if operation not in ("add", "remove", "replace") or not any(b > a for _s, (a, b) in listed):
                return 0, []
            if isinstance(tags, str) and operation == "remove":
                raise NotImplementedError("bulk_tag_folder: tags given as one str (the reference tests substrings) for remove")
            items = list(tags)
            if operation == "remove":
                items = [t for t in items if isinstance(t, str)]            # `piece not in tags`: a non-str never equals a piece
            elif not all(isinstance(t, str) for t in items):
                first = next(a for _s, (a, b) in listed if b > a)
                _edit_one(pm.materialize([first], False)[0]["headers"], items, operation)     # raises as the reference does at its first record
                raise NotImplementedError("bulk_tag_folder: non-str tags")
            try:
                ops = [t.encode("utf-8") for t in items]
            except UnicodeEncodeError:
                raise NotImplementedError("bulk_tag_folder: a tag that is not encodable as UTF-8") from None
            pos, texts = self._tag_edit(pm, folder_path, sorted({s for s, _r in listed}), operation, ops)
            todo = []                                            # (status, listing position, index into texts)
            for status, (a, b) in listed:
                lo, hi = np.searchsorted(pos, a), np.searchsorted(pos, b)
                todo += [(status, p, k) for p, k in zip(pos[lo:hi].tolist(), range(lo, hi))]
            names = [self._file_name(pm, folder_path, status, p) for status, p, _k in todo]
        affected: List[Dict[str, Any]] = []
        touched = set()
        try:
            for (status, _p, k), (filename, uid) in zip(todo, names):
                file_path = os.path.join(U.MEMDIR_BASE, folder_path, status, filename)
                if not os.path.exists(file_path):
                    continue
                subject, old_tags, new_tags_str = texts[k]
                with open(file_path, "r") as f:
                    content = f.read()
                if "Tags:" in content:
                    content = re.sub(r"Tags:.*$", f"Tags: {new_tags_str}", content, flags=re.MULTILINE)
                else:
                    content = re.sub(r"^(.*?)(---)", f"\\1Tags: {new_tags_str}\n\\2", content, flags=re.DOTALL)
                touched.add(status)
                with open(file_path, "w") as f:
                    f.write(content)
                affected.append({"id": uid, "subject": subject, "old_tags": old_tags, "new_tags": new_tags_str})
        finally:
            for status in touched:                               # an in-place write leaves the directory's mtime as it was
                pm.mark_dirty(folder_path, status)
        return len(affected), affected

    @staticmethod
    def _tag_edit(pm: "packer.PackedMemdir", folder: str, statuses: List[str], operation: str, ops: List[bytes]):
        """(listing positions ascending, [(subject, old tags, new tags)] aligned with them) of the records of these directories
        that the operation changes: one fei_corpus_tag_edit per packed corpus (base and delta), tombstones dropped."""
        sbits = 0
        for st in statuses:
            sbits |= 1 << U.STANDARD_FOLDERS.index(st)
        always = Pattern("regex", "", 0)
        pb = ProgramBuilder()
        pb.add_query([Cond(C_SLOT, pattern=always, field="Tags", mode=1, if_missing=1),           # header field 0: Tags
                      Cond(C_SLOT, pattern=always, field="Subject", mode=1, if_missing=1),        # header field 1: Subject
                      Cond(C_FOLDER_SET, set64=1 << pm.folder_ids[folder]), Cond(C_STATUS_SET, set64=sbits)])
        prog = pb.build()
        all_pos, all_texts = [], []
        for corpus, lo in pm._corpora():
            rec, texts = corpus.tag_edit(prog, operation, ops)
            p = pm.pos_of_dev[rec.astype(np.int64) - corpus.global_base + lo]
            keep = np.nonzero(p >= 0)[0]
            all_pos.append(p[keep])
            all_texts += [(s.decode("utf-8") if s is not None else "No subject", o.decode("utf-8"), n.decode("utf-8"))
                          for s, o, n in (texts[k] for k in keep.tolist())]
        pos = np.concatenate(all_pos) if all_pos else np.zeros(0, dtype=np.int64)
        order = np.argsort(pos, kind="stable")
        return pos[order], [all_texts[k] for k in order.tolist()]

    @staticmethod
    def _file_name(pm: "packer.PackedMemdir", folder: str, status: str, p: int) -> Tuple[str, str]:
        """(file name, unique_id) of the record at listing position p, from the directory listing (as materialize has them)."""
        L = pm.segs[(folder, status)].listing
        i = p - pm.segments[(folder, status)][0]
        nb = L.name_bytes(i)
        s0, l0 = int(L.spans[i][0]), int(L.spans[i][1])
        return os.fsdecode(nb), os.fsdecode(nb[s0:s0 + l0])


def _edit_one(headers: Dict[str, str], tags: List[Any], operation: str) -> None:
    """The reference's per-record tag arithmetic (folders.py:531-554) on one record, for operands it cannot hand the device
    (non-str): Python raises exactly where and how the reference does."""
    existing = [tag.strip() for tag in headers["Tags"].split(",")] if "Tags" in headers else []
    updated = existing + [tag for tag in tags if tag not in existing] if operation == "add" else tags
    if sorted(existing) != sorted(updated):
        ", ".join(updated)


def get_folder_stats(folder_path: str, include_subfolders: bool = False) -> Dict[str, Any]:
    return MemdirFolderManager().get_folder_stats(folder_path, include_subfolders)
