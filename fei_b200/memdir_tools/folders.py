"""Folder statistics of the reference's MemdirFolderManager (memdir_tools/folders.py:216-318) over the packed corpus.

Only `get_folder_stats` lives here (SURVEY.md section 8(f) row 4): memory counts come from the packed segments, flag counts
from one GPU pass with four flag queries, newest / oldest from the packed wall-clock column, and the tag statistics from
fei_corpus_token_histogram (the `Tags` values tokenised and counted on the GPU).  Folder creation / moving / bulk operations
are file-system work and stay with the reference."""
from __future__ import annotations

from typing import Any, Dict, List

import numpy as np

from .. import packer
from ..program import C_FLAGS, C_FOLDER_SET, C_SLOT, Cond, ProgramBuilder
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


def get_folder_stats(folder_path: str, include_subfolders: bool = False) -> Dict[str, Any]:
    return MemdirFolderManager().get_folder_stats(folder_path, include_subfolders)
