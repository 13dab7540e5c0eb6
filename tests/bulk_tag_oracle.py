"""TEST INFRASTRUCTURE — CPU restatement of the reference's folder listing and bulk tag edit, next to the oracle
(oracle/memdir_oracle.py), whose directory listing, header parsing and folder statistics it reuses:

  list_folders       <- folders.MemdirFolderManager.list_folders       (folders.py:320-380)
  bulk_tag_folder    <- folders.MemdirFolderManager.bulk_tag_folder    (folders.py:483-587)

Pinned by tests/golden/bulk_tag_golden.json, produced by running the unmodified reference on the same tree
(tests/golden/make_golden_bulk_tag.py).  Only tests and tools import it; it is the checker of fei_corpus_tag_edit and the host
rewrite, never the thing measured or shipped."""
import os
import re
from typing import Any, Dict, List, Optional, Tuple

from oracle.memdir_oracle import STATUS_DIRS, folder_stats, memdir_folders, read_folder


def list_folders(base: str, parent_folder: str = "", recursive: bool = False) -> List[Dict[str, Any]]:
    """MemdirFolderManager.list_folders (folders.py:320-380) on the tree at `base`: the memory counts of get_folder_stats."""
    parent_folder = parent_folder.replace("\\", "/").strip("/")
    all_folders = memdir_folders(base)
    if parent_folder:
        if recursive:
            folders = [f for f in all_folders if f.startswith(parent_folder) and f != parent_folder]
        else:
            folders = [f for f in all_folders if f.startswith(parent_folder + "/") and f.count("/") == parent_folder.count("/") + 1]
    else:
        folders = all_folders if recursive else [f for f in all_folders if "/" not in f and f]
    if not parent_folder and not recursive:
        folders = [""] + folders
    info = []
    for folder in folders:
        stats = folder_stats(base, folder)
        info.append({"path": folder or "Inbox", "name": os.path.basename(folder) or "Inbox",
                     "is_special": folder in (".Trash", ".ToDoLater", ".Projects", ".Archive"),
                     "memory_counts": stats["memory_counts"], "total_memories": stats["total_memories"]})
    info.sort(key=lambda x: (0 if x["is_special"] else 1, x["name"]))
    return info


def bulk_tag_folder(base: str, folder_path: str, tags, statuses: Optional[List[str]] = None,
                    operation: str = "add") -> Tuple[int, List[Dict[str, Any]]]:
    """MemdirFolderManager.bulk_tag_folder (folders.py:483-587) on the tree at `base`: lists every requested directory, then
    edits each record's `Tags` pieces and rewrites the files whose multiset of pieces changes with the reference's re.sub calls."""
    folder_path = folder_path.replace("\\", "/").strip("/")
    if statuses is None:
        statuses = ["cur"]
    memories = []
    for status in statuses:
        if status not in STATUS_DIRS:
            raise ValueError(f"Invalid status: {status}. Must be one of {list(STATUS_DIRS)}")
        memories.extend(read_folder(base, folder_path, status, False))
    affected = []
    for memory in memories:
        file_path = os.path.join(base, folder_path, memory["status"], memory["filename"])
        if not os.path.exists(file_path):
            continue
        existing = [t.strip() for t in memory["headers"]["Tags"].split(",")] if "Tags" in memory["headers"] else []
        if operation == "add":
            updated = existing + [t for t in tags if t not in existing]
        elif operation == "remove":
            updated = [t for t in existing if t not in tags]
        elif operation == "replace":
            updated = tags
        else:
            continue
        if sorted(existing) == sorted(updated):
            continue
        new_tags = ", ".join(updated)
        with open(file_path, "r") as f:
            content = f.read()
        if "Tags:" in content:
            content = re.sub(r"Tags:.*$", f"Tags: {new_tags}", content, flags=re.MULTILINE)
        else:
            content = re.sub(r"^(.*?)(---)", f"\\1Tags: {new_tags}\n\\2", content, flags=re.DOTALL)
        with open(file_path, "w") as f:
            f.write(content)
        affected.append({"id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                         "old_tags": ", ".join(existing), "new_tags": new_tags})
    return len(affected), affected
