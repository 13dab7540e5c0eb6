"""The reference's MemoryArchiver (memdir_tools/archiver.py) on the packed corpus: its criteria predicate and the five
maintenance stages of `run_maintenance` (archiver.py:621-639).

`_memory_matches_criteria` is a per-record predicate over age, tags, header fields and flags; here a criteria dict becomes GPU
conditions (one query per criterion alternative, combined on the host: AND over the criteria keys, OR inside a tag list),
evaluated for every record in one pass.  Every stage selects its records with one scan program (one per 32 queries) over the
packed corpus and materialises only the selected records; the file actions (moves, flag renames, deletions and the `Status`
rewrite) stay host file I/O on those records, with the reference's statistics, in the reference's order.  A real run re-syncs
and scans again only where the reference would list a directory its own moves have changed since the last scan."""
from __future__ import annotations

import calendar
import os
import re
from datetime import datetime, timedelta
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

from .. import packer
from ..program import C_CONST, C_DATE_CMP, C_FLAGS, C_SLOT, CMP, Cond, ProgramBuilder, const
from ..regexc import Pattern
from . import utils as U


def _micros(dt: datetime) -> int:
    return calendar.timegm(dt.timetuple()) * 1000000 + dt.microsecond


def compile_criteria(criteria: Dict[str, Any], now: datetime) -> List[List[List[Cond]]]:
    """criteria -> [per key: [alternative: [conditions]]]; a record matches when every key has a matching alternative."""
    out: List[List[List[Cond]]] = []
    for key, pattern in criteria.items():
        if key in ("age", "min_age", "max_age"):
            if isinstance(pattern, bool) or not isinstance(pattern, int):
                raise NotImplementedError(f"criteria {key!r}: only integer day counts are supported on the GPU")
            # (now - date).days < p  <=>  date > now - p days;  .days > p  <=>  date <= now - (p + 1) days   (timedelta.days floors)
            days = pattern if key in ("age", "min_age") else pattern + 1
            try:
                edge = _micros(now - timedelta(days=days))
            except OverflowError:                              # the edge lies outside datetime's years 1..9999: every date is on one side
                out.append([[const((key == "max_age") == (days > 0))]])
                continue
            out.append([[Cond(C_DATE_CMP, op=CMP["<="] if key in ("age", "min_age") else CMP[">"], i64=edge)]])
        elif key in ("tag", "tags"):
            items = pattern if isinstance(pattern, list) else [pattern.lower()]
            alts = []
            for item in items:
                if not isinstance(item, str):
                    continue                                   # `item in memory_tags`: a non-str never equals a tag
                alts.append([Cond(C_SLOT, pattern=Pattern("has_tag", item), field="Tags", mode=1, empty_if_missing=True)])
            out.append(alts or [[const(False)]])
        else:
            # a header with exactly this key decides; only without one does `flags` mean the file-name flags (archiver.py:158-176)
            if isinstance(pattern, str):
                hdr = Cond(C_SLOT, pattern=Pattern("regex", pattern, re.IGNORECASE), field=key, mode=1, if_missing=2 if key == "flags" else 0)
                out.append([[hdr, Cond(C_FLAGS, pattern=Pattern("regex", pattern, re.IGNORECASE))] if key == "flags" else [hdr]])
            else:
                out.append([[const(False)]])                   # a header value (str) never equals a non-str, nor does the flags string
    return out


class MemoryArchiver:
    def __init__(self):
        self.archive_age = 90
        self.trash_age = 30
        self.archive_folder = ".Archive"
        self.trash_folder = ".Trash"
        self.archive_rules: List[Dict[str, Any]] = []
        self.cleanup_rules: List[Dict[str, Any]] = []
        self.retention_policies: Dict[str, Any] = {}
        self.tag_based_archiving: Dict[str, Any] = {}
        self.scan_passes = 0                             # scan programs run by this archiver (one per 32 queries)

    def set_archive_age(self, days: int) -> None:
        self.archive_age = days

    def set_trash_age(self, days: int) -> None:
        self.trash_age = days

    def add_archive_rule(self, folder: str, age_days: int, target_folder: Optional[str] = None) -> None:
        if target_folder is None:
            target_folder = self.archive_folder
        self.archive_rules.append({"folder": folder, "age_days": age_days, "target_folder": target_folder})

    def add_tag_based_archive_rule(self, tag: str, target_folder: str) -> None:
        self.tag_based_archiving[tag] = target_folder

    def set_retention_policy(self, folder: str, max_count: int, mode: str = "age") -> None:
        self.retention_policies[folder] = {"max_count": max_count, "mode": mode}

    def add_cleanup_rule(self, criteria: Dict[str, Any], action: str = "trash") -> None:
        self.cleanup_rules.append({"criteria": criteria, "action": action})

    # ---- selection: one program per 32 queries, hit lists in listing order
    def _scan(self, pm: "packer.PackedMemdir", queries: Sequence[Sequence[Cond]]) -> List[np.ndarray]:
        """Per query, the listing positions of its hits, ascending."""
        out: List[np.ndarray] = []
        for lo in range(0, len(queries), 32):
            pb = ProgramBuilder()
            for q in queries[lo:lo + 32]:
                pb.add_query(q)
            out.extend(pm.scan_hits(pb.build(), len(queries[lo:lo + 32])))
            self.scan_passes += 1
        return out

    @staticmethod
    def _listed(pm: "packer.PackedMemdir", hits: np.ndarray, folder: str, status: str, report: bool = True) -> np.ndarray:
        """The hits inside one directory, in its listing order (list_memories(folder, status) restricted to the hits).  `report`:
        print the directory's unreadable files, as each listing of the reference does."""
        if report:
            pm.report_skipped([folder], [status])
        r = pm.segments.get((folder, status))
        if r is None:
            if os.path.isdir(U.get_memory_path(folder, status)):
                raise NotImplementedError(f"folder {folder!r} is not spelled the way the tree walk lists it")
            return hits[:0]
        return hits[np.searchsorted(hits, r[0]):np.searchsorted(hits, r[1])]

    @staticmethod
    def _min_age(days: int, now: datetime) -> List[Cond]:
        """(now - date).days >= days, as archiver.py:236-238 and :408-410 test it."""
        return compile_criteria({"min_age": days}, now)[0][0]

    @staticmethod
    def _make_dirs(folder: str, made: set) -> None:
        """The cur / new / tmp directories of a target folder (archiver.py:199-201, :283-284), created once per stage."""
        if folder not in made:
            for status in U.STANDARD_FOLDERS:
                os.makedirs(os.path.join(U.MEMDIR_BASE, folder, status), exist_ok=True)
            made.add(folder)

    # ---- the maintenance stages (archiver.py:205-639)
    def archive_old_memories(self, dry_run: bool = False) -> Dict[str, Any]:
        """archiver.py:205-304.  Age rules archive `cur` of their folder to `.Archive/<year of the date>` (the rule's target_folder
        is not used) and append `S` to the flags; tag rules then move every `cur` record carrying the tag, in every folder the tree
        has after the age rules, to their target.  Directories are created even in a dry run.  One scan holds every rule; a real
        run scans again before it lists a directory its own moves changed (the reference lists after those moves)."""
        stats: Dict[str, Any] = {"archived": 0, "details": []}
        if not self.archive_rules:
            self.add_archive_rule("", self.archive_age, self.archive_folder)
        now = datetime.now()
        tags = list(self.tag_based_archiving.items())
        queries = [self._min_age(rule["age_days"], now) for rule in self.archive_rules]
        queries += [[Cond(C_SLOT, pattern=Pattern("has_tag", tag.lower()), field="Tags", mode=1, empty_if_missing=True)] for tag, _t in tags]
        made: set = set()
        touched: set = set()                            # folders changed by this run's moves since the last scan
        pm = packer.packed()
        with pm.lock:
            hits = self._scan(pm, queries)

            def fresh(folders):
                nonlocal pm, hits
                if touched & set(folders):
                    pm = packer.packed()                # re-sync: renames are carried over without reading the files
                    hits = self._scan(pm, queries)
                    touched.clear()

            for k, rule in enumerate(self.archive_rules):
                folder = rule["folder"]
                fresh([folder])
                for memory in pm.materialize(self._listed(pm, hits[k], folder, "cur"), False):
                    date = memory["metadata"]["date"]
                    target = os.path.join(self.archive_folder, str(date.year))
                    self._make_dirs(target, made)
                    if not dry_run:
                        U.move_memory(memory["filename"], folder, target, "cur", "cur")
                        if "S" not in memory["metadata"]["flags"]:
                            U.update_memory_flags(memory["filename"], target, "cur", "".join(memory["metadata"]["flags"]) + "S")
                        touched.update((folder, target))
                    stats["archived"] += 1
                    stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                             "age": (now - date).days,
                                             "action": f"Archived to {target}" if not dry_run else f"Would archive to {target}"})
            for t, (tag, target) in enumerate(tags):
                if touched:                             # get_memdir_folders() after the moves so far
                    fresh(touched)
                for folder in list(pm.folders):
                    fresh([folder])
                    for memory in pm.materialize(self._listed(pm, hits[len(self.archive_rules) + t], folder, "cur"), False):
                        self._make_dirs(target, made)
                        if not dry_run:
                            U.move_memory(memory["filename"], folder, target, "cur", "cur")
                            touched.update((folder, target))
                        stats["archived"] += 1
                        stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                                 "tag": tag,
                                                 "action": f"Archived to {target} based on tag" if not dry_run else f"Would archive to {target} based on tag"})
        return stats

    def empty_trash(self, age_days: Optional[int] = None, dry_run: bool = False) -> Dict[str, Any]:
        """archiver.py:383-431: every status directory of the trash folder itself (not its subfolders)."""
        if age_days is None:
            age_days = self.trash_age
        stats: Dict[str, Any] = {"deleted": 0, "details": []}
        now = datetime.now()
        pm = packer.packed()
        with pm.lock:
            hits = self._scan(pm, [self._min_age(age_days, now)])[0]
            for status in U.STANDARD_FOLDERS:
                for memory in pm.materialize(self._listed(pm, hits, self.trash_folder, status), False):
                    if not dry_run:
                        path = os.path.join(U.MEMDIR_BASE, self.trash_folder, status, memory["filename"])
                        if os.path.exists(path):
                            os.remove(path)
                    stats["deleted"] += 1
                    stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                             "age": (now - memory["metadata"]["date"]).days,
                                             "action": "Deleted from trash" if not dry_run else "Would delete from trash"})
        return stats

    # importance (archiver.py:465-485): Priority high / medium / low (exact key, lower-cased) = 3 / 2 / 1, +2 for F, +2 for P
    _PRIORITY = ("", "low", "medium", "high")

    @classmethod
    def _importance_queries(cls) -> List[Tuple[int, List[Cond]]]:
        """(score, conjunction) for every combination of priority class and F / P flags: 16 queries, 8 scores."""
        out = []
        for p, name in enumerate(cls._PRIORITY):
            prio = lambda v, neg: Cond(C_SLOT, pattern=Pattern("equals", v), negate=neg, field="Priority", mode=1, empty_if_missing=True)  # noqa: E731
            pc = [prio(name, False)] if p else [prio(v, True) for v in cls._PRIORITY[1:]]
            for f in (0, 1):
                for pp in (0, 1):
                    flags = [Cond(C_FLAGS, pattern=Pattern("exact_contains", "F"), negate=not f),
                             Cond(C_FLAGS, pattern=Pattern("exact_contains", "P"), negate=not pp)]
                    out.append((p + 2 * f + 2 * pp, pc + flags))
        return out

    def apply_retention_policies(self, dry_run: bool = False) -> Dict[str, Any]:
        """archiver.py:433-515: per policy (dict order), the first n - max_count records of `cur` after a stable sort go to
        `.Archive/<year>`.  Mode `age` sorts by timestamp, ascending: the listing is newest first and stable, so this is its runs
        of equal timestamps in reverse order, each run in its own order (a stable argsort of the listing's timestamps).  Mode
        `importance` concatenates the score buckets' hit lists, lowest score first; any other mode keeps the listing order."""
        stats: Dict[str, Any] = {"moved": 0, "details": []}
        policies = list(self.retention_policies.items())
        imp = self._importance_queries() if any(p["mode"] == "importance" for _f, p in policies) else []
        made: set = set()
        touched: set = set()
        pm = packer.packed()
        with pm.lock:
            hits = self._scan(pm, [q for _s, q in imp]) if imp else []
            for folder, policy in policies:
                max_count, mode = policy["max_count"], policy["mode"]
                if folder in touched:
                    pm = packer.packed()
                    hits = self._scan(pm, [q for _s, q in imp]) if imp else []
                    touched.clear()
                pm.report_skipped([folder], ["cur"])
                lo, hi = pm.segments.get((folder, "cur"), (0, 0))
                if (folder, "cur") not in pm.segments and os.path.isdir(U.get_memory_path(folder, "cur")):
                    raise NotImplementedError(f"folder {folder!r} is not spelled the way the tree walk lists it")
                n = hi - lo
                if n <= max_count:
                    continue
                if mode == "age":
                    order = lo + np.argsort(pm.arrays["ts"][lo:hi], kind="stable")
                elif mode == "importance":
                    seg = lambda h: h[np.searchsorted(h, lo):np.searchsorted(h, hi)]        # noqa: E731
                    order = np.concatenate([np.sort(np.concatenate([seg(h) for (s, _q), h in zip(imp, hits) if s == score]))
                                            for score in range(8)])
                else:
                    order = np.arange(lo, hi)
                for memory in pm.materialize(order[:n - max_count], False):
                    target = os.path.join(self.archive_folder, str(memory["metadata"]["date"].year))
                    self._make_dirs(target, made)
                    if not dry_run:
                        U.move_memory(memory["filename"], folder, target, "cur", "cur")
                        touched.update((folder, target))
                    stats["moved"] += 1
                    stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                             "folder": folder,
                                             "action": f"Moved to {target} (retention policy)" if not dry_run else f"Would move to {target} (retention policy)"})
        return stats

    # archiver.py:533-546
    _STATUS_RULES = ({"criteria": {"content": r"\[x\]|\bcompleted\b|\bfinished\b|\bdone\b"}, "new_status": "completed", "flags_add": "S"},
                     {"criteria": {"min_age": 60, "flags": r"^[^SR]*$"}, "new_status": "dormant", "flags_add": "S"})

    def update_memory_statuses(self, dry_run: bool = False) -> Dict[str, Any]:
        """archiver.py:517-619.  Rule r applies to a `cur` record that matches its criteria and whose `Status` header (exact key,
        "" when absent) is not the rule's status, and no earlier rule applied: the reference's `break` sits inside the status
        test, so a record that matches rule 1 but already has its status goes on to rule 2.  The `content` criterion is looked
        up among the headers, so it reads a header literally named `content`.  One query per rule, one scan."""
        stats: Dict[str, Any] = {"updated": 0, "details": []}
        now = datetime.now()
        queries = []
        for rule in self._STATUS_RULES:
            conds = [c for alts in compile_criteria(rule["criteria"], now) for c in alts[0]]        # one alternative per key
            conds.append(Cond(C_SLOT, pattern=Pattern("exact_equals", rule["new_status"]), negate=True, field="Status", mode=1, empty_if_missing=True))
            queries.append(conds)
        pm = packer.packed()
        with pm.lock:
            hits = self._scan(pm, queries)
            for folder in list(pm.folders):
                per_rule = [self._listed(pm, h, folder, "cur", report=k == 0) for k, h in enumerate(hits)]
                sel = np.union1d(per_rule[0], per_rule[1])
                first = np.isin(sel, per_rule[0])
                for memory, r1 in zip(pm.materialize(sel, False), first.tolist()):
                    rule = self._STATUS_RULES[0 if r1 else 1]
                    current_status, new_status = memory["headers"].get("Status", ""), rule["new_status"]
                    if not dry_run:
                        path = os.path.join(U.MEMDIR_BASE, folder, "cur", memory["filename"])
                        with open(path, "r") as f:
                            content = f.read()
                        if "Status: " in content:
                            content = re.sub(r"Status: .*$", f"Status: {new_status}", content, flags=re.MULTILINE)
                        else:
                            content = re.sub(r"^(.*?)---", f"\\1Status: {new_status}\n---", content, flags=re.DOTALL)
                        with open(path, "w") as f:
                            f.write(content)
                        new_flags = "".join(sorted(set("".join(memory["metadata"]["flags"]) + rule["flags_add"])))
                        U.update_memory_flags(memory["filename"], folder, "cur", new_flags)
                    stats["updated"] += 1
                    stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                             "folder": folder,
                                             "action": f"Updated status from '{current_status}' to '{new_status}'" if not dry_run
                                             else f"Would update status from '{current_status}' to '{new_status}'"})
        return stats

    def run_maintenance(self, dry_run: bool = False) -> Dict[str, Any]:
        """archiver.py:621-639.  Each stage syncs the packed corpus with the tree first, as each reference stage lists it again."""
        return {"archive": self.archive_old_memories(dry_run), "cleanup": self.cleanup_memories(dry_run),
                "trash": self.empty_trash(dry_run=dry_run), "retention": self.apply_retention_policies(dry_run),
                "status": self.update_memory_statuses(dry_run)}

    # ---- one GPU pass for any number of criteria dicts
    def match_criteria(self, criteria_list: Sequence[Dict[str, Any]], now: Optional[datetime] = None) -> np.ndarray:
        """bool[len(criteria_list), n]: which packed records match which criteria dict."""
        now = now or datetime.now()
        pm = packer.packed()
        with pm.lock:
            plans = [compile_criteria(c, now) for c in criteria_list]
            queries: List[List[Cond]] = []
            for plan in plans:
                for alts in plan:
                    queries.extend(alts)
            out = np.ones((len(plans), pm.n), dtype=bool)
            masks = np.zeros((0, pm.n), dtype=np.uint32)
            for lo in range(0, len(queries), 32):
                pb = ProgramBuilder()
                for q in queries[lo:lo + 32]:
                    pb.add_query(q)
                masks = np.vstack([masks, pm.scan_masks(pb.build())[None, :]])
                self.scan_passes += 1
            qi = 0
            for r, plan in enumerate(plans):
                for alts in plan:
                    hit = np.zeros(pm.n, dtype=bool)
                    for _ in alts:
                        hit |= (masks[qi // 32] >> np.uint32(qi % 32)) & np.uint32(1) != 0
                        qi += 1
                    out[r] &= hit
        return out

    def _memory_matches_criteria(self, memory: Dict[str, Any], criteria: Dict[str, Any]) -> bool:
        """Single-record form (host): the same rules as compile_criteria, evaluated directly."""
        for key, pattern in criteria.items():
            if key in ("age", "min_age", "max_age"):
                age = (datetime.now() - memory["metadata"]["date"]).days
                if (key != "max_age" and age < pattern) or (key == "max_age" and age > pattern):
                    return False
            elif key in ("tag", "tags"):
                tags = [t.strip() for t in memory["headers"].get("Tags", "").lower().split(",")]
                wanted = pattern if isinstance(pattern, list) else [pattern.lower()]
                if not any(w in tags for w in wanted):
                    return False
            elif key in memory["headers"] or key == "flags":
                value = memory["headers"][key] if key in memory["headers"] else "".join(memory["metadata"]["flags"])
                if not (re.search(pattern, value, re.IGNORECASE) if isinstance(pattern, str) else value == pattern):
                    return False
            else:
                return False
        return True

    def cleanup_memories(self, dry_run: bool = False) -> Dict[str, Any]:
        """archiver.py:306-381: every rule over every folder outside the trash, status cur only."""
        stats: Dict[str, Any] = {"trashed": 0, "deleted": 0, "details": []}
        if not self.cleanup_rules:
            self.add_cleanup_rule({"status": "completed|done"}, "trash")
            self.add_cleanup_rule({"status": "obsolete|deprecated"}, "trash")
        pm = packer.packed()
        matched = self.match_criteria([r["criteria"] for r in self.cleanup_rules])
        gone = np.zeros(pm.n, dtype=bool)               # acted upon by an earlier rule (real runs re-list after every rule)
        for rule, row in zip(self.cleanup_rules, matched):
            action = rule["action"]
            for folder in list(pm.folders):                   # get_memdir_folders(): the packed tree walk, in os.walk order
                if folder.startswith(self.trash_folder):
                    continue
                pm.report_skipped([folder], ["cur"])
                lo, hi = pm.segments.get((folder, "cur"), (0, 0))
                for i in (np.nonzero(row[lo:hi] & ~gone[lo:hi])[0] + lo).tolist():
                    memory = pm.materialize([i], True)[0]
                    if action == "trash":
                        if not dry_run:
                            U.move_memory(memory["filename"], folder, self.trash_folder, "cur", "cur")
                            gone[i] = True
                        stats["trashed"] += 1
                        stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                                 "action": "Moved to trash" if not dry_run else "Would move to trash"})
                    elif action == "delete":
                        if not dry_run:
                            path = os.path.join(U.MEMDIR_BASE, folder, "cur", memory["filename"])
                            if os.path.exists(path):
                                os.remove(path)
                            gone[i] = True
                        stats["deleted"] += 1
                        stats["details"].append({"memory_id": memory["metadata"]["unique_id"], "subject": memory["headers"].get("Subject", "No subject"),
                                                 "action": "Deleted permanently" if not dry_run else "Would delete permanently"})
        return stats
