"""The seeded Memdir tree of the maintenance goldens (tests/golden/make_golden_maintenance.py, maintenance_golden.json), the
archiver settings and cases the goldens run, a frozen `datetime.now()` and a digest of a tree (files with their bytes, directories).

The timestamps spread over about three years before NOW, so the age thresholds and the `.Archive/<year>` folders split the
records.  The tree also holds `.Trash` items (and a `.Trash` subfolder the trash stage must leave alone), records that share a
timestamp, a header named `flags`, one named `content`, repeated `Priority` keys, records that are already `dormant` or
`completed`, `Status: ` inside a body and a record without a `---` separator.  Records that share a timestamp sit only where
no retention cut can fall between them, and every tag rule moves to a folder that does not exist before the rule runs, so no
record moved by a tag rule is listed again by it: the goldens do not depend on the order a file system lists a directory in
(a target the rule's folder walk holds is listed again or not depending on where the walk meets it)."""
import calendar
import hashlib
import os
import random
from datetime import datetime, timedelta

SEED = 20261017
NOW = datetime(2026, 6, 15, 12, 0, 0)
NOW_TS = calendar.timegm(NOW.timetuple())                  # the trees are read with TZ=UTC
SPAN_DAYS = 3 * 365

# folder -> (cur, new) record counts, and whether records of one directory may share a timestamp
LAYOUT = {
    "": (36, 4, False), ".Projects": (24, 3, False), ".Projects/Alpha": (14, 2, True), ".ToDoLater": (10, 2, False),
    ".Trash": (9, 3, True), ".Trash/Old": (4, 0, True), ".Archive": (3, 0, True), ".Archive/2024": (5, 0, True),
}
EMPTY_FOLDERS = [".Empty"]

_TAGS = [None, "python", "Python, work", "misc", "work,urgent", "", "PYTHON ,ai", "notes", "ai"]
_PRIORITY = [None, None, "high", "Medium", "LOW", "urgent", ["low", "high"], ["HIGH", "none"]]
_STATUS = [None, "active", "active", "completed", "dormant", "Completed", "done"]
_FLAGS = ["", "", "S", "F", "P", "FP", "R", "SF", "PS", "RF", "PF"]
_WORDS = ["alpha", "deploy", "done", "notes", "meeting", "completed", "finished", "review", "budget", "[x] item", "draft"]


def frozen_datetime(base=datetime):
    """A datetime subclass whose now() is NOW (assign it to the archiver module's `datetime`)."""
    class Frozen(base):
        @classmethod
        def now(cls, tz=None):
            return cls(NOW.year, NOW.month, NOW.day, NOW.hour, NOW.minute, NOW.second)
    return Frozen


def _record(rng, i, ts, folder):
    uid = f"{rng.getrandbits(32):08x}"
    flags = rng.choice(_FLAGS)
    name = f"{ts}.{uid}.host{i % 3}:2,{flags}"
    lines = [f"Subject: Memory {i} in {folder or 'Inbox'}", f"Date: {(datetime(1970, 1, 1) + timedelta(seconds=ts)).isoformat()}"]
    tags = rng.choice(_TAGS)
    if tags is not None:
        lines.append(f"Tags: {tags}")
    prio = rng.choice(_PRIORITY)
    for p in ([] if prio is None else prio if isinstance(prio, list) else [prio]):
        lines.append(f"Priority: {p}")
    status = rng.choice(_STATUS)
    if status is not None:
        lines.append(f"Status: {status}")
    r = rng.random()
    if r < 0.08:
        lines.append(f"flags: {rng.choice(['S', 'FP', 'x'])}")
    elif r < 0.2:
        lines.append(f"content: {rng.choice(['done', '[x] task', 'nothing here', 'Finished it'])}")
    body = " ".join(rng.choice(_WORDS) for _ in range(rng.randint(3, 12)))
    if rng.random() < 0.1:
        body += "\nStatus: noted in the body"
    if i % 53 == 7:
        return name, body + "\n"                             # no `---`: no headers at all
    return name, "\n".join(lines) + "\n---\n" + body + "\n"


def build_tree(base: str) -> None:
    rng = random.Random(SEED)
    i = 0
    used = set()
    for folder, (n_cur, n_new, ties) in LAYOUT.items():
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(base, folder, st), exist_ok=True)
        for st, n in (("cur", n_cur), ("new", n_new)):
            prev = None
            for _ in range(n):
                if ties and prev is not None and rng.random() < 0.3:
                    ts = prev
                else:
                    while True:
                        ts = NOW_TS - rng.randint(0, SPAN_DAYS * 86400)
                        if ts not in used:
                            break
                used.add(ts)
                prev = ts
                name, text = _record(rng, i, ts, folder)
                i += 1
                with open(os.path.join(base, folder, st, name), "w") as f:
                    f.write(text)
    for folder in EMPTY_FOLDERS:
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(base, folder, st), exist_ok=True)


def _walk(base: str):
    """Every directory, and every file of a cur / new / tmp directory as (folder, status, file name, path)."""
    dirs, files = [], []
    for root, _dnames, fnames in os.walk(base):
        rel = os.path.relpath(root, base)
        if rel != ".":
            dirs.append(rel)
        if os.path.basename(root) in ("cur", "new", "tmp"):
            files += [(os.path.dirname(rel), os.path.basename(root), name, os.path.join(root, name)) for name in fnames]
    return dirs, files


def records(base: str):
    """unique_id -> (folder, status, timestamp) of every record in the tree."""
    return {name.split(".")[1]: (folder, status, int(name.split(".")[0])) for folder, status, name, _p in _walk(base)[1]}


def tree_digest(base: str) -> str:
    """sha256 over every directory and every file (folder, status, name, sha256 of its bytes), sorted: what a stage created,
    moved, renamed, deleted or rewrote."""
    dirs, files = _walk(base)
    rows = []
    for folder, status, name, path in files:
        with open(path, "rb") as f:
            rows.append([folder, status, name, hashlib.sha256(f.read()).hexdigest()])
    return hashlib.sha256(repr((sorted(dirs), sorted(rows))).encode()).hexdigest()


def configure(arch, config: str) -> None:
    """The archiver settings of one golden configuration (the reference's MemoryArchiver or this project's)."""
    if config == "default":
        return
    assert config == "configured"
    arch.set_archive_age(700)
    arch.add_archive_rule(".Projects", 400, ".Elsewhere")          # target_folder is not used: .Archive/<year>
    arch.add_archive_rule(".Projects", 200)                         # the same folder again: sees what the first rule left
    arch.add_archive_rule("", arch.archive_age)
    arch.add_tag_based_archive_rule("Python", ".Archive/Tagged")
    arch.add_tag_based_archive_rule("work", ".Archive/Work")         # a target of its own: see below
    arch.set_trash_age(120)
    arch.set_retention_policy("", 12, "age")
    arch.set_retention_policy(".Projects", 6, "importance")
    arch.set_retention_policy(".ToDoLater", 4, "newest")
    arch.set_retention_policy(".Nowhere", 1, "age")
    arch.add_cleanup_rule({"tags": ["misc", "ai"]}, "trash")
    arch.add_cleanup_rule({"Priority": "urgent"}, "delete")


STAGES = ("archive_old_memories", "cleanup_memories", "empty_trash", "apply_retention_policies", "update_memory_statuses")
# (config, stage, dry_run): every stage dry, run_maintenance for real (its stages each see what the one before left), and a real
# retention run on the fresh tree (run_maintenance's own retention finds the folders under their limits)
CASES = [(c, s, True) for c in ("default", "configured") for s in STAGES] + [
    ("default", "run_maintenance", False), ("configured", "run_maintenance", False), ("configured", "apply_retention_policies", False)]
METHODS = ("set_archive_age", "set_trash_age", "add_archive_rule", "add_tag_based_archive_rule", "set_retention_policy",
           "archive_old_memories", "empty_trash", "apply_retention_policies", "update_memory_statuses", "run_maintenance")


def run_stage(arch, stage: str, dry_run: bool):
    return arch.empty_trash(dry_run=dry_run) if stage == "empty_trash" else getattr(arch, stage)(dry_run)
