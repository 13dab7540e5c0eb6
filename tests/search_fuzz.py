"""Seeded random queries for search_memories, FilterManager and MemoryArchiver.match_criteria, and the tree they run on.

build_fuzz_tree(base) writes the golden Memdir tree (tests/memdir_util.build_tree) plus EXTRA seeded records whose headers hold the
values where the query compiler has the most to get right: date headers of every kind dateutil produces (including one it
overflows on), `Timestamp` / `Hostname` / `Unique_ID` headers that shadow the file-name metadata, one key in several spellings,
a header over 64 KiB, Unicode whitespace around values, the characters whose case mapping is not one-to-one, and records
without a `---` separator.  Only `Due` holds values whose parse depends on today's date; every other date on the tree is
more than a year away from today, so that `now±N` operands cannot flip a verdict between two evaluations.

random_query / random_filter / random_criteria draw from typed pools and depend on the seed of `rng` alone.  oracle_search is
the reference's search_memories restated on the oracle: the oracle's per-record verdicts, then the reference's stable sort with
its "Unable to sort" fallback, then its pagination."""
from __future__ import annotations

import contextlib
import io
import os
import random
import re
from datetime import datetime, timedelta, timezone

from tests.memdir_util import build_tree, key_of
from tests.test_regexc_fuzz import rand_regex

SEED = 0x5EA2C4
N_EXTRA = 96
FOLDERS = ["", ".Fuzz", ".Fuzz/Deep", ".Projects/AI"]
STATUSES = ("cur", "new", "tmp")
DEEP = ".Fuzz/Deep"                     # its Due values are all strings dateutil rejects (no datetime-valued Due in this folder)
OVER = ".Fuzz/Over"                     # the two records whose Due / Created dateutil overflows on

# header values: dates dateutil parses (naive, date-only, aware), rejects, or overflows on; only Due gets today-dependent ones
DATE_VALUES = ["2031-03-04", "2019-07-08 12:30:00", "2031-01-01T10:00:00+02:00", "2018-12-31T23:59:59Z", "10 Jan 2031 08:00",
               "someday", "2024-02-30", "10000-01-01", "", "1/2/2019"]
TODAY_DEPENDENT = ["May 5", "10:30"]
DEEP_DUE = ["someday", "2024-02-30", "", "n/a"]
DATE_KEYS = {"Due": ["Due", "due", "DUE"], "Created": ["Created", "created"], "Modified": ["Modified", "MODIFIED"],
             "DeletedDate": ["DeletedDate", "deleteddate"]}
SUBJECTS = ["Quarterly review", "python tips", "İstanbul trip", "ΣΟΦΙΑ notes", "straße plan", "Kelvin scale", "react vs vue",
            "Meeting: budget", "ǅungla", "empty-ish", "docker, kubernetes", "σοφιας"]
TAGS = ["python", "ai", "learning", "trash", "İzmir", "straße", "Kelvin", "Σ", "books, reading", "x,y , z"]
STATUS_VALUES = ["active", "pending", "completed", "DONE", "in-progress", "Blocked", ""]
PRIORITY = ["high", "low", "HIGH", "medium"]
CATEGORY = ["İ", "ς", "Σσ", "ß", "SS", "K", "k", "plain"]
SHADOW = {"Hostname": ["shadowhost", "HOST-B", "fuzzhost"], "Unique_ID": ["fz000001", "SHADOW", "adv00001"],
          "Timestamp": ["12345", "1600000000", "abc", "99999999999999999999"]}
HOSTS = ["fuzzhost", "host-b", "h.c"]
FLAGS = ["", "S", "FS", "FRSP", "P", "R", "SF"]
WORDS = ["python", "react", "docker", "kubernetes", "review", "İ", "ß", "σοφια", "ΣΟΦΙΑ", "K", "budget", "[x]", "done",
         "café", "\U0001F409", "a.b", "tab\there", "line\nbreak", "999", "2031-03-04"]
SPACES = [" ", " ", "　", "\t", " "]


def _extra_records(seed=SEED):
    """(folder, status, filename, text) of the extra records; deterministic in `seed`."""
    rng = random.Random(seed)
    stamps = rng.sample(range(1_500_000_000, 1_720_000_000), N_EXTRA)
    out = []
    for i, ts in enumerate(stamps):
        folder = DEEP if i < 8 else OVER if i in (8, 9) else FOLDERS[i % len(FOLDERS)]
        status = STATUSES[(i // len(FOLDERS)) % 3]
        name = f"{ts}.fz{i:06x}.{rng.choice(HOSTS)}:2,{rng.choice(FLAGS)}"
        lines = []

        def put(key, value):
            if rng.random() < 0.2:
                value = rng.choice(SPACES) + value + rng.choice(SPACES)
            lines.append(f"{key}: {value}")
        if rng.random() < 0.9:
            put("Subject", rng.choice(SUBJECTS))
        if rng.random() < 0.6:
            put(rng.choice(["Tags", "Tags", "tags"]), ",".join(rng.sample(TAGS, rng.randint(1, 3))))
        if rng.random() < 0.4:
            put(rng.choice(["Priority", "priority", "PRIORITY"]), rng.choice(PRIORITY))
        if rng.random() < 0.4:
            put("Status", rng.choice(STATUS_VALUES))
        if rng.random() < 0.3:
            put("Category", rng.choice(CATEGORY))
        for canon, spellings in DATE_KEYS.items():
            if folder == DEEP:
                if canon == "Due":
                    put(rng.choice(spellings), rng.choice(DEEP_DUE))
                continue
            if rng.random() < 0.45:
                pool = DATE_VALUES + (TODAY_DEPENDENT if canon == "Due" else [])
                put(rng.choice(spellings), rng.choice(pool))
        for key, pool in SHADOW.items():
            if rng.random() < 0.12:
                put(key, rng.choice(pool))
        if i in (8, 9):                                                          # one Due and one Created dateutil overflows on
            lines.append(f"{'Due' if i == 8 else 'Created'}: 99999999999999999999")
        if i == 5:
            put("Notes", "long " * 14000 + "needle-at-the-end")                  # > 64 KiB header
        if i == 7:
            lines += ["Tags: first", "tags: second", "TAGS: third", "Tags: last"]   # one key, several spellings and repeats
        body = " ".join(rng.choice(WORDS) for _ in range(rng.randint(0, 12)))
        rng.shuffle(lines)
        if rng.random() < 0.08:
            text = body + ("\nSubject: not a header" if rng.random() < 0.5 else "")    # no separator: everything is content
        else:
            text = "\n".join(lines) + "\n---\n" + body
        out.append((folder, status, name, text))
    return out


def build_fuzz_tree(base):
    """The golden tree plus the extra records; returns the vocabulary the generators draw operands from."""
    build_tree(base)
    for folder, status, name, text in _extra_records():
        d = os.path.join(base, folder, status)
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, name), "w", encoding="utf-8") as f:
            f.write(text)
    for folder in FOLDERS + [OVER]:
        for status in STATUSES:
            os.makedirs(os.path.join(base, folder, status), exist_ok=True)
    return tree_vocab()


def tree_vocab(seed=SEED):
    """Substrings and tokens of the extra records' values (the golden part is covered by the fixed pools)."""
    toks = set()
    for i, (_f, _s, name, text) in enumerate(_extra_records(seed)):
        if i % 8 == 0:
            toks.add(name.split(".")[1])
        for line in text.split("\n"):
            for piece in re.split(r"[\s:,]+", line):
                if 0 < len(piece) <= 40:
                    toks.add(piece)
    toks.update(SUBJECTS + TAGS + STATUS_VALUES + PRIORITY + CATEGORY + WORDS + ["Fuzz", ".Projects", "AI", "Deep", "cur", "new"])
    return {"tokens": sorted(toks), "folders": sorted(set(FOLDERS + [OVER, ".Projects/Python", ".ToDoLater/Learning", ".Trash", ".Nope"]))}


# ----------------------------------------------------------------------------- queries
SEARCH_FIELDS = (["content"] * 4 + ["flags", "date", "id", "filename", "folder", "status", "maildir_status", "Status", "state", "status_value",
                 "STATE", "Due", "due", "DUE", "Created", "created", "Modified", "MODIFIED", "DeletedDate", "deleteddate", "Date",
                 "timestamp", "Timestamp", "unique_id", "Unique_ID", "hostname", "HOSTNAME", "Subject", "subject", "Tags", "tags",
                 "Priority", "Category", "Notes", "No-Such-Header"] + ["Subject", "Tags", "Due", "Created", "timestamp"])
DATE_HEADERS = ("due", "created", "modified", "deleteddate")
OPS = ["contains", "matches", "startswith", "endswith", "has_tag", "=", "!=", ">", "<", ">=", "<=", "has_flag", "~~"]
SORT_FIELDS = ["Subject", "date", "Due", "Created", "timestamp", "Priority", "content", "folder", "flags", "No-Such-Header", "Status"]
INT_EDGES = [0, 1, -1, 12345, 1600000000, 1650000000, 1700000512, (1 << 63) - 1, -(1 << 63), 1 << 63, -(1 << 63) - 1, 1 << 70, 10 ** 20]
FLOATS = [float("nan"), float("inf"), float("-inf"), 1.5, -2.25, 1600000000.0, 1700000000.5, 0.0]
DATETIMES = [datetime(2019, 1, 1), datetime(2031, 6, 1, 12, 0), datetime(2023, 11, 14, 22, 13, 20),
             datetime(2031, 1, 1, 8, 0, tzinfo=timezone.utc), datetime(2019, 7, 8, 12, 30, tzinfo=timezone(timedelta(hours=2)))]
DATE_STRINGS = ["2023-11-14", "2023-11-14 22:14:00", "2031-01-01T08:00:00+00:00", "2019-07-08 12:30:00", "Jan 10 2031",
                "99999999999999999999", "10000-01-01", "2024-02-30", "not a date"]
NOW_STRINGS = ["now", "now-3d", "now+2w", "now-1y", "now-5m"]


def _case_flip(rng, s):
    return "".join(c.upper() if rng.random() < 0.5 else c.lower() for c in s) if rng.random() < 0.3 else s


def _operand(rng, vocab):
    r = rng.random()
    if r < 0.50:
        tok = rng.choice(vocab["tokens"])
        if len(tok) > 3 and rng.random() < 0.4:
            a = rng.randrange(len(tok) - 2)
            tok = tok[a:a + rng.randint(1, len(tok) - a)]
        return _case_flip(rng, tok)
    if r < 0.60:
        return rand_regex(rng) if rng.random() < 0.85 else rng.choice(["(unclosed", "[z-a]", "*x", "a{2,1}"])
    if r < 0.64:
        return ""
    if r < 0.70:
        return rng.choice(INT_EDGES)
    if r < 0.75:
        return rng.choice(FLOATS)
    if r < 0.77:
        return rng.choice([True, False])
    if r < 0.83:
        return rng.choice(DATETIMES)
    if r < 0.94:
        return rng.choice(DATE_STRINGS)
    return rng.choice(NOW_STRINGS)


def random_query(rng, vocab):
    """(conditions, include_content, folders, statuses, sort, reverse, limit, offset); conditions are (field, op, value)."""
    conds = []
    for _ in range(rng.choice([1, 1, 1, 2, 2, 3, 4])):
        field, op = rng.choice(SEARCH_FIELDS), rng.choice(OPS + ["contains", "contains", "matches", "!=", "<", ">="])
        if field.lower() in DATE_HEADERS and sum(f.lower() in DATE_HEADERS for f, _o, _v in conds) >= 2:
            field = "Subject"               # the scan holds MAX_AUX = 4 host-judged columns, two per date-header condition
        if op == "~~" and rng.random() < 0.7:
            op = rng.choice(OPS[:-1])
        v = _operand(rng, vocab)
        if field.lower() == "timestamp" and rng.random() < 0.5:
            v = rng.choice(INT_EDGES + FLOATS)
        elif field.lower() in ("filename", "id", "unique_id", "hostname") and rng.random() < 0.5:
            v = _case_flip(rng, rng.choice(["fz00", "fz000", "host-b", "h.c", "fuzzhost", ":2,FS", ":2,", "adv000", "17", "15", ".host"]))
        elif field.lower() in ("folder", "status", "maildir_status") and rng.random() < 0.5:
            v = _case_flip(rng, rng.choice(vocab["folders"] + list(STATUSES))[rng.randint(0, 3):])
        conds.append((field, op, v))
    if rng.random() < 0.125:                                    # a keyword pair: Subject and content on the same operand
        v = _case_flip(rng, rng.choice(vocab["tokens"])) if rng.random() < 0.8 else _operand(rng, vocab)
        at = rng.randint(0, len(conds))
        conds[at:at] = [("Subject", "contains", v)]
        conds.insert(rng.randint(0, len(conds)), ("content", "contains", v))
    include_content = rng.random() < 0.6
    folders = None if rng.random() < 0.6 else rng.sample(vocab["folders"], rng.randint(1, 3))
    statuses = None if rng.random() < 0.7 else rng.sample(list(STATUSES), rng.randint(1, 3))
    sort = rng.choice(SORT_FIELDS) if rng.random() < 0.25 else None
    reverse = rng.random() < 0.5
    limit = rng.choice([None, None, 0, 1, 3, 10])
    offset = rng.choice([0, 0, 0, 1, 2, 5])
    return conds, include_content, folders, statuses, sort, reverse, limit, offset


def depends_on_today(q):
    """Does the query's outcome depend on the date it runs (a `now` operand, a Due value whose parse takes today's date)?"""
    conds, _ic, _fo, _st, sort, *_ = q
    return (any(isinstance(v, str) and v.startswith("now") or str(f).lower() == "due" for f, _op, v in conds)
            or (sort or "").lower() == "due")


FILTER_FIELDS = ["content", "flags", "unique_id", "hostname", "timestamp", "date", "Subject", "Tags", "tags", "Priority", "Status",
                 "Due", "Category", "Timestamp", "Hostname", "No-Such-Header"]


def _valid_regex(rng, vocab):
    while True:
        p = rand_regex(rng) if rng.random() < 0.5 else re.escape(_case_flip(rng, rng.choice(vocab["tokens"])))
        try:
            re.compile(p, re.IGNORECASE)
            return p
        except re.error:
            continue


def random_filter(rng, vocab):
    """MemoryFilter conditions [(field, pattern, negate)] (1 to 3; valid patterns)."""
    return [(rng.choice(FILTER_FIELDS), _valid_regex(rng, vocab), rng.random() < 0.3) for _ in range(rng.randint(1, 3))]


CRITERIA_KEYS = ["age", "min_age", "max_age", "tag", "tags", "Subject", "Priority", "Status", "Tags", "Due", "flags", "Category", "No-Such-Header"]


def random_criteria(rng, vocab):
    """A criteria dict for MemoryArchiver.match_criteria (1 to 3 keys)."""
    out = {}
    for key in rng.sample(CRITERIA_KEYS, rng.randint(1, 3)):
        if key in ("age", "min_age", "max_age"):
            out[key] = rng.choice([0, 1, -5, 30, 365, 1000, 3000, 10 ** 6, 10 ** 10])
        elif key in ("tag", "tags"):
            pick = lambda: _case_flip(rng, rng.choice(TAGS + vocab["tokens"][:50]))      # noqa: E731
            out[key] = [pick() for _ in range(rng.randint(0, 3))] + ([7] if rng.random() < 0.1 else []) if rng.random() < 0.5 else pick()
        else:
            out[key] = _valid_regex(rng, vocab) if rng.random() < 0.9 else rng.choice([1, None, True])
    return out


# ----------------------------------------------------------------------------- the reference's search_memories on the oracle
@contextlib.contextmanager
def sorted_fs():
    """os.walk / os.listdir in sorted order: the listing order then does not depend on the file system (for the goldens)."""
    walk, listdir = os.walk, os.listdir

    def sorted_walk(top, *a, **k):
        for root, dirs, files in walk(top, *a, **k):
            dirs.sort()
            yield root, dirs, sorted(files)
    os.walk, os.listdir = sorted_walk, lambda p=".": sorted(listdir(p))
    try:
        yield
    finally:
        os.walk, os.listdir = walk, listdir


def sort_and_page(results, sort, reverse, limit, offset, lookup):
    """search.py:369-388: stable sort by the field (None -> ""), newest first when that raises; then the page."""
    printed = ""
    if sort:
        try:
            results.sort(key=lambda x: lookup(x, sort) or "", reverse=reverse)
        except Exception as e:
            printed = f"Warning: Unable to sort results: {e}\n"
            results.sort(key=lambda x: x["metadata"]["timestamp"], reverse=True)
    if offset or limit:
        results = results[offset:None if limit is None else offset + limit]
    return results, printed


def outcome(run):
    """{"keys", "unable_to_sort"} of a search, or {"raises": [type, message]}; `run` returns (results, printed)."""
    try:
        res, printed = run()
    except Exception as e:
        return {"raises": [type(e).__name__, str(e)]}
    return {"keys": [key_of(m) for m in res], "unable_to_sort": "Unable to sort" in printed}


def oracle_search(base, q, listing_cache=None):
    from oracle import memdir_oracle as mo
    conds, include_content, folders, statuses, sort, reverse, limit, offset = q
    ck = (tuple(folders) if folders is not None else None, tuple(statuses) if statuses is not None else None, include_content)
    if listing_cache is None or ck not in listing_cache:
        with contextlib.redirect_stdout(io.StringIO()):
            mems = mo.listing(base, folders, statuses, include_content)
        if listing_cache is not None:
            listing_cache[ck] = mems
    else:
        mems = listing_cache[ck]

    def run():
        hits = [mems[i] for i in mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in conds])]
        return sort_and_page(hits, sort, reverse, limit, offset, mo.lookup)
    return outcome(run)


def product_search(q):
    from fei_b200.memdir_tools.search import SearchQuery, search_memories
    conds, include_content, folders, statuses, sort, reverse, limit, offset = q
    sq = SearchQuery()
    for f, op, v in conds:
        sq.add_condition(f, op, v)
    sq.with_content(include_content)
    if sort:
        sq.set_sort(sort, reverse)
    sq.set_pagination(limit, offset)

    def run():
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            res = search_memories(sq, folders, statuses)
        return res, buf.getvalue()
    return outcome(run)
