"""Seeded random queries (tests/search_fuzz.py) through search_memories, FilterManager.process_memories and
MemoryArchiver.match_criteria on the GPU, against the oracle on the same tree: the query compiler (search.compile_conditions,
filter._compile_filter_conditions, archiver.compile_criteria) and the program it builds, end to end.

A search must give the oracle's result keys in the oracle's order (on this machine's listing), the same "Unable to sort"
warning, or the same exception type and message; a failure prints the query tuple, ready to paste into REGRESSIONS."""
import contextlib
import io
import random

import numpy as np
import pytest

from oracle import memdir_oracle as mo
from tests import search_fuzz as F
from tests.maintenance_tree import NOW
from tests.memdir_util import key_of

pytestmark = pytest.mark.gpu

N_SEARCH, N_FILTER_RUNS, N_CRITERIA = 1500, 40, 120
BIG = "99999999999999999999"           # dateutil.parser.parse: OverflowError: Python int too large to convert to C long

# (name, query tuple as random_query returns it); run before the random stream
REGRESSIONS = [
    ("date_operand_dateutil_overflows", ([("date", ">", BIG)], False, None, None, None, False, None, 0)),
    ("date_operand_overflow_int", ([("Date", "<=", 10 ** 20)], False, None, None, None, False, None, 0)),
    ("date_operand_overflow_not_reached", ([("Subject", "=", "no such subject"), ("date", ">", BIG)], False, None, None, None, False, None, 0)),
    ("due_value_overflows_any_operator", ([("Due", "contains", "x")], False, None, None, None, False, None, 0)),
    ("created_value_overflows_for_has_tag", ([("created", "has_tag", "2031")], False, [F.OVER, ""], None, None, False, None, 0)),
    ("due_value_overflow_not_reached", ([("Due", "contains", "some")], False, [F.DEEP], None, None, False, None, 0)),
    ("due_operand_overflows_only_string_dues_reached", ([("Due", ">", BIG)], False, [F.DEEP], None, None, False, None, 0)),
    ("due_operand_overflows_after_a_rejecting_condition", ([("Subject", "=", "no such subject"), ("Due", ">", BIG)], False, None, None, None, False, None, 0)),
    ("due_operand_overflows", ([("Due", ">", BIG)], False, None, None, None, False, None, 0)),
    ("modified_operand_overflows_on_datetimes", ([("Modified", "<", BIG)], False, ["", ".Fuzz"], None, None, False, None, 0)),
    ("string_dues_raise_typeerror_others_do_not", ([("Due", ">", 5)], False, [F.DEEP, ".Fuzz"], None, None, False, None, 0)),
    ("timestamp_header_or_metadata_first", ([("timestamp", ">", "now")], False, None, None, None, False, None, 0)),
    ("timestamp_str_cmp_header_records_only", ([("Timestamp", ">", "abc")], False, None, None, None, False, None, 0)),
    ("sort_by_overflowing_due", ([("Subject", "contains", "")], False, [F.OVER, ".Fuzz"], None, "Due", False, 5, 1)),
]


@pytest.fixture(scope="module")
def fuzz(gpu, tmp_path_factory):
    from fei_b200 import packer
    from fei_b200.memdir_tools import utils as U
    base = str(tmp_path_factory.mktemp("search_fuzz_gpu") / "Memdir")
    vocab = F.build_fuzz_tree(base)
    old = U.MEMDIR_BASE
    U.set_memdir_base(base)
    yield {"base": base, "vocab": vocab, "cache": {}, "queries": [], "filters": []}
    U.set_memdir_base(old)
    packer.drop(base)


def _check(fuzz, q, where):
    want = F.oracle_search(fuzz["base"], q, fuzz["cache"])
    got = F.product_search(q)
    fuzz["queries"].append((q, got))
    return None if got == want else f"{where}: query={q!r}\n  product={got}\n  oracle={want}"


def test_regression_cases(fuzz):
    bad = [m for name, q in REGRESSIONS for m in [_check(fuzz, q, name)] if m]
    assert not bad, "\n".join(bad)
    for name in ("date_operand_dateutil_overflows", "due_value_overflows_any_operator", "due_operand_overflows"):
        q = dict(REGRESSIONS)[name]
        assert F.product_search(q)["raises"][0] == "OverflowError", name
    assert F.product_search(dict(REGRESSIONS)["due_operand_overflows_only_string_dues_reached"]).get("keys")


def test_parsed_dates_cache_holds_the_overflow(fuzz):
    """The per-value parse cache keeps the overflow, and a query after it still raises it afresh."""
    from fei_b200 import packer
    q = dict(REGRESSIONS)["due_value_overflows_any_operator"]
    first = F.product_search(q)
    assert isinstance(packer.packed().parsed_dates[BIG][0], OverflowError)
    assert F.product_search(q) == first == F.oracle_search(fuzz["base"], q, fuzz["cache"])


def test_random_search(fuzz):
    rng = random.Random(0x5EA4C8)
    bad = []
    for k in range(N_SEARCH):
        q = F.random_query(rng, fuzz["vocab"])
        m = _check(fuzz, q, f"query {k}")
        if m:
            print(m, flush=True)
            bad.append(m)
    assert not bad, f"{len(bad)} of {N_SEARCH} queries differ\n" + "\n".join(bad[:12])


def test_random_filters(fuzz):
    from fei_b200.memdir_tools import filter as Fl
    rng = random.Random(0xF117)
    base, bad = fuzz["base"], []
    for k in range(N_FILTER_RUNS):
        filters = []
        for j in range(rng.randint(1, 3)):
            acts = rng.sample(["move", "flag", "copy"], rng.randint(0, 2))
            filters.append({"name": f"f{j}", "conditions": [{"field": f, "pattern": p, "negate": n} for f, p, n in F.random_filter(rng, fuzz["vocab"])],
                            "actions": [{"type": a} for a in acts]})
        folders = None if rng.random() < 0.6 else rng.sample(fuzz["vocab"]["folders"], rng.randint(1, 3))
        statuses = rng.choice([None, ["new"], ["cur"], ["cur", "new", "tmp"], ["tmp", "cur"]])
        fuzz["filters"] += [flt["conditions"] for flt in filters]
        mgr = Fl.FilterManager()
        for flt in filters:
            f = Fl.MemoryFilter(flt["name"])
            for c in flt["conditions"]:
                f.add_condition(c["field"], c["pattern"], c["negate"])
            for a in flt["actions"]:
                f.add_action(a["type"])
            mgr.add_filter(f)
        with contextlib.redirect_stdout(io.StringIO()):
            got = mgr.process_memories(folders=folders, statuses=statuses, dry_run=True)
            mems = mo.listing(base, folders, statuses or ["new"], True)
        want = mo.run_filters(mems, filters)
        counts = lambda s: {k: v for k, v in s.items() if k != "details"}          # noqa: E731
        by_id = lambda s: {d["memory_id"]: d for d in s["details"]}                # noqa: E731
        if counts(got) != counts(want) or by_id(got) != by_id(want) or len(got["details"]) != len(want["details"]):
            bad.append(f"run {k}: filters={filters!r} folders={folders!r} statuses={statuses!r}\n  product={counts(got)}\n  oracle={counts(want)}")
    assert not bad, "\n".join(bad[:10])


def test_random_criteria(fuzz):
    from fei_b200 import packer
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    rng = random.Random(0xC417)
    crits = [F.random_criteria(rng, fuzz["vocab"]) for _ in range(N_CRITERIA)]
    with contextlib.redirect_stdout(io.StringIO()):
        rows = MemoryArchiver().match_criteria(crits, now=NOW)
        pm = packer.packed()
        mems = mo.listing(fuzz["base"], None, None, True)
    idx = np.concatenate([np.arange(a, b) for a, b in pm.ranges(None, None)])
    assert idx.size == len(mems)
    bad, hit_some = [], 0
    for c, row in zip(crits, rows):
        got = [key_of(mems[k]) for k in np.nonzero(row[idx])[0].tolist()]
        want = [key_of(m) for m in mems if mo.matches_criteria(m, c, now=NOW)]
        hit_some += 0 < len(want) < len(mems)
        if got != want:
            bad.append(f"criteria={c!r}\n  product={len(got)} records\n  oracle={len(want)} records")
    assert not bad, "\n".join(bad[:10])
    assert hit_some >= N_CRITERIA // 40


def test_random_queries_reach_every_path(fuzz):
    """Every Cond kind, every C_NAME field, C_SLOT modes 0 and 1 with each if_missing and the host-judged aux columns decided
    some record each way in at least one compiled query (search queries and filters); a raising condition was reached in one
    search and left unreached in another."""
    from fei_b200 import packer
    from fei_b200.memdir_tools import filter as Fl, search as S
    from fei_b200.program import C_CONST, C_NAME, C_RECBITS, C_SLOT
    assert len(fuzz["queries"]) >= N_SEARCH and fuzz["filters"], "runs after test_random_search and test_random_filters"
    pm = packer.packed()
    need = {("kind", k) for k in range(10)} | {("name", w) for w in range(5)} | {("slot", m, i) for m in (0, 1) for i in (0, 1, 2)}
    need |= {("recbits",), ("raises", "reached"), ("raises", "unreached")}
    seen = set()

    def visit(items, ranges, total):
        for j, c in enumerate(items):
            if isinstance(c, S._Raises):
                c = c.presence
                if c is None:
                    continue
            group = [c]
            if c.kind == C_SLOT and c.if_missing == 2:             # the next condition is its fallback: scan the pair
                if j + 1 >= len(items) or not isinstance(items[j + 1], type(c)):
                    continue
                group.append(items[j + 1])
            tags = [("kind", c.kind)] + ([("name", c.which)] if c.kind == C_NAME else []) + \
                ([("slot", c.mode, c.if_missing)] if c.kind == C_SLOT else []) + ([("recbits",)] if c.kind == C_RECBITS else [])
            if c.kind == C_CONST:
                seen.add(("const", c.value))
                continue
            if all(t in seen for t in tags):
                continue
            n = len(S._scan_ranges(pm, group, ranges))
            if 0 < n < total:
                seen.update(tags)

    with contextlib.redirect_stdout(io.StringIO()), pm.lock:
        for q, got in fuzz["queries"]:
            conds, include_content, folders, statuses = q[:4]
            ranges = pm.ranges(folders, statuses)
            pm.begin_query()
            try:
                compiled = S.compile_conditions([{"field": f, "operator": op, "value": v} for f, op, v in conds], include_content, pm)
            except Exception:
                continue
            if any(isinstance(c, S._Raises) for c in compiled):
                seen.add(("raises", "reached" if "raises" in got else "unreached"))
            visit(compiled, ranges, sum(b - a for a, b in ranges))
        ranges = pm.ranges(None, None)
        for conds in fuzz["filters"]:
            visit(Fl._compile_filter_conditions(conds), ranges, sum(b - a for a, b in ranges))
    if {("const", True), ("const", False)} <= seen:
        seen.add(("kind", C_CONST))
    assert need <= seen, sorted(need - seen)
