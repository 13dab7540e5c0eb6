"""k_body's per-lane early exit against the oracle: a lane stops reading its record once every content bit its alive
queries read is set, and must still write the hit mask a scan of the whole record would write."""
import re

import numpy as np
import pytest

from fei_b200 import synth
from fei_b200.program import C_BODY, C_SLOT, Cond, ProgramBuilder
from fei_b200.regexc import Pattern, compile_patterns
from oracle import memdir_oracle as mo

pytestmark = pytest.mark.gpu

L = "abcdefghijklmnopqrstuvwxyz"
SMALL = ["ka", "kb", "kc", "kd", "ke", "kf"]                   # all six fit in the first 16-byte row: "kakbkckdkekf"
ALT2 = ["|".join(L[i] + L[j] + L[k] for j, k in [(1, 2), (3, 4)]) for i in range(20)]           # 40 accepting states
ALT4 = ["|".join(L[i] + L[j] + L[k] for j, k in [(1, 2), (3, 4), (5, 6), (7, 8)]) for i in range(20)]   # 80
_rng = np.random.default_rng(5)
LONG = ["".join(L[int(x)] for x in _rng.integers(0, 26, 14)) for _ in range(32)]          # > 385 states: class-indexed rows


def _sample(p):
    return p.split("|")[0]


def _tokens():
    return [_sample(p) for p in SMALL + ALT2 + ALT4 + LONG] + ["kh", "ki"]


def _records():
    """Window 0 (4096 records, tiles sorted by length): groups 0-1 are 64 records of 3008 bytes whose every token sits at
    the start, group 2 is 32 records of 2512 bytes of which only the first carries tokens; the other records mix tokens
    placed at the start, in the middle, in the last row and at the very end.  Window 1 holds 70 records: its last group
    has 26 padded lanes."""
    rng = np.random.default_rng(20261015)
    toks = _tokens()
    head = "".join(SMALL).encode() + b"." + b".".join(t.encode() for t in toks[len(SMALL):]) + b"."

    def filler(n):
        return bytes(rng.choice(np.frombuffer(b"0123456789.", dtype=np.uint8), n).astype(np.uint8))

    def build(n, mode):
        body = bytearray(filler(n))
        if mode == "early":
            body[0:len(head)] = head
        elif mode == "mixed":
            for t in toks:
                tb = t.encode()
                where = int(rng.integers(6))                      # start, a third in, middle, last row, very end, absent
                if where < 5:
                    pos = [0, n // 3, n // 2, n - 16 + int(rng.integers(16)), n - len(tb)][where]
                    pos = min(pos, n - len(tb))
                    body[pos:pos + len(tb)] = tb
        elif mode == "late-one":                                  # every token early but one, which ends the record
            t = toks[int(rng.integers(len(toks)))].encode()
            body[0:len(head)] = head.replace(t, b"9" * len(t), 1)
            body[n - len(t):] = t
        return bytes(body)

    recs = []
    n = 4096 + 70
    for i in range(n):
        r = synth.record(23, i)
        if i < 64:
            r["body"] = build(3008, "early")
        elif i < 96:
            r["body"] = build(2512, "early" if i == 64 else "none")
        else:
            mode = ["mixed", "mixed", "late-one", "early", "none"][i % 5]
            r["body"] = build(int(rng.integers(len(head) + 2, 2400)), mode)
        tags = [b"qone"] if i % 3 == 0 else [b"qtwo"] if i % 3 == 1 else []
        r["hdr"] = re.sub(rb"Tags: [^\n]*\n", b"", r["hdr"]) + b"Tags: " + b",".join(tags + [b"misc"]) + b"\n"
        recs.append(r)
    return recs


@pytest.fixture(scope="module")
def corpus(gpu):
    from fei_b200.corpus import Corpus
    recs = _records()
    mems = [mo.make_memory(r["filename"], r["folder"], r["status"], synth.file_text(r), True) for r in recs]
    c = Corpus().load(synth.arrays_from_records(recs))
    yield c, mems
    c.close()


def _body(p, negate=False):
    return Cond(C_BODY, pattern=Pattern("regex", p, re.IGNORECASE), negate=negate)


def _tag(t):
    return Cond(C_SLOT, pattern=Pattern("has_tag", t), field="Tags")


def _want(mems, conds):
    """Records for which every condition holds, each condition judged by the oracle on its own."""
    every = set(range(len(mems)))
    out = set(every)
    for c in conds:
        if c.kind == C_BODY:
            s = set(mo.run_search(mems, [{"field": "content", "operator": "matches", "value": c.pattern.text}]))
            out &= (every - s) if c.negate else s
        else:
            out &= set(mo.run_search(mems, [{"field": "Tags", "operator": "has_tag", "value": c.pattern.text}]))
    return sorted(out)


def _check(corpus, queries):
    c, mems = corpus
    pb = ProgramBuilder()
    for q in queries:
        pb.add_query(q)
    masks = c.scan_masks(pb.build())
    for qi, q in enumerate(queries):
        got = np.nonzero((masks >> np.uint32(qi)) & np.uint32(1))[0].tolist()
        assert got == _want(mems, q), (qi, [x.pattern.text for x in q])
    return c.timing()


def _accepting(pats):
    d = compile_patterns([Pattern("regex", p, re.IGNORECASE) for p in pats])
    return int((d.out != 0).sum()), d.n_states


def test_decided_early_negated_and_two_conditions(corpus):
    """Six short patterns (<= 32 accepting states): the records of groups 0-1 are decided in their first row; a negated
    condition and a query with two content conditions are decided early too."""
    assert _accepting(SMALL)[0] <= 32
    queries = [[_body("ka")], [_body("kb")], [_body("kc"), _body("kd")], [_body("ke"), _body("kf", negate=True)], [_body("kf", negate=True)]]
    tm = _check(corpus, queries)
    assert tm["body_bytes_read"] < tm["body_bytes_touched"]        # lanes really stopped early


def test_end_anchored_patterns_are_read_to_the_end(corpus):
    """Bits that only the end-of-record verdict (endout) sets: records that need them are never decided early."""
    _check(corpus, [[_body("ka")], [_body("kh$")], [_body(r"ki\Z")], [_body("kb"), _body(r"kh\Z", negate=True)]])


def test_header_conditions_narrow_what_a_record_needs(corpus):
    """Head + body program: a record's alive queries decide which content bits it needs (a strict subset of the
    program's), so it may stop before the bits of queries its header already rejected are set."""
    queries = [[_tag("qone"), _body("ka"), _body("kh$")], [_tag("qtwo"), _body("kb")], [_tag("qone"), _body(_sample(LONG[3]))],
               [_body("kc"), _tag("qtwo")], [_tag("qtwo"), _body("kd", negate=True)]]
    _check(corpus, queries)


@pytest.mark.parametrize("name,pats,lo,hi", [("<=32 accepting states, class-indexed", LONG, 1, 32),
                                             ("33-64 accepting states", ALT2, 33, 64),
                                             (">64 accepting states", ALT4, 65, 10 ** 6)])
def test_accept_modes(corpus, name, pats, lo, hi):
    """The three ways k_body records accepting states (bits of a 32- / 64-bit register, or out[] per step)."""
    n_acc, n_states = _accepting(pats)
    assert lo <= n_acc <= hi, (name, n_acc)
    if pats is LONG:
        assert n_states > 385                                      # too big for byte-indexed rows (program.py)
    queries = [[_body(p)] for p in pats]
    queries[0] = [_body(pats[0]), _body(pats[1], negate=True)]
    tm = _check(corpus, queries)
    assert tm["body_bytes_read"] < tm["body_bytes_touched"]
