"""k_body's two row loops against the oracle.  Rows that hold 16 bytes of every one of a group's 32 records (all rows
but the shortest member's last) run in a loop without per-row lane counts or a partial-row test; the other rows keep the
ragged loop.  The groups here put the border between the two everywhere it can fall: on, just below and just above a
block of 16 rows, at 0, 1 and 2 rows, and in a window's last group with padded lanes."""
import numpy as np
import pytest

from fei_b200 import synth
from oracle import memdir_oracle as mo
from tests.test_body_early_exit_gpu import ALT2, ALT4, LONG, SMALL, _body, _check, _tokens

pytestmark = pytest.mark.gpu

# (units of the longer half, units of the shorter half) of successive groups of window 0, longest first: the shorter
# half's units less one is where the plain rows end
SHAPES = [(70, 49), (49, 49), (49, 48), (48, 34), (34, 33), (33, 33), (33, 32), (32, 31), (31, 18), (18, 17), (17, 17), (17, 16),
          (16, 15), (15, 3), (3, 3), (3, 2), (2, 2), (2, 1), (1, 1), (1, 0), (0, 0)]


def _group_units():
    """Units of the 4096 records of window 0, in an order the length sort keeps: 21 shaped groups between longer and
    shorter uniform ones, and the 70 records of window 1 (its last group has 26 padded lanes)."""
    units = []
    for g in range(100):
        units += [400 - 3 * g] * 32                                # 400 .. 103 units: every row plain but the last
    for hi, lo in SHAPES:
        units += [hi] * 16 + [lo] * 16
    units += [0] * (4096 - len(units))
    assert len(units) == 4096 and units == sorted(units, reverse=True)
    return units + [40] * 32 + [39] * 20 + [21] * 18


def _records():
    rng = np.random.default_rng(20261016)
    toks = [t.encode() for t in _tokens()]
    head = b".".join(toks) + b"."
    recs = []
    for i, u in enumerate(_group_units()):
        # a last row of 1, 15 or 16 bytes, or anything between
        n = 0 if u == 0 else 16 * (u - 1) + int([1, 15, 16, rng.integers(1, 17)][i % 4])
        body = bytearray(rng.choice(np.frombuffer(b"0123456789.", dtype=np.uint8), n).astype(np.uint8).tobytes())
        mode = i % 5
        if mode == 0 and n >= len(head):                           # decided in its first block while its neighbours read on
            body[0:len(head)] = head
        elif mode in (1, 2):
            for t in toks:
                where = int(rng.integers(7))                       # start, across the first block border, middle, last row, very end, absent
                if where < 5 and n >= len(t):
                    pos = [0, 256 - len(t) // 2, n // 2, n - 16 + int(rng.integers(16)), n - len(t)][where]
                    pos = max(0, min(pos, n - len(t)))
                    body[pos:pos + len(t)] = t
        elif mode == 3 and n >= 2:                                 # one token, ending the record
            t = toks[int(rng.integers(len(toks)))][:n]
            body[n - len(t):] = t
        r = synth.record(29, i)
        r["body"] = bytes(body)
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


@pytest.mark.parametrize("name,pats", [("<=32 accepting states", SMALL), ("<=32 accepting states, class-indexed", LONG),
                                       ("33-64 accepting states", ALT2), (">64 accepting states", ALT4)])
def test_plain_and_ragged_rows(corpus, name, pats):
    queries = [[_body(p)] for p in pats]
    queries[0] = [_body(pats[0]), _body(pats[1], negate=True)]
    queries[-1] = [_body(pats[2] + "$")]                           # read to the end: never decided early
    tm = _check(corpus, queries)
    assert tm["body_kernel"] == 3 and tm["body_acc_mode"] != 3, tm   # k_body, and not its single-pattern instance
