"""Ordered hit lists built inside the multi-pattern body kernel, window by window (build_window_lists in scan.cu): the lists
of fei_scan_count / fei_scan_fetch_hits / fei_scan_hits must be the set bits of each query's column of the hit masks, in
record order, offset by the corpus' first global index; counts and (A, S) checksums must agree with them."""
import re

import numpy as np
import pytest

from fei_b200.program import C_BODY, C_SLOT, Cond, ProgramBuilder
from fei_b200.regexc import Pattern

pytestmark = pytest.mark.gpu

SEED = 0xB0D1
BASE = 123_456_789
SIZES = [1, 31, 4095, 4096, 4097, 3 * 4096 + 17, 80 * 4096 + 123]
BODY = 3                                                           # fei_scan_timing.body_kernel of k_body

BATCH32 = ["python", "docker|kubernetes", "neural networks", "react", "angular", "rust", "django", "flask", "terraform", "ansible",
           "microservices", "big data", "ci/cd", "git", "aws|azure|gcp", "spring boot", r"vue\.js", r"node\.js", "devops", "security",
           "blockchain", "testing", "databases", "algorithms", "cloud computing", "mobile development", "computer vision",
           "reinforcement learning", "ui/ux", "web development", "data structures", "machine learning"]
L = "abcdefghijklmnopqrstuvwxyz"
ALT4 = ["|".join(L[i] + L[j] + L[k] for j, k in [(1, 2), (3, 4), (5, 6), (7, 8)]) for i in range(20)]     # 80 accepting states
_rng = np.random.default_rng(7)
LONG = ["".join(L[int(x)] for x in _rng.integers(0, 26, 14)) for _ in range(24)]                   # > 385 states: class-indexed rows


def _body(p, negate=False):
    return Cond(C_BODY, pattern=Pattern("regex", p, re.IGNORECASE), negate=negate)


def _tag(t):
    return Cond(C_SLOT, pattern=Pattern("has_tag", t), field="Tags")


# name -> (queries, (body_direct, body_acc_mode) or None when the program has head conditions too)
PROGRAMS = {
    "batch32": ([[_body(p)] for p in BATCH32], (1, 2)),
    "acc1-negated-zero": ([[_body("python")], [_body("docker"), _body("rust", negate=True)], [_body("git", negate=True)],
                           [_body("zqxjzqxj")], [_body("react"), _body("angular")]], (1, 1)),
    "acc0": ([[_body(p)] for p in ALT4] + [[_body(p)] for p in BATCH32[:12]], (1, 0)),
    "class-indexed": ([[_body(p)] for p in LONG] + [[_body(p)] for p in BATCH32[:8]], (0, None)),
    "head-and-content": ([[_tag("python"), _body("docker")], [_tag("rust"), _body("kubernetes|terraform")], [_body("security")],
                          [_tag("python"), _body("git", negate=True)], [_tag("qzqzqz"), _body("python")]], None),
}
_built = {}


def _prog(name):
    if name not in _built:
        pb = ProgramBuilder()
        for q in PROGRAMS[name][0]:
            pb.add_query(q)
        _built[name] = pb.build()
    return _built[name], len(PROGRAMS[name][0])


@pytest.fixture(scope="module", params=SIZES)
def corpus(gpu, request):
    from fei_b200.corpus import Corpus
    c = Corpus().synth(SEED, BASE, request.param)
    yield c
    c.close()


def _checksums(lists):
    a, s = [], []
    for v in lists:
        k = np.arange(1, len(v) + 1, dtype=np.uint64)
        with np.errstate(over="ignore"):
            a.append(int((k * v).sum(dtype=np.uint64))); s.append(int(v.sum(dtype=np.uint64)))
    return a, s


def _check(c, name):
    prog, nq = _prog(name)
    expect = PROGRAMS[name][1]
    masks = c.scan_masks(prog)
    want = [np.nonzero((masks >> np.uint32(q)) & np.uint32(1))[0].astype(np.uint64) + np.uint64(BASE) for q in range(nq)]
    got = c.scan_hits(prog, nq)                                    # fei_scan_count, then fei_scan_fetch_hits
    tm = c.timing()
    assert tm["body_kernel"] == BODY, tm
    if expect is not None:
        assert tm["body_direct"] == expect[0], tm
        if expect[1] is not None:
            assert tm["body_acc_mode"] == expect[1], tm
        assert tm["kernel_launches"] == 1, tm                      # body only: the lists need no kernel of their own
    for q in range(nq):
        assert np.array_equal(got[q], want[q]), (name, q, len(got[q]), len(want[q]))
    a, s = c.list_checksums(nq)
    wa, ws = _checksums(want)
    assert [int(x) for x in a] == wa and [int(x) for x in s] == ws, name
    got2 = c.scan_hits(prog, nq, cap=max(1, c.n))                   # fei_scan_hits
    for q in range(nq):
        assert np.array_equal(got2[q], want[q]), (name, q)
    return want


@pytest.mark.parametrize("name", list(PROGRAMS))
def test_window_lists_equal_the_masks(corpus, name):
    want = _check(corpus, name)
    if corpus.n >= 4096 and name != "class-indexed":
        assert any(len(w) for w in want)                           # not vacuous


def test_two_programs_back_to_back(corpus):
    """The descriptors and window counters of one scan are reset for the next, whatever its query count."""
    want_a = _check(corpus, "batch32")
    _check(corpus, "acc1-negated-zero")
    prog, nq = _prog("batch32")
    got = corpus.scan_hits(prog, nq)
    for q in range(nq):
        assert np.array_equal(got[q], want_a[q])


def test_zero_hit_query_has_an_empty_list(corpus):
    prog, nq = _prog("acc1-negated-zero")
    counts = corpus.scan_count(prog, nq)
    assert int(counts[3]) == 0
