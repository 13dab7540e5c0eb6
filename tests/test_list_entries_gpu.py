"""The ordered hit lists are kept on the device as corpus-local 32-bit record indices and handed out as 64-bit global ones:
fei_scan_hits, fei_scan_fetch_hits (Corpus.scan_hits) and fei_scan_list_checksum must give global_base + local index for both
producers of the lists -- the multi-pattern body kernel (window by window) and the compaction after the scan (single-pattern,
header-only and gathered scans) -- with a global_base that puts every global index above 2^32 while the local ones stay small."""
import re

import numpy as np
import pytest

from fei_b200.program import C_BODY, C_SLOT, Cond, ProgramBuilder
from fei_b200.regexc import Pattern

pytestmark = pytest.mark.gpu

SEED = 0x5EED
BASE = (1 << 32) + 4_321                                           # global indices above 2^32, local ones far below
SIZES = [1, 31, 3 * 4096 + 17, 20 * 4096 + 5, 70_000]            # short last windows; 70 000 >= the gather kernel's minimum
WINDOW_KERNEL = 3                                                  # fei_scan_timing.body_kernel of k_body

BATCH = ["python", "docker|kubernetes", "neural networks", "react", "angular", "rust", "django", "flask", "terraform",
         "ansible", "microservices", "big data", "ci/cd", "git", "aws|azure|gcp"]


def _body(p, negate=False):
    return Cond(C_BODY, pattern=Pattern("regex", p, re.IGNORECASE), negate=negate)


def _tag(t):
    return Cond(C_SLOT, pattern=Pattern("has_tag", t), field="Tags")


# name -> (queries, whether k_body builds the lists inside the scan)
PROGRAMS = {
    "multi-15": ([[_body(p)] for p in BATCH], True),               # 15 queries: the last emit slice is partly empty
    "multi-3-negated": ([[_body("python")], [_body("docker"), _body("rust", negate=True)], [_body("zqxjzqxj")]], True),
    "single-pattern": ([[_body("kubernetes.*docker|docker.*kubernetes")]], False),
    "header-only": ([[_tag("python")], [_tag("rust")]], False),
    "header-and-one-pattern": ([[_tag("python"), _body("docker")]], False),
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
    n = request.param
    src = Corpus().synth(SEED, 0, n)
    a = src.fetch(0, n)
    src.close()
    a.update(n=n, global_base=BASE)
    c = Corpus().load(a)
    yield c
    c.close()


def _checksums(lists):
    a, s = [], []
    for v in lists:
        k = np.arange(1, len(v) + 1, dtype=np.uint64)
        with np.errstate(over="ignore"):
            a.append(int((k * v).sum(dtype=np.uint64))); s.append(int(v.sum(dtype=np.uint64)))
    return a, s


def _want(c, prog, nq):
    masks = c.scan_masks(prog)
    return [np.nonzero((masks >> np.uint32(q)) & np.uint32(1))[0].astype(np.uint64) + np.uint64(BASE) for q in range(nq)]


def _check_lists(c, name, want):
    prog, nq = _prog(name)
    got = c.scan_hits(prog, nq)                                    # fei_scan_count, then fei_scan_fetch_hits
    assert (c.timing()["body_kernel"] == WINDOW_KERNEL) == PROGRAMS[name][1], c.timing()
    for q in range(nq):
        assert got[q].dtype == np.uint64
        assert np.array_equal(got[q], want[q]), (name, q, len(got[q]), len(want[q]))
    a, s = c.list_checksums(nq)
    wa, ws = _checksums(want)
    assert [int(x) for x in a] == wa and [int(x) for x in s] == ws, name
    got2 = c.scan_hits(prog, nq, cap=max(1, c.n))                   # fei_scan_hits
    for q in range(nq):
        assert np.array_equal(got2[q], want[q]), (name, q)


@pytest.mark.parametrize("name", list(PROGRAMS))
def test_lists_hold_global_indices_above_2_32(corpus, name):
    prog, nq = _prog(name)
    want = _want(corpus, prog, nq)
    _check_lists(corpus, name, want)
    hits = [w for w in want if len(w)]
    if corpus.n >= 4096:
        assert hits                                                # not vacuous
    for w in hits:
        assert int(w[0]) >= 1 << 32 and int(w[-1]) - BASE < corpus.n


def test_short_caps_take_a_prefix(corpus):
    """fei_scan_hits with room for fewer entries than a list holds copies the list's first entries and reports FEI_E_CAPACITY."""
    import ctypes as C
    from fei_b200 import _abi
    prog, nq = _prog("multi-15")
    want = _want(corpus, prog, nq)
    cap_n = 5
    bufs = [np.full(cap_n, 7, dtype=np.uint64) for _ in range(nq)]
    ptrs = (C.c_void_p * 32)(*[b.ctypes.data for b in bufs])
    cap = np.zeros(32, dtype=np.uint64); cap[:nq] = cap_n
    nh = np.zeros(32, dtype=np.uint64)
    rc = _abi.lib().fei_scan_hits(corpus.handle, prog, len(prog), ptrs, _abi.ptr(cap), _abi.ptr(nh))
    assert rc == (_abi.FEI_E_CAPACITY if any(len(w) > cap_n for w in want) else _abi.FEI_OK)
    for q in range(nq):
        k = min(cap_n, len(want[q]))
        assert int(nh[q]) == len(want[q])
        assert np.array_equal(bufs[q][:k], want[q][:k]) and (bufs[q][k:] == 7).all(), q


def test_list_scan_then_mask_scan(corpus):
    """A mask-only scan after a list-building one (and the next list-building scan after it) sees nothing of the other."""
    prog_b, _ = _prog("header-and-one-pattern")
    masks_b = corpus.scan_masks(prog_b)
    prog_a, nq = _prog("multi-15")
    want = _want(corpus, prog_a, nq)
    _check_lists(corpus, "multi-15", want)
    assert np.array_equal(corpus.scan_masks(prog_b), masks_b)
    _check_lists(corpus, "multi-15", want)
    _check_lists(corpus, "single-pattern", _want(corpus, *_prog("single-pattern")))
