"""Differential fuzz of every content-scan kernel path against plain CPython: re.search(p, body, re.I) for `matches`,
needle in body.lower() for `contains`.  Which path a scan takes (k_body_sticky, k_body_gather, or k_body by row layout and
accept mode) is decided at scan time from the content automaton; every case asserts the path the scan reported
(Corpus.timing()) before it compares masks, ordered hit lists and counts bit for bit.  On a mismatch the message carries
the verdict of the CPU model of the serialized automaton (tests/blob_model.py), which tells a kernel bug from a table bug."""
import random
import re
import string

import numpy as np
import pytest

from fei_b200 import synth
from fei_b200.program import C_BODY, C_SLOT, Cond, ProgramBuilder
from fei_b200.regexc import Pattern
from tests.blob_model import BlobDfa
from tests.test_body_early_exit_gpu import ALT2, ALT4
from tests.test_regexc_fuzz import rand_regex

pytestmark = pytest.mark.gpu

STICKY, GATHER, BODY = 1, 2, 3                 # fei_scan_timing.body_kernel
ALL_PATHS = {(STICKY, 1, 3), (GATHER, 1, 3)} | {(BODY, 1, 3), (BODY, 0, 3)} | {(BODY, d, a) for d in (0, 1) for a in (0, 1, 2)}
SEEN = set()

_rng = random.Random(20261015)


def _words(k, n):
    return ["".join(_rng.choice(string.ascii_lowercase) for _ in range(n)) for _ in range(k)]


W8, W10, W14, W14B = _words(20, 8), _words(45, 10), _words(32, 14), _words(80, 14)
# @ ` [ { and the letters are exactly the bytes the tile permutation swaps (bit 5 ^= bit 6): @ <-> `, [ <-> {, A <-> a
SHORT = ["q@a", "z`b", "x[c", "w{d", "v\0e", "u@`f"]
STICKY_PAT = "k@j`b"
SIGMA = ["aσb", "aς", "ςz", "σ"]              # contains-needles: exact over text with capital sigmas (DESIGN 3.4)


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


def _anchored(pats, a, b):
    return pats + [_rx(re.escape(a) + "$"), _rx(re.escape(b) + r"\Z")]


# name -> (content patterns, the path they must take or None)
CASES = {
    "sticky": ([_rx(STICKY_PAT)], (STICKY, 1, 3)),
    "sticky-end": ([_rx(STICKY_PAT + "$")], (STICKY, 1, 3)),
    "direct-acc3": ([_rx("|".join(W8))], (BODY, 1, 3)),
    "class-acc3": ([_rx("|".join(W10))], (BODY, 0, 3)),
    "direct-acc1": (_anchored([_rx(re.escape(p)) for p in SHORT], SHORT[0], SHORT[1]), (BODY, 1, 1)),
    "class-acc1": (_anchored([_rx(p) for p in W14[:30]], W14[30], W14[31]), (BODY, 0, 1)),
    "direct-acc2": (_anchored([_rx(p) for p in ALT2], "abc", "bde"), (BODY, 1, 2)),
    "class-acc2": (_anchored([_rx("|".join(W14B[2 * i:2 * i + 2])) for i in range(20)], W14B[0], W14B[3]), (BODY, 0, 2)),
    "direct-acc0": ([_rx(p) for p in ALT4], (BODY, 1, 0)),
    "class-acc0": ([_rx("|".join(W14B[4 * i:4 * i + 4])) for i in range(20)], (BODY, 0, 0)),
    "sigma-contains": ([Pattern("contains", s) for s in SIGMA] + [_rx(STICKY_PAT + "$"), _rx("σ[a-z]")], None),
}
for _seed, _k in [(1, 3), (4, 6), (6, 6)]:
    _r = random.Random(_seed)
    _pats = []
    while len(_pats) < _k:
        _p = rand_regex(_r)
        try:
            re.compile(_p, re.IGNORECASE)
            _pats.append(_rx(_p))
        except re.error:
            pass
    CASES[f"rand-union-{_seed}"] = (_pats, None)

TOKENS = (W8 + W10 + W14 + W14B + SHORT + [STICKY_PAT] + [p.split("|")[0] for p in ALT2 + ALT4] + ["abc", "bde"]
          + ["AΣB", "aσb", "xAΣ", "AΣ.", "ςz", "σq", "ΣΣ"])

_ALPHA = list(string.ascii_letters) * 2 + ["@", "`", "[", "{", "\0", "é", "ß", "Ж", "日", "€", "\U0001F409", "K",
                                          "Σ", "ς", "σ", "İ", "\n", " "]
_ALPHA_B = [ch.encode() for ch in _ALPHA]
_ALPHA_LEN = np.array([len(b) for b in _ALPHA_B])


def _filler(rng, k):
    """Exactly k bytes of valid UTF-8 (1- to 4-byte characters, padded with ASCII)."""
    if k <= 0:
        return b""
    idx = rng.integers(len(_ALPHA), size=k)
    m = int(np.searchsorted(np.cumsum(_ALPHA_LEN[idx]), k, side="right"))
    out = b"".join([_ALPHA_B[i] for i in idx[:m]])
    return out + b"x" * (k - len(out))


def _body(rng, total, plants):
    """`total` bytes with the (offset, token) plants that fit without overlapping; stored bodies are stripped."""
    out, pos = [], 0
    for off, tok in sorted(plants):
        if off < pos or off + len(tok) > total:
            continue
        out += [_filler(rng, off - pos), tok]
        pos = off + len(tok)
    out.append(_filler(rng, total - pos))
    b = bytearray(b"".join(out))
    assert len(b) == total
    if total and b[:1] in (b" ", b"\n"):
        b[0:1] = b"x"
    if total and b[-1:] in (b" ", b"\n"):
        b[-1:] = b"x"
    return bytes(b)


def _length(rng, i):
    r = i % 20
    if r == 0:
        return 0
    if r in (1, 2):
        return int(rng.integers(1, 16))
    if r in (3, 4):
        return 16 * int(rng.integers(1, 300))                      # whole rows: no ragged tail
    if r == 5:
        return int(rng.choice([255, 256, 257, 4095, 4096, 4097]))    # around the 16-row decision block
    if r == 6 and i % 1000 == 6:
        return int(rng.integers(262150, 264000))
    if r == 7 and i % 200 == 7:
        return int(rng.integers(16400, 18000))
    return int(rng.integers(16, 5000))


def _plant(rng, total, tok):
    cands = [0, 4095, 4096, 4097, 16383, 16384, 16385, 262143, 262144, 262145, total - len(tok)]
    if total >= 32:
        cands.append(16 * int(rng.integers(1, total // 16)) - int(rng.integers(1, max(2, len(tok)))))   # straddles a row end
    cands.append(int(rng.integers(0, max(1, total))))
    return int(rng.choice(cands)), tok


def _token(rng):
    t = TOKENS[int(rng.integers(len(TOKENS)))]
    return (t.upper() if rng.random() < 0.3 else t).encode()


def _with_tags(r, tags):
    r["hdr"] = re.sub(rb"Tags: [^\n]*\n", b"", r["hdr"]) + b"Tags: " + b",".join([t.encode() for t in tags] + [b"misc"]) + b"\n"
    return r


class Reference:
    """Per-condition verdicts over the records' body strings, computed once per distinct condition."""

    def __init__(self, bodies, tags):
        self.texts = [b.decode() for b in bodies]
        self.lower = [t.lower() for t in self.texts]
        self.bodies = bodies
        self.tags = tags
        self.cache = {}

    def cond(self, c):
        key = (c.kind, c.pattern.kind, c.pattern.text)
        v = self.cache.get(key)
        if v is None:
            p = c.pattern
            if c.kind == C_SLOT:
                v = np.array([p.text in t for t in self.tags])
            elif p.kind == "contains":
                v = np.array([p.text in t for t in self.lower])
            else:
                rx = re.compile(p.text, re.IGNORECASE)
                v = np.array([rx.search(t) is not None for t in self.texts])
            self.cache[key] = v
        return v != c.negate

    def masks(self, queries):
        m = np.zeros(len(self.texts), dtype=np.uint32)
        for qi, q in enumerate(queries):
            ok = np.ones(len(self.texts), dtype=bool)
            for c in q:
                ok &= self.cond(c)
            m |= ok.astype(np.uint32) << np.uint32(qi)
        return m


def _load(recs):
    from fei_b200.corpus import Corpus
    return Corpus().load(synth.arrays_from_records(recs))


@pytest.fixture(scope="module")
def corpus(gpu):
    """2 windows of 4096 records + 37: the last group has padded lanes."""
    rng = np.random.default_rng(20261016)
    n = 2 * 4096 + 37
    recs, bodies, tags = [], [], []
    for i in range(n):
        total = _length(rng, i)
        b = _body(rng, total, [_plant(rng, total, _token(rng)) for _ in range(int(rng.integers(0, 5)))])
        t = ["ta"] if i % 3 == 0 else ["tb"] if i % 3 == 1 else []
        r = _with_tags(synth.record(31, i), t)
        r["body"] = b
        recs.append(r); bodies.append(b); tags.append(t + ["misc"])
    c = _load(recs)
    yield c, Reference(bodies, tags)
    c.close()


def _bc(p, negate=False):
    return Cond(C_BODY, pattern=p, negate=negate)


def _tag(t):
    return Cond(C_SLOT, pattern=Pattern("has_tag", t), field="Tags")


def _queries(pats, head):
    """Every pattern in a query of its own (the first 22) or paired with the next, a negated condition, a query with a
    content condition and a negated one, the first pattern in two queries; `head` adds header + content queries, so
    that a record's alive queries are a strict subset of the program's."""
    n = len(pats)
    qs = [[_bc(p)] for p in pats[:22]]
    rest = pats[22:]
    qs += [[_bc(rest[i]), _bc(rest[i + 1] if i + 1 < len(rest) else pats[0])] for i in range(0, len(rest), 2)]
    qs += [[_bc(pats[0]), _bc(pats[-1], negate=True)], [_bc(pats[n // 2], negate=True)], [_bc(pats[0])]]
    if head:
        qs += [[_tag("ta"), _bc(pats[1 % n])], [_bc(pats[-1], negate=True), _tag("tb")]]
    assert len(qs) <= 32
    return qs


def _program(queries):
    pb = ProgramBuilder()
    for q in queries:
        pb.add_query(q)
    return pb.build()


def predicted_path(prog):
    """The k_body variant run_scan picks for this program's content automaton (the sticky / gather choice aside)."""
    d = BlobDfa.from_program(prog)
    acc = 3 if d.sticky else 1 if d.n_acc <= 32 else 2 if d.n_acc <= 64 else 0
    direct = d.n_cols == 256
    sticky = direct and acc == 3 and d.n_states * d.row_stride * 2 + 4096 <= 65535
    return (STICKY if sticky else BODY, int(direct), acc)


def _path(tm):
    return (tm["body_kernel"], tm["body_direct"], tm["body_acc_mode"])


def _explain(prog, ref, queries, want, got):
    bad = np.nonzero(want != got)[0]
    r = int(bad[0])
    q = int(np.nonzero((want[r] ^ got[r]) >> np.arange(32, dtype=np.uint32) & 1)[0][0])
    m = BlobDfa.from_program(prog)
    return (f"{bad.size} records differ; record {r} (len {len(ref.bodies[r])}) query {q} "
            f"{[(c.pattern.kind, c.pattern.text, c.negate) for c in queries[q]]}: want {want[r] >> q & 1}, got {got[r] >> q & 1}; "
            f"CPU model of the serialized automaton gives content bits {m.run(ref.bodies[r]):#x}")


def _scan_all_ways(c, ref, queries, expect, monkeypatch, head):
    """head: the program has header conditions too, so it also runs with the unfused header pass."""
    prog = _program(queries)
    nq = len(queries)
    want = ref.masks(queries)
    want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
    ways = [{}, {"FEI_HEAD_FUSE": "0"}] if head else [{}]
    # body only: one scan launch; k_body builds the ordered lists itself, k_body_sticky's are compacted by three kernels after it
    launches = None if head else {BODY: 1, STICKY: 4}[expect[0]]
    for env in ways:
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            got = c.scan_masks(prog)
            tm = c.timing()
            assert _path(tm) == expect, (env, _path(tm), expect)
            SEEN.add(_path(tm))
            assert np.array_equal(got, want), (env, _explain(prog, ref, queries, want, got))
            hits = c.scan_hits(prog, nq)
            assert _path(c.timing()) == expect
            if launches is not None:
                assert c.timing()["kernel_launches"] == launches, (env, c.timing())
            counts = c.scan_count(prog, nq)
            if launches is not None:
                assert c.timing()["kernel_launches"] == launches, (env, c.timing())
        for q in range(nq):
            assert np.array_equal(hits[q], want_lists[q]), (env, q)
            assert int(counts[q]) == want_lists[q].size, (env, q)
    return want


@pytest.mark.parametrize("name", list(CASES))
def test_content_paths_agree_with_cpython(corpus, name, monkeypatch):
    c, ref = corpus
    pats, expect = CASES[name]
    for head in (False, True):
        queries = _queries(pats, head)
        path = predicted_path(_program(queries))
        if expect is not None:
            assert path == expect, (name, path)
        want = _scan_all_ways(c, ref, queries, path, monkeypatch, head=head)
        assert want.any() and (want != want[0]).any()                  # the case is not vacuous


# ---- the k_body_gather / k_body_sticky switch-over: 65536 records, so at most 4096 may be alive for k_body_gather
GATHER_N = 65536


@pytest.fixture(scope="module")
def gather_corpus(gpu):
    rng = np.random.default_rng(20261017)
    order = rng.permutation(GATHER_N)
    sel = {s: set(order[:s].tolist()) for s in (1, 4096, 4097)}
    base = [synth.record(37, i) for i in range(64)]
    recs, bodies, tags = [], [], []
    tok = STICKY_PAT.encode()
    for i in range(GATHER_N):
        t = [f"g{s}" for s in (1, 4096, 4097) if i in sel[s]]
        total = int(rng.integers(0, 700)) if rng.random() < 0.9 else int(rng.integers(700, 3000))
        if t:                                      # a record some query can select: the pattern at the start, the end or inside
            where = int(rng.integers(4))
            plants = [] if where == 3 or total < len(tok) else [(0 if where == 0 else total - len(tok) if where == 1 else int(rng.integers(0, total - len(tok) + 1)), tok)]
            b = _body(rng, total, plants)
        else:
            b = bytes((np.arange(total) % 26 + 97).astype(np.uint8))
        r = _with_tags(dict(base[i % 64]), t)
        r["body"] = b
        recs.append(r); bodies.append(b); tags.append(t + ["misc"])
    c = _load(recs)
    yield c, Reference(bodies, tags)
    c.close()


@pytest.mark.parametrize("selected,kernel", [(0, GATHER), (1, GATHER), (4096, GATHER), (4097, STICKY)])
def test_gather_switch_over(gather_corpus, selected, kernel, monkeypatch):
    """k_body_gather takes the scan when 0 < alive <= n / 16 records survive the header conditions, k_body_sticky
    above that; with none alive neither reads a byte."""
    c, ref = gather_corpus
    p = _rx(STICKY_PAT)
    g = f"g{selected}"
    queries = [[_tag(g), _bc(p)], [_tag(g), _bc(p, negate=True)], [_bc(p), _tag(g), _tag("misc")]]
    want = _scan_all_ways(c, ref, queries, (kernel, 1, 3), monkeypatch, head=True)
    if selected:
        assert (want & 1).any() and (selected == 1 or (want & 2).any())
    else:
        assert c.timing()["body_bytes_read"] == 0


def test_every_path_was_taken():
    assert SEEN == ALL_PATHS, sorted(ALL_PATHS - SEEN)
