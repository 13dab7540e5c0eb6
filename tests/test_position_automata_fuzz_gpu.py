"""Differential fuzz of the position-automaton kernels (k_body_nfa for content, nfa_run in the head kernels for header, flags
and name fields) against plain CPython re.search(p, text, re.I), with seeded random patterns up to the automaton's limits.

Patterns come from the grammar of tests/test_regexc_fuzz.rand_regex (atoms, classes, anchors, inline flags, quantifiers),
extended with bounded gaps and built together with a string each one matches, which is planted into bodies and header values
with gap lengths just inside and just outside the gap's bounds.  A size-targeted mode picks patterns by the serialized
section they give: position vectors of 32, 33, 64, 65, 128, 129, 255 and 256 bits, 128 classes, more than 1000 code point
ranges, 60 to 64 follow or accept groups.

Routing a random gap pattern the natural way costs seconds per pattern (the subset construction has to fail first), so most
cases mark their automaton-only patterns and a stand-in for fei_b200.program.cached_dfa refuses those at once; everything
else goes through the real ProgramBuilder.  A few cases route naturally.  On a content mismatch the message carries the CPU
model's verdict (tests/blob_nfa_model.py), which tells a table bug from a kernel bug.  test_generated_programs_agree_on_cpu
runs in the CPU suite: the generator, the size targets and the CPU model of every program against re."""
import random
import re
import string
import struct

import numpy as np
import pytest

from fei_b200 import program as P
from fei_b200 import synth
from fei_b200.program import (C_BODY, C_FLAGS, C_FOLDER_SET, C_NAME, C_SLOT, NAME_DATE_STR, NAME_FILENAME, NAME_HOST, NAME_ID,
                              NAME_TS_STR, VERSION_NFA, Cond, ProgramBuilder)
from fei_b200.regexc import PNA_MAX_CLASSES, Pattern, PatternTooLarge, compile_positions
from tests.blob_nfa_model import BlobNfa, program_content_bits
from tests.test_content_kernels_fuzz_gpu import Reference, _body, _length, _load, _plant, _queries, _with_tags
from tests.test_head_nfa_gpu import _arrays, _env, _head_sections, _records, _value, _want
from tests.test_regexc_fuzz import ATOMS

gpu = pytest.mark.gpu
NFA_KERNEL = 4                                   # fei_scan_timing.body_kernel
ALL_INSTANCES = {(w, d) for w in (1, 2, 4, 8) for d in (False, True)}    # k_body_nfa<W, kHasDfa>
SEEN = set()
_REAL_CACHED_DFA = P.cached_dfa


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


# ---------------------------------------------------------------- patterns with an example each
ANCHORS = ("^", "$", r"\b", r"\B", r"\A", r"\Z", "(?m:^)", "(?m:$)")
# strings each atom matches under re.I: case variants, the Kelvin sign and long s (which fold to k and s), 4-byte UTF-8
_EX = {"a": ["a", "A"], "b": ["b", "B"], "k": ["k", "K", "K"], "s": ["s", "S", "ſ"], "K": ["k", "K"], r"\.": ["."],
       ".": ["x", "é", "日", "-", "\U0001F409"], r"\w": ["a", "Z", "é", "日", "_", "5", "Σ", "K", "ſ"], r"\W": [" ", "-", "@", "€", "\n"],
       r"\d": ["0", "7"], r"\s": [" ", "\t", "\n"], r"\S": ["x", "é", "-"], "[ab]": ["a", "B"], "[^a]": ["b", "é", " "],
       "[a-k]": ["c", "K"], "[k-s]": ["m", "S", "ſ"], r"[\w-]": ["-", "a", "é"], "é": ["é", "É"], "ß": ["ß"], "日": ["日"], " ": [" "],
       "-": ["-"], ",": [","], "[é日]": ["é", "日"], r"[^\W\d]": ["a", "é", "Σ", "ſ"], "/": ["/"], "\n": ["\n"], "Σ": ["σ", "Σ", "ς"],
       "ſ": ["s", "ſ"], "K": ["k", "K"]}
ATOMS_X = ATOMS + ["(?m:^)", "(?m:$)", "\n", "Σ", "ſ", "K"]
_QUANTIFIED = re.compile(r"(?<!\()[*+?]|\{\d")
_QUANT = {"*": (0, 3), "+": (1, 3), "?": (0, 1), "{2}": (2, 2), "{1,2}": (1, 2), "{0,1}": (0, 1), "*?": (0, 3), "+?": (1, 3)}


def _example_regex(rng, depth=0):
    """rand_regex's grammar, each part with a string it matches on its own: (regex, example)."""
    parts, ex = [], []
    for _ in range(rng.randint(1, 4)):
        r = rng.random()
        if depth < 2 and r < 0.2:
            p, e = _example_regex(rng, depth + 1)
            p = rng.choice(["(%s)", "(?:%s)", "(?i:%s)", "(?-i:%s)", "(?s:%s)", "(?m:%s)"]) % p
        elif depth < 2 and r < 0.3:
            (p1, e1), (p2, e2) = _example_regex(rng, depth + 1), _example_regex(rng, depth + 1)
            p, e = "(?:%s|%s)" % (p1, p2), rng.choice([e1, e2])
        else:
            p = rng.choice(ATOMS_X)
            e = rng.choice(_EX[p]) if p in _EX else ""
        # no quantifier on a group that holds one: nested repeats make CPython's backtracking, the reference, exponential
        if p not in ANCHORS and rng.random() < 0.3 and not _QUANTIFIED.search(p):
            q = rng.choice(list(_QUANT))
            p, e = p + q, e * rng.randint(*_QUANT[q])
        parts.append(p); ex.append(e)
    return "".join(parts), "".join(ex)


def example_regex(rng, nonempty=False):
    """A random regex and a string re.search(regex, string, re.I) matches; drawn again until the example matches."""
    while True:
        p, e = _example_regex(rng)
        if nonempty and not e:
            continue
        try:
            if re.search(p, e, re.IGNORECASE):
                return p, e
        except re.error:
            pass


_FILL = {"dot": ["x", "é", "日", "-", " ", "\U0001F409", "Σ", "K", "@", "`"], "notx": ["a", "é", " ", "-", "日", "\n", "ſ"],
         "any": ["x", "\n", "é", " ", "\U0001F409"], "nonword": [" ", "-", "@", "€", ",", "\n", "`"]}
_GAP_KINDS = [(".{%d,%d}", "dot"), ("[^x]{%d,%d}", "notx"), ("(?s:.){%d,%d}", "any"), (r"\W{%d,%d}", "nonword"), ("words", "words")]
_WORDS = ["alpha", "é", "日本", "x1", "Σς", "KING"]


def _fill(rng, kind, k):
    """k characters (k words for the word gap) a gap of this kind takes."""
    if kind == "words":
        return " " + "".join(rng.choice(_WORDS) + rng.choice([" ", ", ", "-"]) for _ in range(k))
    return "".join(rng.choice(_FILL[kind]) for _ in range(k))


def gap_ends(rng, kinds=_GAP_KINDS):
    """The two ends (regex, example) of a gap pattern and the gap's kind."""
    return example_regex(rng, nonempty=True), example_regex(rng, nonempty=True), rng.choice(kinds)


def gap_regex(rng, m, n, ends=None):
    """A + bounded gap + B, and examples with gap lengths m - 1, m, n and n + 1 (word counts for \\W+(?:\\w+\\W+){0,n}):
    (regex, [example, ...]).  The ends are drawn again until the examples inside the bounds match (an anchor at an end can
    rule a gap out); the examples outside the bounds may or may not match.  With `ends` given: None when it does not."""
    while True:
        (a, ea), (b, eb), (g, kind) = ends or gap_ends(rng)
        if kind == "words":
            m, gap = 0, r"\W+(?:\w+\W+){0,%d}" % n
            a, b, ea, eb = a + "x", "x" + b, ea + "x", "x" + eb        # a word character on both sides of the gap
        else:
            gap = g % (m, n)
        p = "(?:%s)%s(?:%s)" % (a, gap, b)
        lens = sorted({max(0, m - 1), m, n, n + 1})
        exs = [ea + _fill(rng, kind, k) + eb for k in lens]
        if all(re.search(p, e, re.IGNORECASE) for e, k in zip(exs, lens) if m <= k <= n):
            return p, exs
        if ends:
            return None


def _compiles(pats):
    try:
        return compile_positions([_rx(p) for p in pats])
    except PatternTooLarge:
        return None


def sized(rng, fixed, n_pos, kinds=_GAP_KINDS[:4]):
    """One gap pattern whose upper bound is tuned until the automaton of `fixed` + it has exactly n_pos positions:
    (the gap pattern, its examples)."""
    while True:
        ends, m = gap_ends(rng, kinds), rng.randint(0, 3)
        n, a = max(m, n_pos // 2), None
        for _ in range(12):
            got = gap_regex(rng, m, n, ends)
            if got is None:
                break
            p, exs = got
            a = _compiles(fixed + [p])
            if a is None or a.n_pos == n_pos or n + n_pos - a.n_pos < m:
                break
            n += n_pos - a.n_pos
        if a is not None and a.n_pos == n_pos:
            return p, exs


ENDS = ["", r"\b", r"\B", "$", "(?m:$)", r"\Z"]
_END_EX = {"": "", r"\b": " ", r"\B": "", "$": "", "(?m:$)": "\n", r"\Z": ""}


def anchored(rng):
    """An alternation of one-character branches, each behind a different end anchor: several accept groups per pattern
    (regex, [example of each branch])."""
    br = [(rng.choice(["a", "é", "k", "s", "日", r"\w", "-", "[ab]", "Σ"]), e) for e in rng.sample(ENDS, rng.randint(3, 6))]
    return "(?:%s)" % "|".join(c + e for c, e in br), [rng.choice(_EX.get(c, ["a"])) + _END_EX[e] for c, e in br]


def _cjk(k, step=1):
    return "".join(chr(0x4E00 + step * i) for i in range(k))


# ---------------------------------------------------------------- content programs
# name -> (automaton-only patterns, DFA patterns, examples to plant, natural routing)
def _content_case(name):
    rng = random.Random(f"content-{name}")
    words = ["".join(rng.choice(string.ascii_lowercase) for _ in range(rng.randint(4, 9))) for _ in range(24)]
    dfa = [re.escape(w) for w in words[:rng.randint(1, 4)]]
    exs = list(words[:4])
    nfa = []

    def add(p, e):
        """Add p when the automaton of the case's patterns with it stays within the limits."""
        if p not in nfa and p not in dfa and _compiles(nfa + [p]) is not None:
            nfa.append(p); exs.extend(e)

    kind, _, arg = name.partition("-")
    if kind == "gap":                              # 1 to 6 gap patterns, a DFA beside them in every other case
        for _ in range(rng.randint(1, 6)):
            m = rng.randint(0, 8)     # n - m from 0 to 70: one- to eight-word vectors
            add(*gap_regex(rng, m, m + rng.choice([0, 1, 5, 20, 40, 70])))
        if rng.random() < 0.4:
            p, e = example_regex(rng)
            add(p, [e])
        if int(arg) % 2:
            dfa = []
    elif kind == "size":                           # exactly n_pos positions: W and the word edges
        n_pos, has_dfa = int(arg.split(".")[0]), arg.endswith("dfa")
        fixed = [gap_regex(rng, 1, 3)] if n_pos > 40 else []
        for p, e in fixed:
            add(p, e)
        add(*sized(rng, nfa[:], n_pos))
        if not has_dfa:
            dfa = []
    elif kind == "classes":                        # 128 code point classes: one per CJK letter
        for k in range(PNA_MAX_CLASSES, 100, -1):
            p = "x.{0,8}" + _cjk(k - 4, 3)
            a = _compiles([p])
            if a and len(a.cls_b) == PNA_MAX_CLASSES:
                break
        add(p, ["x" + "é" * 8 + _cjk(k - 4, 3), "x日" + _cjk(k - 4, 3)])
    elif kind == "ranges":                         # Unicode word classes: more than 1000 ranges
        add(r"[^\W\d].{0,40}\w\b", ["Σ" + "x" * 40 + "ſ", "ſ-K", "日" * 50])
        add(r"\d\W{2,30}[^\W\d]", ["7  é", "0" + "@" * 30 + "ſ"])
        dfa = dfa if int(arg) else []
    elif kind == "follow":                         # 60 to 64 follow groups
        while True:
            pats = list(dict(example_regex(rng) for _ in range(rng.randint(24, 30))).items())
            a = _compiles([p for p, _e in pats])
            if a and 60 <= len(a.follow) <= 64:
                break
        for p, e in pats:
            add(p, [e])
        dfa = dfa[:32 - len(pats)]
    elif kind == "accept":                         # 60 to 64 accept groups
        while True:
            pats = list(dict(anchored(rng) for _ in range(rng.randint(12, 20))).items())
            a = _compiles([p for p, _e in pats])
            if a and 60 <= len(a.accept) <= 64:
                break
        for p, e in pats:
            add(p, e)
        dfa = dfa[:32 - len(pats)]
    elif kind == "bits32":                         # 24 DFA patterns + 8 automaton ones: an automaton output at bit 31
        dfa = [re.escape(w) for w in words]
        exs = list(words)
        while len(nfa) < 8:
            add(*gap_regex(rng, 1, rng.choice([3, 12, 20])))
    elif kind == "empty":                          # patterns that match the empty string, end-only accepts
        for p in (r"(?:%s)?\Z", r"^(?:%s)?$", r"(?:%s|\A)(?m:$)", r"(?:%s)*\B"):
            g, e = gap_regex(rng, 0, rng.choice([6, 30]))
            add(p % g, e)
        add(*gap_regex(rng, 2, 9))
    elif kind == "natural":                        # no stand-in: the DFA refuses the gap patterns itself
        a, b = rng.sample(["kubernetes", "docker", "deploy", "fail", "python", "rust"], 2)
        n = rng.choice([50, 70])
        add(r"\b%s\b.{0,%d}\b%s" % (a, n, b), [f"{a} {'x' * (n - 2)} {b}", f"{a} -{'é' * n} {b}", f"{a}{b}"])
        return nfa, dfa, exs, True
    else:
        raise KeyError(name)
    return nfa, dfa, exs, False


CONTENT = ([f"gap-{i}" for i in range(10)] + [f"size-{n}.{d}" for n, d in ((32, "dfa"), (32, "no"), (33, "no"), (64, "dfa"), (65, "dfa"),
           (128, "no"), (129, "no"), (255, "dfa"), (256, "no"), (256, "dfa"))]
           + ["classes-0", "ranges-0", "ranges-1", "follow-0", "accept-0", "bits32-0", "empty-0", "natural-0", "natural-1"])
_CASES = {}


def content_case(name):
    if name not in _CASES:
        _CASES[name] = _content_case(name)
    return _CASES[name]


def _forced(automaton_only):
    """A stand-in for fei_b200.program.cached_dfa that refuses every pattern set holding an automaton-only pattern."""
    texts = set(automaton_only)

    def cached_dfa(patterns, sticky=False):
        if any(p.text in texts for p in patterns):
            raise PatternTooLarge("automaton-only in this test")
        return _REAL_CACHED_DFA(patterns, sticky)
    return cached_dfa


def _build(queries, automaton_only, monkeypatch):
    with monkeypatch.context() as mp:
        if automaton_only:
            mp.setattr(P, "cached_dfa", _forced(automaton_only))
        pb = ProgramBuilder()
        for q in queries:
            pb.add_query(q)
        return pb.build()


_PROGS = {}


def content_program(name, head, monkeypatch):
    """(queries, program, the patterns in content-bit order) of a content case."""
    key = (name, head)
    if key not in _PROGS:
        nfa, dfa, _exs, natural = content_case(name)
        rng = random.Random(f"order-{name}")
        pats = [_rx(p) for p in nfa + dfa]
        rng.shuffle(pats)
        queries = _queries(pats, head)
        _PROGS[key] = (queries, _build(queries, [] if natural else nfa, monkeypatch))
    return _PROGS[key]


def _check_content_program(name, prog):
    """The program holds what the case asks for: its automaton sizes and whether a body DFA steps alongside."""
    nfa, dfa, _exs, natural = content_case(name)
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA, name
    m = BlobNfa.from_program(prog)
    has_dfa = struct.unpack_from("<I", prog, 40)[0] != 0
    if not natural:
        a = compile_positions([_rx(p) for p in nfa])
        assert (m.W, m.n_pos, m.n_patterns, m.first_bit, has_dfa) == (a.n_words, a.n_pos, len(nfa), len(dfa), bool(dfa)), name
    kind, _, arg = name.partition("-")
    if kind == "size":
        assert m.n_pos == int(arg.split(".")[0]) and m.W == {32: 1, 33: 2, 64: 2, 65: 4, 128: 4}.get(m.n_pos, 8), name
    elif kind == "classes":
        assert m.n_classes == PNA_MAX_CLASSES, m.n_classes
    elif kind == "ranges":
        assert m.n_ranges > 1000, m.n_ranges
    elif kind == "follow":
        assert 60 <= m.n_follow <= 64, m.n_follow
    elif kind == "accept":
        assert 60 <= m.n_accept <= 64, m.n_accept
    elif kind == "bits32":
        assert (m.first_bit, m.n_patterns) == (24, 8)
    elif kind == "empty":
        assert any(eo for _s, _m, _b, eo in m.accept), "no end-only accept"
    return m, has_dfa


# ---------------------------------------------------------------- content scans (k_body_nfa)
N_CONTENT = 4096 + 37                            # one window and a group with padded lanes


def _smem_words():
    rng = random.Random(2206)
    return ["".join(rng.choice(string.ascii_lowercase) for _ in range(12)) for _ in range(178)]


def _content_tokens():
    smem = _smem_words()[:6] + ["q" + "-" * n + chr(0x4E00 + 2 * j) for n in (0, 119, 120, 121) for j in (0, 500)]
    return [e.encode() for e in smem + [e for name in CONTENT for e in content_case(name)[2]]]


def _content_length(rng, i):
    """_length's shapes with the long bodies (262 KiB, 16 KiB, up to 5000 bytes) kept to a few records: the reference runs
    CPython's re over every body for every pattern."""
    t = _length(rng, i)
    if t > 640 and i % 20 != 5 and i not in (6, 7, 207):
        t = int(rng.integers(16, 640))
    return t


@pytest.fixture(scope="module")
def corpus(gpu):
    """The shapes of the content-kernel fuzz (empty bodies, ragged rows, lengths around 16 and 4096 bytes, multi-byte UTF-8,
    the bytes the tile permutation swaps) with the cases' examples planted, one in the first row or at the last byte of
    every third record."""
    tokens = _content_tokens()
    rng = np.random.default_rng(20261018)
    recs, bodies, tags = [], [], []
    for i in range(N_CONTENT):
        total = _content_length(rng, i)
        tok = lambda: tokens[int(rng.integers(len(tokens)))]            # noqa: E731
        plants = [_plant(rng, total, tok()) for _ in range(int(rng.integers(0, 5)))]
        if i % 3 == 0:
            t = tok()
            plants.append((0, t) if i % 2 else (total - len(t), t))
        b = _body(rng, total, plants)
        t = ["ta"] if i % 3 == 0 else ["tb"] if i % 3 == 1 else []
        r = _with_tags(synth.record(43, i), t)
        r["body"] = b
        recs.append(r); bodies.append(b); tags.append(t + ["misc"])
    c = _load(recs)
    yield c, Reference(bodies, tags)
    c.close()


def _explain(prog, ref, queries, want, got):
    bad = np.nonzero(want != got)[0]
    r = int(bad[0])
    q = int(np.nonzero((want[r] ^ got[r]) >> np.arange(32, dtype=np.uint32) & 1)[0][0])
    return (f"{bad.size} records differ; record {r} (len {len(ref.bodies[r])}) query {q} "
            f"{[(c.pattern.text, c.negate) for c in queries[q]]}: want {want[r] >> q & 1}, got {got[r] >> q & 1}; "
            f"CPU model of the serialized automata gives content bits {program_content_bits(prog, ref.bodies[r]):#x}")


def _scan_content(c, ref, queries, prog, words, monkeypatch, head):
    nq = len(queries)
    want = ref.masks(queries)
    want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
    for env in ([{}, {"FEI_HEAD_FUSE": "0"}] if head else [{}]):
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            got = c.scan_masks(prog)
            tm = c.timing()
            assert (tm["body_kernel"], tm["body_nfa_words"]) == (NFA_KERNEL, words), (env, tm)
            assert np.array_equal(got, want), (env, _explain(prog, ref, queries, want, got))
            hits = c.scan_hits(prog, nq)
            assert c.timing()["body_kernel"] == NFA_KERNEL
            counts = c.scan_count(prog, nq)
        for q in range(nq):
            assert np.array_equal(hits[q], want_lists[q]), (env, q)
            assert int(counts[q]) == want_lists[q].size, (env, q)
    return want


@gpu
@pytest.mark.parametrize("name", CONTENT)
def test_content_automata_agree_with_cpython(corpus, name, monkeypatch):
    c, ref = corpus
    for head in (False, True):
        queries, prog = content_program(name, head, monkeypatch)
        m, has_dfa = _check_content_program(name, prog)
        want = _scan_content(c, ref, queries, prog, m.W, monkeypatch, head)
        SEEN.add((m.W, has_dfa))
        # the case is not vacuous: most queries hit some records and miss others (a random pattern may match everywhere, or
        # only in a context no planted example has)
        split = [q for q in range(len(queries)) if (want >> np.uint32(q) & 1).any() and not (want >> np.uint32(q) & 1).all()]
        assert 2 * len(split) >= len(queries), (name, head, len(split), len(queries))


BODY_SMEM = 220 * 1024                           # the body kernels' dynamic shared memory (scan.cu)


def _smem_case(over, monkeypatch):
    """A body DFA of some 200 KiB and a position automaton whose range table is grown, 12 bytes per CJK letter of a class,
    until the two tables together come just under (or just over) the body kernels' shared memory: (program, queries,
    DFA table bytes, automaton table bytes)."""
    words = _smem_words()
    big = "|".join(words)
    dfa_bytes = P._table_bytes(_REAL_CACHED_DFA([_rx(big)]), 0)
    k = 100
    for _ in range(6):
        gap = r"q.{0,120}[%s]" % _cjk(k, 2)
        nfa_bytes = P._nfa_table_bytes(compile_positions([_rx(gap)]))
        room = BODY_SMEM - dfa_bytes - nfa_bytes
        if (-256 < room <= 0) if over else (0 <= room < 256):
            break
        k += (room - (-128 if over else 128)) // 12
    queries = [[Cond(C_BODY, pattern=_rx(big))], [Cond(C_BODY, pattern=_rx(gap))], [Cond(C_BODY, pattern=_rx(gap), negate=True)],
               [Cond(C_BODY, pattern=_rx(big)), Cond(C_BODY, pattern=_rx(gap))]]
    with monkeypatch.context() as mp:
        if over:                                 # the builder refuses it too: let it through to see the scan refuse it
            mp.setattr(P, "BODY_SMEM_LIMIT", 227 * 1024)
        prog = _build(queries, [gap], mp)
    return prog, queries, dfa_bytes, nfa_bytes, words, gap, k


@gpu
def test_tables_at_the_shared_memory_ceiling(corpus, monkeypatch):
    c, ref = corpus
    prog, queries, dfa_bytes, nfa_bytes, words, gap, k = _smem_case(False, monkeypatch)
    m, has_dfa = BlobNfa.from_program(prog), struct.unpack_from("<I", prog, 40)[0] != 0
    assert has_dfa and m.table_bytes == nfa_bytes and struct.unpack_from("<I", prog, struct.unpack_from("<I", prog, 40)[0] + 44)[0] == dfa_bytes
    assert BODY_SMEM - 256 < dfa_bytes + nfa_bytes <= BODY_SMEM, (dfa_bytes, nfa_bytes)
    assert dfa_bytes > 6 * 32768 and dfa_bytes % 32768, dfa_bytes        # several bulk copies; the automaton starts mid-chunk
    want = _scan_content(c, ref, queries, prog, m.W, monkeypatch, False)
    assert all((want >> np.uint32(q) & 1).any() for q in range(3)), "a query without hits"
    SEEN.add((m.W, True))
    over, *_ = _smem_case(True, monkeypatch)
    total = struct.unpack_from("<I", over, struct.unpack_from("<I", over, 40)[0] + 44)[0] + BlobNfa.from_program(over).table_bytes
    assert BODY_SMEM < total < BODY_SMEM + 256, total
    with pytest.raises(NotImplementedError, match="220 KiB"):          # FEI_E_UNSUPPORTED, before any launch
        c.scan_masks(over)
    assert np.array_equal(c.scan_masks(prog), ref.masks(queries))       # the context still scans


@gpu
def test_every_content_instance_was_taken():
    assert SEEN == ALL_INSTANCES, sorted(ALL_INSTANCES - SEEN)


# ---------------------------------------------------------------- head fields (nfa_run in the head kernels)
N_HEAD = 4096 + 300
HEAD_LENS = [15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65]     # around the 16-byte units and the 64-byte value column
_HEAD_PAD = ["a", "Z", "-", "0", " ", "é", "日", "\U0001F409", "Σ", "K", "ſ"]
HOSTS = ["h", "db01", "build-box-17", "mail.example.org", "x" * 16, "node-" + "7" * 28, "edge-é"[:5]]
FLAG_LETTERS = "ABDFPRST"


def _pad(rng, k):
    out = []
    while k > 0:
        ch = rng.choice(_HEAD_PAD)
        if len(ch.encode()) <= k:
            out.append(ch); k -= len(ch.encode())
    return "".join(out)


def head_value(rng, token, length):
    """A header value of `length` UTF-8 bytes (more when the token is longer) holding `token`, padded with 1- to 4-byte
    characters that straddle the 16-byte units; no blank at either end (the headers dict holds stripped values)."""
    room = max(0, length - len(token.encode()))
    left = rng.choice([0, room, rng.randint(0, room)])
    v = _pad(rng, left) + token + _pad(rng, room - left)
    if v[:1].isspace():
        v = "x" + v[1:]
    if v[-1:].isspace():
        v = v[:-1] + "x"
    return v


def _head_patterns(seed):
    """Automaton patterns for header values and their examples (no line breaks): gap patterns of every width and random
    grammar patterns."""
    rng = random.Random(seed)
    out = []
    while len(out) < 24:
        if len(out) % 3 == 2:
            p, e = example_regex(rng, nonempty=True)
            exs = [e]
        else:
            m = rng.randint(0, 4)
            p, exs = gap_regex(rng, m, m + rng.choice([2, 10, 40, 90, 180]))
        exs = [e for e in exs if "\n" not in e and "\r" not in e]
        if exs and _compiles([p]) is not None:
            out.append((p, exs))
    return out


_HEAD_SIZED = []


def head_sized():
    """Slot patterns of 32, 33, 64, 65, 128, 129, 255 and 256 positions, with examples that fit a header line."""
    if not _HEAD_SIZED:
        rng = random.Random(20261020)
        for n in (32, 33, 64, 65, 128, 129, 255, 256):
            while True:
                p, exs = sized(rng, [], n, _GAP_KINDS[:1])
                exs = [e for e in exs if "\n" not in e and "\r" not in e]
                if exs:
                    break
            _HEAD_SIZED.append((p, exs))
    return _HEAD_SIZED


def head_records():
    """_records with generated header values planted at the unit and column edges, flags of up to 7 letters (all flags8
    holds) and file names over several host names."""
    recs, heads = _records(N_HEAD, 20261019)
    rng = random.Random(20261019)
    pool = [e for _p, exs in _head_patterns(1) + head_sized() for e in exs]
    for i, (r, h) in enumerate(zip(recs, heads)):
        for k in list(h):
            if rng.random() < 0.7:
                h[k] = head_value(rng, rng.choice(pool) if rng.random() < 0.8 else "", rng.choice(HEAD_LENS))
        r["hdr"] = "".join(f"{k}: {v}\n" for k, v in h.items()).encode()
        n_flags = 7 if i % 11 == 0 else rng.randint(0, 6)
        r["flags"] = "".join(sorted(rng.sample(FLAG_LETTERS, n_flags)))
        r["filename"] = f"{r['ts']}.{r['uid']}.{HOSTS[i % len(HOSTS)]}:2,{r['flags']}"
    return recs, heads


def _name_value(rec, which):
    return _value(rec, {}, Cond(C_NAME, which=which))


def derived(rng, values):
    """A gap pattern cut out of one of the values: two pieces with a gap whose bounds are just around the distance between
    them, or just outside it."""
    while True:
        v = rng.choice(values)
        a, b = rng.randint(1, 3), rng.randint(1, 2)
        if len(v) < a + b:
            continue
        i = rng.randint(0, len(v) - a - b)
        j = rng.randint(i + a, len(v) - b)
        g = j - i - a
        m, n = rng.choice([(g, g), (max(0, g - 2), g), (g, g + 3), (g + 1, g + 4), (0, max(0, g - 1))])
        gap = rng.choice([".{%d,%d}", "[^x]{%d,%d}", "(?s:.){%d,%d}", r"\S{%d,%d}"]) % (m, n)
        return rng.choice(["", "^", r"\b"]) + re.escape(v[i:i + a]) + gap + re.escape(v[j:j + b])


def flag_regex(rng):
    a, b = rng.choice(FLAG_LETTERS), rng.choice(FLAG_LETTERS)
    return rng.choice(["", "^"]) + a + rng.choice([".{%d,%d}", r"\w{%d,%d}", "[^x]{%d,%d}"]) % (0, rng.randint(0, 5)) + b + rng.choice(["", "$"])


def _slot(field, p, mode=0, **kw):
    return Cond(C_SLOT, pattern=_rx(p), field=field, mode=mode, **kw)


def _head_program(name, recs, heads):
    """(queries, automaton-only patterns) of a head case; every query is drawn again until it hits some records and misses
    others."""
    rng = random.Random(f"head-{name}")
    pats = _head_patterns(1)
    pat = lambda: rng.choice(pats)[0]                                  # noqa: E731
    names = {w: sorted({_name_value(r, w) for r in recs[:200]}) for w in (NAME_FILENAME, NAME_ID, NAME_HOST, NAME_TS_STR, NAME_DATE_STR)}
    if name == "slots":                    # modes 0, 1, 2, empty_if_missing, negation
        makes = [lambda: [_slot("subject", pat())], lambda: [_slot("Subject", pat(), 1)], lambda: [_slot("x", pat(), 2)],
                 lambda: [_slot("Status", "^(?:%s)?$" % pat(), 1, empty_if_missing=True)],
                 lambda: [_slot("Status", "(?:%s)|^$" % pat(), 1, empty_if_missing=True, negate=True), _slot("SUBJECT", pat())],
                 lambda: [_slot("X-Note", pat(), 1)], lambda: [_slot("x-note", pat(), negate=True)], lambda: [_slot("status", pat())]]
    elif name == "sizes":                  # one- to eight-word vectors on the slots
        sized_pats = [p for p, _exs in head_sized()]
        slots = [("subject", 0), ("Subject", 1), ("x-note", 0), ("X-Note", 1), ("status", 0), ("Status", 1), ("a", 2), ("b", 2)]
        makes = [(lambda f=f, mode=mode, p=p: [_slot(f, p, mode)]) for (f, mode), p in zip(slots, sized_pats)]
    elif name == "flags":                  # flags8 and both header-or-fallback pairs
        makes = [lambda: [Cond(C_FLAGS, pattern=_rx(flag_regex(rng)))], lambda: [Cond(C_FLAGS, pattern=_rx(flag_regex(rng)), negate=True)],
                 lambda: [_slot("flags", pat(), if_missing=2), Cond(C_FLAGS, pattern=_rx(flag_regex(rng)))],
                 lambda: [_slot("unique_id", pat(), if_missing=2), Cond(C_NAME, which=NAME_ID, pattern=_rx(derived(rng, names[NAME_ID])))],
                 lambda: [Cond(C_FLAGS, pattern=_rx(flag_regex(rng))), _slot("Subject", pat())]]
    elif name == "names":                  # all five name fields
        makes = [(lambda w=w, neg=neg: [Cond(C_NAME, which=w, pattern=_rx(derived(rng, names[w])), negate=neg)])
                 for w in names for neg in (False, True)]
    elif name == "mixed":                  # a DFA and an automaton on the same fields; a folder predicate: meta pass + survivors
        makes = [lambda: [_slot("Subject", "z")], lambda: [_slot("Subject", pat())], lambda: [_slot("subject", "é")],
                 lambda: [Cond(C_NAME, which=NAME_HOST, pattern=_rx("db"))],
                 lambda: [Cond(C_NAME, which=NAME_HOST, pattern=_rx(derived(rng, names[NAME_HOST])))],
                 lambda: [Cond(C_FOLDER_SET, set64=0b1011), _slot("x-note", pat())],
                 lambda: [Cond(C_NAME, which=NAME_DATE_STR, pattern=_rx(derived(rng, names[NAME_DATE_STR]))), _slot("Subject", pat(), 2)]]
    else:
        raise KeyError(name)
    queries = []
    for make in makes:
        for _ in range(200):
            q = make()
            col = _want(recs, heads, [q]) & 1
            if col.any() and not col.all():
                break
        else:
            raise AssertionError(f"{name}: no query of this shape both hits and misses")
        queries.append(q)
    dfa_texts = {"z", "é", "db"}
    automaton = [c.pattern.text for q in queries for c in q if c.pattern is not None and c.pattern.text not in dfa_texts]
    return queries, automaton


HEAD = ["slots", "sizes", "flags", "names", "mixed"]
_HEAD_PROGS = {}


def head_program(name, recs, heads, monkeypatch):
    if name not in _HEAD_PROGS:
        queries, automaton = _head_program(name, recs, heads)
        _HEAD_PROGS[name] = (queries, _build(queries, automaton, monkeypatch))
    return _HEAD_PROGS[name]


HEAD_WORDS = set()


@pytest.fixture(scope="module")
def head_loads(gpu):
    from fei_b200.corpus import Corpus
    recs, heads = head_records()
    out = {"default": Corpus().load(_arrays(recs))}
    for var in ("FEI_HDIR", "FEI_HCOLS"):
        with _env(**{var: "0"}):
            out[var] = Corpus().load(_arrays(recs))
    yield recs, heads, out
    for c in out.values():
        c.close()


@gpu
@pytest.mark.parametrize("name", HEAD)
def test_head_automata_agree_with_cpython(head_loads, name, monkeypatch):
    recs, heads, corpora = head_loads
    queries, prog = head_program(name, recs, heads, monkeypatch)
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA
    sections = _head_sections(prog)
    assert sections, name
    HEAD_WORDS.update(w for _f, w in sections)
    if name == "names":
        assert {f for f, _w in sections} >= {"head1", "head2", "head3", "head4", "head5"}       # all five name fields
    nq = len(queries)
    want = _want(recs, heads, queries)
    want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
    in_global = bytearray(prog)
    struct.pack_into("<I", in_global, 76, 0)                            # head_bytes = 0: the head kernels read global memory
    for load, c in corpora.items():
        for leg, p, env in (("smem", prog, {}), ("global", bytes(in_global), {}), ("unfused", prog, {"FEI_HEAD_FUSE": "0"})):
            with _env(**env):
                got = c.scan_masks(p)
                bad = np.nonzero(got != want)[0]
                assert bad.size == 0, (name, load, leg, int(bad[0]), recs[int(bad[0])]["hdr"], recs[int(bad[0])]["filename"],
                                       int(want[bad[0]]), int(got[bad[0]]))
                hits = c.scan_hits(p, nq)
                counts = c.scan_count(p, nq)
            for q in range(nq):
                assert np.array_equal(hits[q], want_lists[q]), (name, load, leg, q)
                assert int(counts[q]) == want_lists[q].size, (name, load, leg, q)


@gpu
def test_every_head_vector_width_was_taken():
    assert HEAD_WORDS == {1, 2, 4, 8}, HEAD_WORDS


# ---------------------------------------------------------------- CPU leg
def _texts(rng, exs, k):
    """Short texts of the alphabet of the examples with examples planted."""
    out = ["", "\n"]
    while len(out) < k:
        parts = [rng.choice(exs) if rng.random() < 0.5 else "".join(rng.choice(_FILL["any"] + ["a", "-", "\n", "K"]) for _ in range(rng.randint(0, 6)))
                 for _ in range(rng.randint(1, 4))]
        out.append("".join(parts))
    return out


def test_generated_programs_agree_on_cpu(monkeypatch):
    """The generator's examples match, the size targets are reached, and the CPU model of every content program agrees with
    re on texts built from the examples (the naturally routed cases aside: their DFA refusal alone takes seconds)."""
    rng = random.Random(99)
    for _ in range(200):
        p, e = example_regex(rng)
        assert re.search(p, e, re.IGNORECASE), (p, e)
        m = rng.randint(0, 5)
        g, exs = gap_regex(rng, m, m + rng.randint(0, 20))
        assert any(re.search(g, x, re.IGNORECASE) for x in exs), (g, exs)
    for name in CONTENT:
        nfa, dfa, exs, natural = content_case(name)
        if natural:
            continue
        queries, prog = content_program(name, False, monkeypatch)
        _check_content_program(name, prog)
        off_conds, k, bits = struct.unpack_from("<I", prog, 20)[0], 0, {}
        for q in queries:                                                # the content bit each pattern was given
            for c in q:
                bits[c.pattern.text] = prog[off_conds + 32 * k + 2]
                k += 1
        for t in _texts(random.Random(name), exs, 12):
            want = sum(1 << b for p, b in bits.items() if re.search(p, t, re.IGNORECASE))
            assert program_content_bits(prog, t.encode()) == want, (name, t)
