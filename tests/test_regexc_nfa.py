"""The content position automaton (CPU suite): fei_b200.regexc.compile_positions against CPython's re, the serialized
section (tests/blob_nfa_model.py, stepping the way k_body_nfa does) against re, and the routing of content patterns in
ProgramBuilder: a pattern set the DFA holds keeps its version-1 program byte for byte, patterns the DFA refuses go to the
position automaton with their content bits renumbered behind the DFA's."""
import random
import re
import struct

import pytest

from fei_b200 import program as P
from fei_b200.program import C_BODY, C_SLOT, VERSION, VERSION_NFA, Cond, ProgramBuilder, content_automaton, content_batch_program
from fei_b200.regexc import Pattern, PatternTooLarge, compile_patterns, compile_positions
from tests.blob_model import BlobDfa
from tests.blob_nfa_model import BlobNfa, program_content_bits
from tests.test_regexc_fuzz import rand_regex

PROXIMITY = [r"kubernetes.*docker", r"kubernetes.{0,20}docker", r"kubernetes.{0,60}docker", r"kubernetes.{0,200}docker",
             r"\bdocker\b.{0,40}\bkubernetes\b", r"(error|fail).{0,80}(disk|memory)", r"docker\W+(?:\w+\W+){0,5}kubernetes",
             r"\bpython\b.{0,60}\b(rust|django)\b"]
TEXT_ALPHABET = list("abkKsS \n.-_,/09xy") + ["K", "ſ", "İ", "Σ", "σ", "ς", "é", "日", "\U0001F409", "@", "`", "[", "{"]
WORDS = ["kubernetes", "docker", "Kubernetes", "DOCKER", "error", "fail", "disk", "memory", "python", "rust", "django", "KUBERNETEſ"]


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


def _texts(rng, k, words=WORDS):
    out = ["", "\n", "docker", "kubernetes docker", "kubernetes\ndocker\n", "python, then rust", "error on disk\n"]
    while len(out) < k:
        parts = []
        for _ in range(rng.randint(0, 6)):
            if rng.random() < 0.4:
                parts.append(rng.choice(words))
            else:
                parts.append("".join(rng.choice(TEXT_ALPHABET) for _ in range(rng.choice([0, 1, 3, 15, 40, 70]))))
        out.append(" ".join(parts) if rng.random() < 0.5 else "".join(parts))
    return out


def test_proximity_patterns_agree_with_re():
    rng = random.Random(3)
    texts = _texts(rng, 300)
    for p in PROXIMITY:
        a = compile_positions([_rx(p)])
        assert a.n_pos <= 256
        rx = re.compile(p, re.IGNORECASE)
        for t in texts:
            assert bool(a.run(t.encode()) & 1) == (rx.search(t) is not None), (p, t)


def test_proximity_patterns_sizes():
    """The unrolled gaps stay small as position vectors (the start bit included)."""
    sizes = {p: compile_positions([_rx(p)]).n_pos for p in PROXIMITY[2:6]}
    assert sizes == {PROXIMITY[2]: 78, PROXIMITY[3]: 218, PROXIMITY[4]: 58, PROXIMITY[5]: 101}
    assert compile_positions([_rx(PROXIMITY[3])]).n_words == 8
    with pytest.raises(PatternTooLarge):
        compile_positions([_rx(r"kubernetes.{0,300}docker")])


def test_random_gap_patterns_agree_with_re():
    rng = random.Random(20261017)
    checked = patterns = 0
    while patterns < 220:
        p = rand_regex(rng) + ".{0,%d}" % rng.randint(0, 12) + rand_regex(rng)
        if rng.random() < 0.3:
            p = "(?m)" + p
        try:
            rx = re.compile(p, re.IGNORECASE)
        except re.error:
            continue
        try:
            a = compile_positions([_rx(p)])
        except PatternTooLarge:
            continue
        patterns += 1
        for _ in range(25):
            t = "".join(rng.choice(TEXT_ALPHABET) for _ in range(rng.randint(0, 16)))
            assert bool(a.run(t.encode()) & 1) == (rx.search(t) is not None), (p, t)
            checked += 1
    assert checked >= 5000


def test_union_agrees_with_re():
    rng = random.Random(8)
    for _ in range(20):
        pats = []
        while len(pats) < 5:
            p = rand_regex(rng) + ".{0,%d}" % rng.randint(0, 6) + rand_regex(rng)
            try:
                re.compile(p, re.IGNORECASE); pats.append(p)
            except re.error:
                pass
        try:
            a = compile_positions([_rx(p) for p in pats])
        except PatternTooLarge:
            continue
        for _ in range(40):
            t = "".join(rng.choice(TEXT_ALPHABET) for _ in range(rng.randint(0, 16)))
            m = a.run(t.encode())
            for k, p in enumerate(pats):
                assert bool(m >> k & 1) == (re.search(p, t, re.IGNORECASE) is not None), (p, t, pats)


def test_string_operators_agree_with_str():
    a = compile_positions([Pattern("contains", "ab"), Pattern("startswith", "k"), Pattern("endswith", "s"), Pattern("equals", "İx"),
                           Pattern("has_tag", "aσb")])
    rng = random.Random(2)
    for _ in range(400):
        v = "".join(rng.choice(TEXT_ALPHABET + ["ab", ",", " aΣb "]) for _ in range(rng.randint(0, 8)))
        vl = v.lower()
        want = [("ab" in vl), vl.startswith("k"), vl.endswith("s"), vl == "İx".lower(), "aσb" in [x.strip() for x in vl.split(",")]]
        m = a.run(v.encode())
        assert [bool(m >> k & 1) for k in range(5)] == want, (v, m)


def test_empty_string_verdict_falls_back_to_the_position_automaton():
    for p, want in [(r"kubernetes.{0,60}docker", 0), (r"(?:x.{0,60}y)?", 1), (r"^.{0,60}$", 1)]:
        a = content_automaton(_rx(p))
        assert a.run(b"") == want, p


def _program(queries):
    pb = ProgramBuilder()
    for q in queries:
        pb.add_query(q)
    return pb.build()


def test_serialized_section_agrees_with_re():
    rng = random.Random(41)
    texts = _texts(rng, 200)
    for pats in (PROXIMITY[1:3], [PROXIMITY[3]], [PROXIMITY[4], PROXIMITY[6], PROXIMITY[7]], [PROXIMITY[5], r"a$", r"(?m)^k.{0,3}s$"]):
        a = compile_positions([_rx(p) for p in pats])
        blob = bytearray(b"\0" * 48)
        off = P.serialize_nfa(a, blob, 3)
        m = BlobNfa(bytes(blob), off)
        assert (m.W, m.first_bit, m.n_patterns) == (a.n_words, 3, len(pats))
        for t in texts:
            raw = t.encode()
            want = sum(1 << (3 + k) for k, p in enumerate(pats) if re.search(p, t, re.IGNORECASE))
            assert m.run(raw) == want, (pats, t)


BATCH32 = ["python", "docker|kubernetes", "neural networks", "react", "angular", "rust", "django", "flask", "terraform", "ansible",
           "microservices", "big data", "ci/cd", "git", "aws|azure|gcp", "spring boot", r"vue\.js", r"node\.js", "devops", "security",
           "blockchain", "testing", "databases", "algorithms", "cloud computing", "mobile development", "computer vision",
           "reinforcement learning", "ui/ux", "web development", "data structures", "machine learning"]


def _version_and_nfa(prog):
    return struct.unpack_from("<I", prog, 4)[0], struct.unpack_from("<I", prog, 88)[0]


def test_dfa_programs_keep_version_1():
    assert _version_and_nfa(content_batch_program([_rx(p) for p in BATCH32])) == (VERSION, 0)
    from fei_b200.memdir_tools import filter as F
    pb = ProgramBuilder()
    for f in F.create_default_filters().filters:
        pb.add_query(F._compile_filter_conditions(f.conditions))
    assert _version_and_nfa(pb.build()) == (VERSION, 0)
    assert _version_and_nfa(content_batch_program([_rx(PROXIMITY[1])])) == (VERSION, 0)     # 524 states: the DFA holds it


def test_mixed_program_routes_and_renumbers():
    """Query order: DFA-able, proximity, DFA-able, proximity (negated), a header condition with a proximity one.  The DFA takes
    content bits 0 and 1, the position automaton 2 and 3, and every C_BODY condition reads its pattern's new bit."""
    pats = [_rx("python"), _rx(PROXIMITY[2]), _rx("rust|django"), _rx(PROXIMITY[5])]
    tag = Cond(C_SLOT, pattern=Pattern("has_tag", "ta"), field="Tags")
    queries = [[Cond(C_BODY, pattern=pats[0])], [Cond(C_BODY, pattern=pats[1])], [Cond(C_BODY, pattern=pats[2])],
               [Cond(C_BODY, pattern=pats[3], negate=True)], [tag, Cond(C_BODY, pattern=pats[1])]]
    prog = _program(queries)
    version, off_nfa = _version_and_nfa(prog)
    assert version == VERSION_NFA and off_nfa
    dfa = BlobDfa.from_program(prog)
    nfa = BlobNfa.from_program(prog)
    assert dfa.n_patterns == 2 and dfa.n_cols < 256 and dfa.sticky == 0
    assert (nfa.first_bit, nfa.n_patterns) == (2, 2)
    off_conds = struct.unpack_from("<I", prog, 20)[0]
    n_conds = struct.unpack_from("<I", prog, 16)[0]
    body_bits = [struct.unpack_from("<4B", prog, off_conds + 32 * k) for k in range(n_conds)]
    assert [(b[2], b[3]) for b in body_bits if b[0] == C_BODY] == [(0, 0), (2, 0), (1, 0), (3, 1), (2, 0)]
    rng = random.Random(5)
    order = [pats[0], pats[2], pats[1], pats[3]]                     # content bit k reads this pattern
    for t in _texts(rng, 150):
        want = sum(1 << k for k, p in enumerate(order) if re.search(p.text, t, re.IGNORECASE))
        assert program_content_bits(prog, t.encode()) == want, t


def test_nfa_only_program():
    prog = content_batch_program([_rx(PROXIMITY[3])])
    assert _version_and_nfa(prog)[0] == VERSION_NFA
    assert struct.unpack_from("<I", prog, 40)[0] == 0                # no body DFA
    assert BlobNfa.from_program(prog).W == 8


def test_largest_patterns_move_until_the_union_fits(monkeypatch):
    """Each pattern fits the DFA alone but the union does not: the largest move to the position automaton."""
    monkeypatch.setattr(P, "BODY_SMEM_LIMIT", 40 * 1024)
    pats = [_rx("ab"), _rx(PROXIMITY[1]), _rx("cd"), _rx(r"docker.{0,12}kubernetes")]
    alone = [P._table_bytes(P.cached_dfa([p]), 0) for p in pats]
    assert max(alone) <= 40 * 1024
    dfa, nfa, a = P._route_body(pats)
    assert nfa and set(dfa) >= {0, 2} and a.n_patterns == len(nfa)
    sizes = {i: P.cached_dfa([pats[i]]).n_states for i in range(4)}
    assert min(sizes[i] for i in nfa) >= max(sizes[i] for i in dfa)


def test_refused_dfa_is_cached():
    p = _rx(r"kubernetes.{0,60}docker")
    with pytest.raises(PatternTooLarge):
        P.cached_dfa([p])
    key = ((("regex", p.text, int(p.flags)),), False)
    assert key in P._DFA_FAIL
    calls = []
    real = P.compile_patterns
    P.compile_patterns = lambda *a, **k: calls.append(a) or real(*a, **k)
    try:
        with pytest.raises(PatternTooLarge):
            P.cached_dfa([p])
    finally:
        P.compile_patterns = real
    assert calls == []


def test_non_regular_constructs_still_raise():
    for p in (r"(a)\1", r"(?=a)b", r"(?>a)"):
        with pytest.raises(NotImplementedError):
            compile_positions([_rx(p)])
    with pytest.raises(NotImplementedError):
        content_batch_program([_rx(r"(a).{0,60}\1")])
