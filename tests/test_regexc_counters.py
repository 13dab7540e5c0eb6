"""Position automata with counters (CPU suite): fei_b200.regexc.compile_positions_counted against CPython's
re.search(p, s, re.I) on fixed cases and a seeded fuzz (bounds from 239 to 100000, the usual gap classes, lower bounds, lazy
repeats, anchors next to the gap, nested and several patterns), the serialized counter section (tests/blob_nfa_model.py)
against Pna.run, the refusals, and the routing: only content patterns the plain automaton refuses get counters and a version-3
program; head fields keep their limits."""
import random
import re
import struct

import pytest

from fei_b200.program import (C_BODY, C_SLOT, VERSION_CTR, VERSION_NFA, Cond, ProgramBuilder, _route_body, content_automaton,
                              content_batch_program)
from fei_b200.regexc import PNA_MAX_COUNTERS, Pattern, PatternTooLarge, compile_positions, compile_positions_counted
from tests.blob_nfa_model import BlobNfa, program_content_bits

BOUNDS = [239, 300, 1000, 5000, 100000]
CLASSES = [".", "(?s:.)", r"[\s\S]", r"[^\n]", r"\W", "[^x]", r"\w"]
FILL = {".": "a-é日", "(?s:.)": "a\né日", r"[\s\S]": " \né日", r"[^\n]": "ab é日", r"\W": " -.,\n", "[^x]": "ab\né日", r"\w": "abé日_9"}


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


def _agree(p, texts, a=None):
    a = a or compile_positions_counted([_rx(p)])
    rx = re.compile(p, re.IGNORECASE)
    for t in texts:
        assert bool(a.run(t.encode()) & 1) == (rx.search(t) is not None), (p, len(t), t[:40], t[-40:])
    return a


def _gaps(k, fill, left="q", right="z"):
    """Texts with gaps of k - 1, k and k + 1 code points of `fill` (cycled) between `left` and `right`, and a run broken once."""
    out = []
    for g in (k - 1, k, k + 1):
        gap = (fill * (g // len(fill) + 1))[:g]
        out += [left + gap + right, "x" + left + gap + right + "x", left + gap[: g // 2] + "x" + gap[g // 2 + 1:] + right]
    return out


@pytest.mark.parametrize("k", BOUNDS)
def test_long_gaps_agree_with_re(k):
    for cls in CLASSES if k <= 5000 else [".", r"[^\n]"]:
        p = f"q{cls}{{0,{k}}}z"
        a = _agree(p, _gaps(k, FILL[cls]) + ["", "qz", "q\nz", "z q", "Q" + FILL[cls][:3] + "Z"])
        assert [b for _p, b in a.counters] == [k] and a.n_words == 1, p


def test_utf8_gaps_count_code_points():
    """A gap of 300 three-byte characters is 900 bytes and still inside `.{0,300}`; 301 of them is not."""
    a = _agree("q.{0,300}z", ["q" + "日" * 300 + "z", "q" + "日" * 301 + "z", "q" + "\U0001F409" * 300 + "z", "q" + "é" * 299 + "z"])
    assert a.run(("q" + "日" * 300 + "z").encode()) == 1 and a.run(("q" + "日" * 301 + "z").encode()) == 0


def test_shapes_next_to_the_gap_agree_with_re():
    cases = {
        r"q.{3,900}z": _gaps(900, "ab") + ["qabz", "qabcz", "qaz"],
        r"q.{0,1000}?z": _gaps(1000, "ab"),
        r"q.{0,300}$": ["q" + "a" * 300, "q" + "a" * 301, "q" + "a" * 300 + "\n", "q" + "a" * 301 + "\n", "q" + "a" * 10 + "\nb"],
        r"q.{0,300}\Z": ["q" + "a" * 300, "q" + "a" * 300 + "\n", "q" + "a" * 301],
        r"(?m)q.{0,300}$": ["q" + "a" * 300 + "\nb", "q" + "a" * 301 + "\nb", "q" + "a" * 300],
        r"\bq.{0,300}\bz": ["q" + " " * 299 + "z", "q" + "a" * 299 + "z", "aq" + " " * 200 + "z", "q" + " " * 300 + "z"],
        r"(?:a.{0,300}b){2}": ["a" + "x" * 300 + "ba" + "y" * 300 + "b", "a" + "x" * 301 + "ba" + "y" * 300 + "b", "ab" * 2,
                               "a" + "x" * 300 + "b" + "a" + "y" * 301 + "b"],
        r"(?:x[^\n]{0,500})+y": ["x" + "a" * 500 + "x" + "a" * 500 + "y", "x" + "a" * 501 + "y", "x" + "a" * 400 + "\ny"],
        r"q.{0,60}w.{0,400}z": ["q" + "a" * 60 + "w" + "b" * 400 + "z", "q" + "a" * 61 + "w" + "b" * 400 + "z",
                                "q" + "a" * 60 + "w" + "b" * 401 + "z"],
    }
    for p, texts in cases.items():
        _agree(p, texts)


def test_fuzz_agrees_with_re():
    rng = random.Random(20261018)
    alphabet = ["a", "b", "q", "z", " ", "\n", "-", "é", "日", "\U0001F409", "x", "_"]
    for trial in range(60):
        k = rng.choice([239, 240, 300, 777, 1000, 2500])
        cls = rng.choice(CLASSES)
        lo = rng.choice([0, 0, 1, 3])
        lazy = "?" if rng.random() < 0.3 else ""
        tail = rng.choice(["z", "z$", r"z\Z", r"\bz", "(?:z|b)"])
        head = rng.choice(["q", "qa", r"\bq", "^q", "(?m)^q"])
        p = f"{head}{cls}{{{lo},{k}}}{lazy}{tail}"
        a = compile_positions_counted([_rx(p)])
        texts = []
        for _ in range(12):
            g = rng.choice([k - 1, k, k + 1, lo - 1, lo, rng.randrange(k + 2)])
            gap = "".join(rng.choice(FILL[cls]) for _ in range(max(g, 0)))
            if rng.random() < 0.2 and gap:
                j = rng.randrange(len(gap))
                gap = gap[:j] + rng.choice(alphabet) + gap[j + 1:]
            pre = "".join(rng.choice(alphabet) for _ in range(rng.randrange(4)))
            post = "".join(rng.choice(alphabet) for _ in range(rng.randrange(4)))
            texts.append(pre + rng.choice(["q", "Q", "qa"]) + gap + rng.choice(["z", "Z", "b", "z\n", "zz"]) + post)
        _agree(p, texts, a)


def test_several_patterns_in_one_automaton():
    pats = [r"kubernetes.{0,1000}docker", r"python[^\n]{0,500}rust", r"error.{0,20}disk", "plain"]
    a = compile_positions_counted([_rx(p) for p in pats])
    assert len(a.counters) == 2                                    # the small gap stays expanded
    texts = ["kubernetes" + "x" * 1000 + "docker", "kubernetes" + "x" * 1001 + "docker python" + "y" * 500 + "rust",
             "python" + "y" * 200 + "\nrust", "error" + "." * 20 + "disk plain", "error" + "." * 21 + "disk"]
    for t in texts:
        want = sum(1 << i for i, p in enumerate(pats) if re.search(p, t, re.IGNORECASE))
        assert a.run(t.encode()) == want, t[:30]


def test_largest_repeats_are_counted_first_and_only_as_needed():
    a = compile_positions_counted([_rx(r"a.{0,200}b.{0,100}c")])          # 302 positions expanded: one counter is enough
    assert [k for _p, k in a.counters] == [200]
    a = compile_positions_counted([_rx(r"a.{0,200}b.{0,150}c")])
    assert sorted(k for _p, k in a.counters) == [200]
    a = compile_positions_counted([_rx(r"a.{0,260}b.{0,260}c")])
    assert sorted(k for _p, k in a.counters) == [260, 260]


def test_serialized_counters_agree_with_the_automaton():
    rng = random.Random(7)
    for pats in ([r"kubernetes.{0,1000}docker"], [r"q\W{0,300}z", "plain"], [r"docker", r"(?:a.{0,300}b){2}", r"q.{0,60}z"]):
        prog = content_batch_program([_rx(p) for p in pats])
        assert struct.unpack_from("<I", prog, 4)[0] == VERSION_CTR
        m = BlobNfa.from_program(prog)
        assert m.counters
        dfa, nfa, _a = _route_body([_rx(p) for p in pats])
        bit = {i: b for b, i in enumerate(dfa + nfa)}                           # content bits: the DFA's first
        texts = ["kubernetes" + "日" * 1000 + "docker", "a" + "-" * 300 + "ba" + "b" * 299 + "b", "q" + " " * 300 + "z", "q" + "-" * 301 + "z"]
        texts += ["".join(rng.choice("abqz -日\n") for _ in range(rng.randrange(700))) for _ in range(20)]
        for t in texts:
            want = sum(1 << bit[i] for i, p in enumerate(pats) if re.search(p, t, re.IGNORECASE))
            assert program_content_bits(prog, t.encode()) == want, (pats, t[:30])


def test_refusals():
    with pytest.raises(PatternTooLarge):
        compile_positions_counted([_rx(f"a{i}.{{0,300}}b") for i in range(PNA_MAX_COUNTERS + 1)])       # 9 counters
    compile_positions_counted([_rx(f"a{i}.{{0,300}}b") for i in range(PNA_MAX_COUNTERS)])
    for p in (r"a.{300,}b", r"a.{400,900}b", r"(?:ab){0,500}c", r"a.{1001,2000}b"):
        with pytest.raises(PatternTooLarge):
            compile_positions_counted([_rx(p)])
    with pytest.raises(NotImplementedError):
        compile_positions_counted([_rx(r"(a).{0,300}\1")])
    with pytest.raises(NotImplementedError):
        content_batch_program([_rx(r"(a).{0,300}\1")])
    pb = ProgramBuilder()                                           # head fields keep the plain automaton and its limits
    pb.add_query([Cond(C_SLOT, pattern=_rx(r"a.{0,300}b"), field="Subject")])
    with pytest.raises(PatternTooLarge):
        pb.build()


def test_programs_that_fit_keep_their_automaton():
    """`.{0,238}` still fits 256 positions: no counters, version 2, the plain automaton's bytes; one more needs a counter."""
    fit = content_batch_program([_rx(r"kubernetes.{0,238}docker")])
    assert struct.unpack_from("<I", fit, 4)[0] == VERSION_NFA
    off = struct.unpack_from("<I", fit, 88)[0]
    assert struct.unpack_from("<I", fit, off)[0] == 8
    assert compile_positions([_rx(r"kubernetes.{0,238}docker")]).n_pos == 256
    with pytest.raises(PatternTooLarge):
        compile_positions([_rx(r"kubernetes.{0,239}docker")])
    big = content_batch_program([_rx(r"kubernetes.{0,239}docker")])
    assert struct.unpack_from("<I", big, 4)[0] == VERSION_CTR
    off = struct.unpack_from("<I", big, 88)[0]
    assert struct.unpack_from("<3I", big, off)[:2] == (1, 19)                   # one word, 19 positions
    assert struct.unpack_from("<I", big, off + 64)[0] == 1                      # one counter


def test_counted_content_next_to_a_dfa_and_head_conditions():
    pb = ProgramBuilder()
    pb.add_query([Cond(C_BODY, pattern=_rx("python"))])
    pb.add_query([Cond(C_BODY, pattern=_rx(r"kubernetes.{0,5000}docker"), negate=True), Cond(C_SLOT, pattern=Pattern("has_tag", "ops"), field="Tags")])
    prog = pb.build()
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_CTR and struct.unpack_from("<I", prog, 40)[0]
    for t in ("python", "kubernetes" + "x" * 5000 + "docker", "kubernetes" + "x" * 5001 + "docker python"):
        want = int(bool(re.search("python", t, re.I))) | int(bool(re.search(r"kubernetes.{0,5000}docker", t, re.I))) << 1
        assert program_content_bits(prog, t.encode()) == want


def test_host_verdicts_use_the_counted_automaton():
    a = content_automaton(_rx(r"p.{0,1000}ai"))
    assert a.counters and a.run(b"projects/ai") == 1 and a.run(b"p" + b"x" * 1001 + b"ai") == 0
    assert content_automaton(_rx(r"(?:k.{0,1000}d|\A)\Z")).run(b"") == 1
