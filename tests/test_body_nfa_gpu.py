"""k_body_nfa, the content position automaton kernel, against plain CPython re.search(p, body, re.I): masks, ordered hit
lists and counts for position vectors of 1, 2, 4 and 8 words, with and without a body DFA stepped alongside, negated and
header-gated conditions with header fusion on and off, and a pattern that matches the empty string; counter positions
(version-3 programs) alone, next to a body DFA and next to expanded gap positions; sharded scans; malformed sections and
counter sections refused before any launch; the public API (search_memories, a folder= regex, FilterManager) with proximity
queries and long gaps against the oracle.  Two corpora: one with the body shapes of the content-kernel fuzz (empty bodies,
ragged rows, multi-byte UTF-8, the bytes the tile permutation swaps) and short gaps, one with bodies up to about 12 KB and
planted gaps of k - 1, k and k + 1 code points (ASCII and two-byte UTF-8) for k up to 5000.  On a mismatch the message
carries the verdict of the CPU model of the serialized automata (tests/blob_nfa_model.py)."""
import contextlib
import io
import re
import struct

import numpy as np
import pytest

from fei_b200 import synth
from fei_b200.program import VERSION_CTR, VERSION_NFA, content_batch_program
from fei_b200.regexc import Pattern
from tests.blob_nfa_model import program_content_bits
from tests.test_content_kernels_fuzz_gpu import Reference, _body, _length, _load, _plant, _program, _queries, _with_tags

pytestmark = pytest.mark.gpu

NFA_KERNEL = 4                    # fei_scan_timing.body_kernel


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


# name -> (corpus, content patterns, program version, words per position vector, counters of the content automaton)
CASES = {
    "w1": ("short_gaps", [_rx(r"q.{0,20}z")], VERSION_NFA, 1, 0),
    "w2": ("short_gaps", [_rx(r"k.{0,40}d"), _rx(r"\bx.{0,8}\by")], VERSION_NFA, 2, 0),
    "w4": ("short_gaps", [_rx(r"kubernetes.{0,60}docker")], VERSION_NFA, 4, 0),
    "w8": ("short_gaps", [_rx(r"kubernetes.{0,200}docker")], VERSION_NFA, 8, 0),
    "mixed-w2": ("short_gaps", [_rx("python"), _rx(r"\bdocker\b.{0,40}\bkubernetes\b"), _rx("rust|django"), _rx("[@`]{2}")],
                 VERSION_NFA, 2, 0),
    "mixed-w8": ("short_gaps", [_rx("docker"), _rx(r"kubernetes.{0,60}docker"), _rx("ß|日"), _rx(r"(error|fail).{0,80}(disk|memory)$")],
                 VERSION_NFA, 8, 0),
    "empty-match": ("short_gaps", [_rx(r"(?:k.{0,20}d|\A)\Z"), _rx("python")], VERSION_NFA, 1, 0),
    "counters": ("long_gaps", [_rx(r"q.{0,300}z"), _rx(r"kubernetes.{0,1000}docker"), _rx(r"xyzzy[^\n]{0,5000}plugh")],
                 VERSION_CTR, 2, 3),
    "counters-dfa": ("long_gaps", [_rx("python"), _rx(r"kubernetes.{0,1000}docker"), _rx("rust|django"), _rx(r"xyzzy(?s:.){0,5000}plugh")],
                     VERSION_CTR, 1, 2),
    "counters-gaps": ("long_gaps", [_rx(r"q.{0,300}z"), _rx(r"k.{0,40}d"), _rx(r"kubernetes.{0,5000}docker"), _rx(r"\bpython\b.{0,60}\brust\b")],
                      VERSION_CTR, 8, 2),
}

_GAPS = [b"", b" ", b"x" * 19, b"x" * 20, b"y" * 21, b"-" * 39, b"-" * 40, b"z" * 60, b"z" * 61, "é".encode() * 30, b"\n" * 5, b"@`[{" * 50]
_ENDS = [(b"q", b"z"), (b"k", b"d"), (b"x", b"y"), (b"kubernetes", b"docker"), (b"KUBERNETES", b"Docker"), (b"docker", b"kubernetes"),
         (b"error", b"disk"), (b"fail", b"memory"), (b"python", b"rust"), (b"@", b"`")]
_LONG_ENDS = [(b"q", b"z"), (b"kubernetes", b"docker"), (b"KUBERNETES", b"Docker"), (b"xyzzy", b"plugh"), (b"k", b"d"),
              (b"python ", b" rust")]


def _short_token(rng):
    a, b = _ENDS[int(rng.integers(len(_ENDS)))]
    return a + _GAPS[int(rng.integers(len(_GAPS)))] + b


def _long_token(rng):
    a, b = _LONG_ENDS[int(rng.integers(len(_LONG_ENDS)))]
    k = int(rng.choice([40, 60, 300, 1000, 5000]))
    g = k + int(rng.integers(-1, 2))
    fill = "é" if rng.random() < 0.4 else "x" if rng.random() < 0.7 else "\n"
    return a + (fill * g).encode() + b


def _long_length(rng, i):
    return 0 if i % 50 == 0 else int(rng.integers(1, 40)) if i % 7 == 0 else int(rng.integers(40, 12000))


def _corpus(seed, salt, length, token, max_plants):
    """2 windows of 4096 records + 37, each body with up to max_plants - 1 tokens planted; tags ta / tb / none in turn."""
    rng = np.random.default_rng(seed)
    n = 2 * 4096 + 37
    recs, bodies, tags = [], [], []
    for i in range(n):
        total = length(rng, i)
        b = _body(rng, total, [_plant(rng, total, token(rng)) for _ in range(int(rng.integers(0, max_plants)))])
        t = ["ta"] if i % 3 == 0 else ["tb"] if i % 3 == 1 else []
        r = _with_tags(synth.record(salt, i), t)
        r["body"] = b
        recs.append(r); bodies.append(b); tags.append(t + ["misc"])
    return _load(recs), Reference(bodies, tags)


@pytest.fixture(scope="module")
def short_gaps(gpu):
    c, ref = _corpus(20261018, 41, _length, _short_token, 5)
    yield c, ref
    c.close()


@pytest.fixture(scope="module")
def long_gaps(gpu):
    c, ref = _corpus(20261019, 43, _long_length, _long_token, 4)
    yield c, ref
    c.close()


def _nfa_timing(c):
    tm = c.timing()
    return tm["body_kernel"], tm["body_nfa_words"], tm["body_nfa_counters"]


def _explain(prog, ref, queries, want, got):
    bad = np.nonzero(want != got)[0]
    r = int(bad[0])
    q = int(np.nonzero((want[r] ^ got[r]) >> np.arange(32, dtype=np.uint32) & 1)[0][0])
    return (f"{bad.size} records differ; record {r} (len {len(ref.bodies[r])}) query {q} "
            f"{[(c.pattern.kind, c.pattern.text, c.negate) for c in queries[q]]}: want {want[r] >> q & 1}, got {got[r] >> q & 1}; "
            f"CPU model of the serialized automata gives content bits {program_content_bits(prog, ref.bodies[r]):#x}")


@pytest.mark.parametrize("name", list(CASES))
def test_nfa_scans_agree_with_cpython(request, name, monkeypatch):
    corpus, pats, version, words, n_ctr = CASES[name]
    c, ref = request.getfixturevalue(corpus)
    for head in (False, True):
        queries = _queries(pats, head)
        prog = _program(queries)
        assert struct.unpack_from("<I", prog, 4)[0] == version, name
        nq = len(queries)
        want = ref.masks(queries)
        want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
        for env in ([{}, {"FEI_HEAD_FUSE": "0"}] if head else [{}]):
            with monkeypatch.context() as mp:
                for k, v in env.items():
                    mp.setenv(k, v)
                got = c.scan_masks(prog)
                assert _nfa_timing(c) == (NFA_KERNEL, words, n_ctr), (name, env, c.timing())
                assert np.array_equal(got, want), (name, env, _explain(prog, ref, queries, want, got))
                hits = c.scan_hits(prog, nq)
                assert _nfa_timing(c) == (NFA_KERNEL, words, n_ctr), (name, env, c.timing())
                counts = c.scan_count(prog, nq)
            for q in range(nq):
                assert np.array_equal(hits[q], want_lists[q]), (name, env, q)
                assert int(counts[q]) == want_lists[q].size, (name, env, q)
        assert want.any() and (want != want[0]).any(), name          # the case is not vacuous
    for p in pats:                                                   # every pattern matches somewhere and misses somewhere
        v = np.array([re.search(p.text, t, re.I) is not None for t in ref.texts])
        assert v.any() and not v.all(), (name, p.text)


def test_plain_programs_report_no_counters(long_gaps):
    c, _ref = long_gaps
    prog = content_batch_program([_rx(r"kubernetes.{0,238}docker")])
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA
    c.scan_masks(prog)
    assert _nfa_timing(c) == (NFA_KERNEL, 8, 0)


@pytest.mark.parametrize("pats, version, words, n_ctr", [
    pytest.param(["python", r"\bpython\b.{0,60}\b(rust|django)\b", r"kubernetes.{0,60}docker"], VERSION_NFA, 8, 0, id="plain"),
    pytest.param(["python", r"\bpython\b.{0,1000}\b(rust|django)\b", r"kubernetes.{0,5000}docker"], VERSION_CTR, 2, 2, id="counters")])
def test_sharded_nfa_scan_equals_unsharded(gpu, pats, version, words, n_ctr):
    from fei_b200 import shard
    from fei_b200.corpus import Corpus
    n = 4100
    prog = content_batch_program([_rx(p) for p in pats])
    assert struct.unpack_from("<I", prog, 4)[0] == version
    whole_c = Corpus().synth(0xFE1, 0, n)
    whole = whole_c.scan_hits(prog, len(pats))
    assert _nfa_timing(whole_c) == (NFA_KERNEL, words, n_ctr)
    for world in (2, 4):
        per_rank = [Corpus().synth(0xFE1, a, b - a).scan_hits(prog, len(pats)) for a, b in shard.shard_ranges(n, world)]
        got = shard.concat_in_rank_order(per_rank)
        for q in range(len(pats)):
            assert np.array_equal(got[q], whole[q]), (world, q)


def _patched(blob, at, fmt, *v):
    b = bytearray(blob)
    struct.pack_into(fmt, b, at, *v)
    return bytes(b)


def _broken_sections(plain, counted):
    off = struct.unpack_from("<I", plain, 88)[0]
    off_ascii = struct.unpack_from("<I", plain, off + 32)[0]
    truncated = bytearray(plain[:off + 32])                  # the section's descriptor is cut in half
    struct.pack_into("<I", truncated, 8, len(truncated))
    return [bytes(truncated),
            _patched(plain, off, "<I", 3),                   # W must be 1, 2, 4 or 8
            _patched(plain, off_ascii + 2 * ord("k"), "<H", 200)]    # class id beyond n_classes


def _broken_counters(plain, counted):
    off = struct.unpack_from("<I", counted, 88)[0]
    n_pos = struct.unpack_from("<I", counted, off + 4)[0]
    off_ctr = struct.unpack_from("<I", counted, off + 68)[0]
    return [_patched(counted, 4, "<I", 1),                   # a position automaton in a version-1 program
            _patched(plain, 4, "<I", VERSION_CTR),           # version 3 without a counter descriptor
            _patched(counted, off + 64, "<I", 0),            # no counters
            _patched(counted, off + 64, "<I", 9),            # more than 8
            _patched(counted, off + 68, "<I", off_ctr + 8),  # table not 16-byte aligned
            _patched(counted, off + 68, "<I", off),          # table outside the section's tables
            _patched(counted, off_ctr, "<I", 0),             # the start bit
            _patched(counted, off_ctr, "<I", n_pos),         # past n_pos
            _patched(counted, off_ctr + 4, "<I", 0)]         # bound 0


@pytest.mark.parametrize("broken", [_broken_sections, _broken_counters], ids=["plain", "counters"])
def test_malformed_nfa_section_is_refused(gpu, broken):
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    plain = content_batch_program([_rx(r"kubernetes.{0,60}docker")])
    counted = content_batch_program([_rx(r"kubernetes.{0,1000}docker")])
    c = Corpus().synth(0xFE1, 0, 1000)
    for blob in broken(plain, counted):
        with pytest.raises(_abi.FeiError) as e:
            c.scan_masks(blob)
        assert e.value.code == _abi.FEI_E_BADARG
    for prog, words, n_ctr in ((plain, 4, 0), (counted, 1, 1)):     # the well-formed programs still scan
        c.scan_masks(prog)
        assert _nfa_timing(c) == (NFA_KERNEL, words, n_ctr)
    c.close()


# tree -> (long-gap memories added to the test tree, search strings, filters: (name, content pattern, negate, action, arguments))
API_CASES = {
    "proximity": ([], ["content:/kubernetes.{0,60}docker/ with_content", "content:/kubernetes.{0,60}docker/",
                       r"content:/\bpython\b.{0,60}\b(rust|django)\b/ with_content", "content:/(?:k.{0,20}d|\\A)\\Z/"],
                  [("Proximity", r"python.{0,60}(rust|django)", False, "move", {"target_folder": ".Projects/Python", "target_status": "cur"}),
                   ("Far", r"kubernetes.{0,60}docker", True, "flag", {"flags": "F"})]),
    "long-gaps": ([10, 999, 1000, 1001, 4000],
                  ["content:/kubernetes.{0,1000}docker/ with_content", "content:/kubernetes.{0,1000}docker/", "folder=/p.{0,1000}ai/",
                   "content:/(?:k.{0,1000}d|\\A)\\Z/"],
                  [("Near", r"kubernetes.{0,1000}docker", False, "flag", {"flags": "F"}),
                   ("Far", r"kubernetes.{0,500}docker", True, "flag", {"flags": "S"})]),
}


@pytest.fixture(scope="module", params=list(API_CASES))
def api(gpu, tmp_path_factory, request):
    from tests.memdir_util import build_tree
    from fei_b200.memdir_tools import utils as U
    base = str(tmp_path_factory.mktemp(f"memdir_{request.param}") / "Memdir")
    build_tree(base)
    U.set_memdir_base(base)
    for k, gap in enumerate(API_CASES[request.param][0]):
        U.save_memory(".Projects/AI" if k % 2 else "", "kubernetes" + "é" * gap + "docker\n", {"Subject": f"gap {gap}", "Tags": "ops"})
    return base, request.param


def test_search_and_filters_match_oracle(api):
    from fei_b200.memdir_tools import filter as F
    from fei_b200.memdir_tools.search import parse_search_args, search_memories
    from oracle import memdir_oracle as mo
    from tests.memdir_util import key_of
    base, name = api
    _gaps, searches, filters = API_CASES[name]
    for text in searches:
        q = parse_search_args(text)
        with contextlib.redirect_stdout(io.StringIO()):
            res = search_memories(q)
            mems = mo.listing(base, None, None, q.include_content)
        want = [mems[i] for i in mo.run_search(mems, q.conditions)]
        assert [key_of(m) for m in res] == [key_of(m) for m in want], text
        if text.endswith("with_content"):
            assert want and len(want) < len(mems), text
    mgr = F.FilterManager()
    for fname, pattern, negate, action, args in filters:
        mgr.add_filter(F.MemoryFilter(fname).add_condition("content", pattern, negate=negate).add_action(action, **args))
    for statuses in (["new"], ["cur", "new"]):
        with contextlib.redirect_stdout(io.StringIO()):
            stats = mgr.process_memories(statuses=statuses, dry_run=True)
            mems = [m for s in statuses for m in mo.listing(base, None, [s], True)]
        want = mo.run_filters(mems, [{"name": f.name, "conditions": f.conditions, "actions": f.actions} for f in mgr.filters])
        for k in ("total_memories", "filters_applied", "actions_taken", "memories_modified"):
            assert stats[k] == want[k], (statuses, k, stats[k], want[k])
        assert sorted(d["memory_id"] for d in stats["details"]) == sorted(d["memory_id"] for d in want["details"])
