"""k_body_nfa with counter positions (version-3 programs) against plain CPython re.search(p, body, re.I): masks, ordered hit
lists and counts on bodies up to about 12 KB with planted gaps of k - 1, k and k + 1 code points (ASCII and two-byte UTF-8) for
k = 300, 1000 and 5000 -- counters alone, next to a body DFA, next to expanded gap positions, with negated and header-gated
queries and header fusion on and off; a sharded scan; malformed counter sections refused before any launch; the public API
(search_memories, a folder= regex, FilterManager) with long gaps against the oracle.  On a mismatch the message carries the
verdict of the CPU model of the serialized automata (tests/blob_nfa_ctr_model.py)."""
import contextlib
import io
import re
import struct

import numpy as np
import pytest

from fei_b200 import synth
from fei_b200.program import VERSION_CTR, VERSION_NFA, content_batch_program
from fei_b200.regexc import Pattern
from tests.blob_nfa_ctr_model import program_content_bits
from tests.test_content_kernels_fuzz_gpu import Reference, _body, _load, _plant, _program, _queries, _with_tags

pytestmark = pytest.mark.gpu

NFA_KERNEL = 4                    # fei_scan_timing.body_kernel


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


# name -> (content patterns, counters of the content automaton)
CASES = {
    "counters": ([_rx(r"q.{0,300}z"), _rx(r"kubernetes.{0,1000}docker"), _rx(r"xyzzy[^\n]{0,5000}plugh")], 3),
    "counters-dfa": ([_rx("python"), _rx(r"kubernetes.{0,1000}docker"), _rx("rust|django"), _rx(r"xyzzy(?s:.){0,5000}plugh")], 2),
    "counters-gaps": ([_rx(r"q.{0,300}z"), _rx(r"k.{0,40}d"), _rx(r"kubernetes.{0,5000}docker"), _rx(r"\bpython\b.{0,60}\brust\b")], 2),
}
_ENDS = [(b"q", b"z"), (b"kubernetes", b"docker"), (b"KUBERNETES", b"Docker"), (b"xyzzy", b"plugh"), (b"k", b"d"),
         (b"python ", b" rust")]


def _token(rng):
    a, b = _ENDS[int(rng.integers(len(_ENDS)))]
    k = int(rng.choice([40, 60, 300, 1000, 5000]))
    g = k + int(rng.integers(-1, 2))
    fill = "é" if rng.random() < 0.4 else "x" if rng.random() < 0.7 else "\n"
    return a + (fill * g).encode() + b


@pytest.fixture(scope="module")
def corpus(gpu):
    rng = np.random.default_rng(20261019)
    n = 2 * 4096 + 37
    recs, bodies, tags = [], [], []
    for i in range(n):
        total = 0 if i % 50 == 0 else int(rng.integers(1, 40)) if i % 7 == 0 else int(rng.integers(40, 12000))
        b = _body(rng, total, [_plant(rng, total, _token(rng)) for _ in range(int(rng.integers(0, 4)))])
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
            f"{[(c.pattern.kind, c.pattern.text, c.negate) for c in queries[q]]}: want {want[r] >> q & 1}, got {got[r] >> q & 1}; "
            f"CPU model of the serialized automata gives content bits {program_content_bits(prog, ref.bodies[r]):#x}")


@pytest.mark.parametrize("name", list(CASES))
def test_counted_scans_agree_with_cpython(corpus, name, monkeypatch):
    c, ref = corpus
    pats, n_ctr = CASES[name]
    for head in (False, True):
        queries = _queries(pats, head)
        prog = _program(queries)
        assert struct.unpack_from("<I", prog, 4)[0] == VERSION_CTR, name
        nq = len(queries)
        want = ref.masks(queries)
        want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
        for env in ([{}, {"FEI_HEAD_FUSE": "0"}] if head else [{}]):
            with monkeypatch.context() as mp:
                for k, v in env.items():
                    mp.setenv(k, v)
                got = c.scan_masks(prog)
                tm = c.timing()
                assert (tm["body_kernel"], tm["body_nfa_counters"]) == (NFA_KERNEL, n_ctr), (name, env, tm)
                assert np.array_equal(got, want), (name, env, _explain(prog, ref, queries, want, got))
                hits = c.scan_hits(prog, nq)
                assert c.timing()["body_nfa_counters"] == n_ctr
                counts = c.scan_count(prog, nq)
            for q in range(nq):
                assert np.array_equal(hits[q], want_lists[q]), (name, env, q)
                assert int(counts[q]) == want_lists[q].size, (name, env, q)
        assert want.any() and (want != want[0]).any(), name          # the case is not vacuous
        for p in pats:                                               # every pattern matches somewhere and misses somewhere
            v = np.array([re.search(p.text, t, re.I) is not None for t in ref.texts])
            assert v.any() and not v.all(), (name, p.text)


def test_plain_programs_report_no_counters(corpus):
    c, _ref = corpus
    prog = content_batch_program([_rx(r"kubernetes.{0,238}docker")])
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA
    c.scan_masks(prog)
    tm = c.timing()
    assert (tm["body_kernel"], tm["body_nfa_words"], tm["body_nfa_counters"]) == (NFA_KERNEL, 8, 0)


def test_sharded_counted_scan_equals_unsharded(gpu):
    from fei_b200 import shard
    from fei_b200.corpus import Corpus
    n = 4100
    pats = ["python", r"\bpython\b.{0,1000}\b(rust|django)\b", r"kubernetes.{0,5000}docker"]
    prog = content_batch_program([_rx(p) for p in pats])
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_CTR
    whole_c = Corpus().synth(0xFE1, 0, n)
    whole = whole_c.scan_hits(prog, len(pats))
    assert whole_c.timing()["body_nfa_counters"] == 2
    for world in (2, 4):
        per_rank = [Corpus().synth(0xFE1, a, b - a).scan_hits(prog, len(pats)) for a, b in shard.shard_ranges(n, world)]
        got = shard.concat_in_rank_order(per_rank)
        for q in range(len(pats)):
            assert np.array_equal(got[q], whole[q]), (world, q)


def test_malformed_counter_sections_are_refused(gpu):
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    prog = content_batch_program([_rx(r"kubernetes.{0,1000}docker")])
    plain = content_batch_program([_rx(r"kubernetes.{0,60}docker")])
    off = struct.unpack_from("<I", prog, 88)[0]
    n_pos = struct.unpack_from("<I", prog, off + 4)[0]
    off_ctr = struct.unpack_from("<I", prog, off + 68)[0]
    c = Corpus().synth(0xFE1, 0, 1000)

    def patched(blob, at, fmt, *v):
        b = bytearray(blob)
        struct.pack_into(fmt, b, at, *v)
        return bytes(b)

    bad = [patched(prog, 4, "<I", 1),                            # a position automaton in a version-1 program
           patched(plain, 4, "<I", VERSION_CTR),                 # version 3 without a counter descriptor
           patched(prog, off + 64, "<I", 0),                     # no counters
           patched(prog, off + 64, "<I", 9),                     # more than 8
           patched(prog, off + 68, "<I", off_ctr + 8),           # table not 16-byte aligned
           patched(prog, off + 68, "<I", off),                   # table outside the section's tables
           patched(prog, off_ctr, "<I", 0),                      # the start bit
           patched(prog, off_ctr, "<I", n_pos),                  # past n_pos
           patched(prog, off_ctr + 4, "<I", 0)]                  # bound 0
    for blob in bad:
        with pytest.raises(_abi.FeiError) as e:
            c.scan_masks(blob)
        assert e.value.code == _abi.FEI_E_BADARG
    c.scan_masks(prog)                                       # the well-formed program still scans
    assert c.timing()["body_nfa_counters"] == 1
    c.close()


@pytest.fixture(scope="module")
def api(gpu, tmp_path_factory):
    from tests.memdir_util import build_tree
    from fei_b200.memdir_tools import utils as U
    base = str(tmp_path_factory.mktemp("memdir_ctr") / "Memdir")
    build_tree(base)
    U.set_memdir_base(base)
    for k, gap in enumerate([10, 999, 1000, 1001, 4000]):
        U.save_memory(".Projects/AI" if k % 2 else "", "kubernetes" + "é" * gap + "docker\n", {"Subject": f"gap {gap}", "Tags": "ops"})
    return base


def test_long_gap_search_and_filters_match_oracle(api):
    from fei_b200.memdir_tools import filter as F
    from fei_b200.memdir_tools.search import parse_search_args, search_memories
    from oracle import memdir_oracle as mo
    from tests.memdir_util import key_of
    base = api
    for text in ("content:/kubernetes.{0,1000}docker/ with_content", "content:/kubernetes.{0,1000}docker/",
                 "folder=/p.{0,1000}ai/", "content:/(?:k.{0,1000}d|\\A)\\Z/"):
        q = parse_search_args(text)
        with contextlib.redirect_stdout(io.StringIO()):
            res = search_memories(q)
            mems = mo.listing(base, None, None, q.include_content)
        want = [mems[i] for i in mo.run_search(mems, q.conditions)]
        assert [key_of(m) for m in res] == [key_of(m) for m in want], text
        if text.endswith("with_content"):
            assert want and len(want) < len(mems), text
    flt = F.MemoryFilter("Near").add_condition("content", r"kubernetes.{0,1000}docker").add_action("flag", flags="F")
    neg = F.MemoryFilter("Far").add_condition("content", r"kubernetes.{0,500}docker", negate=True).add_action("flag", flags="S")
    mgr = F.FilterManager()
    mgr.add_filter(flt); mgr.add_filter(neg)
    for statuses in (["new"], ["cur", "new"]):
        with contextlib.redirect_stdout(io.StringIO()):
            stats = mgr.process_memories(statuses=statuses, dry_run=True)
            mems = [m for s in statuses for m in mo.listing(base, None, [s], True)]
        want = mo.run_filters(mems, [{"name": f.name, "conditions": f.conditions, "actions": f.actions} for f in mgr.filters])
        for k in ("total_memories", "filters_applied", "actions_taken", "memories_modified"):
            assert stats[k] == want[k], (statuses, k, stats[k], want[k])
        assert sorted(d["memory_id"] for d in stats["details"]) == sorted(d["memory_id"] for d in want["details"])
