"""k_body_nfa, the content position automaton kernel, against plain CPython re.search(p, body, re.I): masks, ordered hit
lists and counts for position vectors of 1, 2, 4 and 8 words, with and without a body DFA stepped alongside, negated and
header-gated conditions, and a pattern that matches the empty string; the public API (search_memories, process_memories)
with a proximity query against the oracle; sharded scans; a malformed section refused before any launch.  The corpus
has the body shapes of the content-kernel fuzz (empty bodies, ragged rows, multi-byte UTF-8, the bytes the tile
permutation swaps).  On a mismatch the message carries the verdict of the CPU model of the serialized automata
(tests/blob_nfa_model.py)."""
import contextlib
import io
import re
import struct

import numpy as np
import pytest

from fei_b200.program import VERSION_NFA, content_batch_program
from fei_b200.regexc import Pattern
from tests.blob_nfa_model import program_content_bits
from tests.test_content_kernels_fuzz_gpu import Reference, _body, _length, _load, _plant, _program, _queries, _with_tags
from fei_b200 import synth

pytestmark = pytest.mark.gpu

NFA_KERNEL = 4                    # fei_scan_timing.body_kernel


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


# name -> (content patterns, words per position vector)
CASES = {
    "w1": ([_rx(r"q.{0,20}z")], 1),
    "w2": ([_rx(r"k.{0,40}d"), _rx(r"\bx.{0,8}\by")], 2),
    "w4": ([_rx(r"kubernetes.{0,60}docker")], 4),
    "w8": ([_rx(r"kubernetes.{0,200}docker")], 8),
    "mixed-w2": ([_rx("python"), _rx(r"\bdocker\b.{0,40}\bkubernetes\b"), _rx("rust|django"), _rx("[@`]{2}")], 2),
    "mixed-w8": ([_rx("docker"), _rx(r"kubernetes.{0,60}docker"), _rx("ß|日"), _rx(r"(error|fail).{0,80}(disk|memory)$")], 8),
    "empty-match": ([_rx(r"(?:k.{0,20}d|\A)\Z"), _rx("python")], 1),
}

_GAPS = [b"", b" ", b"x" * 19, b"x" * 20, b"y" * 21, b"-" * 39, b"-" * 40, b"z" * 60, b"z" * 61, "é".encode() * 30, b"\n" * 5, b"@`[{" * 50]
_ENDS = [(b"q", b"z"), (b"k", b"d"), (b"x", b"y"), (b"kubernetes", b"docker"), (b"KUBERNETES", b"Docker"), (b"docker", b"kubernetes"),
         (b"error", b"disk"), (b"fail", b"memory"), (b"python", b"rust"), (b"@", b"`")]


def _token(rng):
    a, b = _ENDS[int(rng.integers(len(_ENDS)))]
    return a + _GAPS[int(rng.integers(len(_GAPS)))] + b


@pytest.fixture(scope="module")
def corpus(gpu):
    rng = np.random.default_rng(20261018)
    n = 2 * 4096 + 37
    recs, bodies, tags = [], [], []
    for i in range(n):
        total = _length(rng, i)
        b = _body(rng, total, [_plant(rng, total, _token(rng)) for _ in range(int(rng.integers(0, 5)))])
        t = ["ta"] if i % 3 == 0 else ["tb"] if i % 3 == 1 else []
        r = _with_tags(synth.record(41, i), t)
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
def test_nfa_scans_agree_with_cpython(corpus, name, monkeypatch):
    c, ref = corpus
    pats, words = CASES[name]
    for head in (False, True):
        queries = _queries(pats, head)
        prog = _program(queries)
        assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA, name
        nq = len(queries)
        want = ref.masks(queries)
        want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
        for env in ([{}, {"FEI_HEAD_FUSE": "0"}] if head else [{}]):
            with monkeypatch.context() as mp:
                for k, v in env.items():
                    mp.setenv(k, v)
                got = c.scan_masks(prog)
                tm = c.timing()
                assert (tm["body_kernel"], tm["body_nfa_words"]) == (NFA_KERNEL, words), (name, env, tm)
                assert np.array_equal(got, want), (name, env, _explain(prog, ref, queries, want, got))
                hits = c.scan_hits(prog, nq)
                assert c.timing()["body_kernel"] == NFA_KERNEL
                counts = c.scan_count(prog, nq)
            for q in range(nq):
                assert np.array_equal(hits[q], want_lists[q]), (name, env, q)
                assert int(counts[q]) == want_lists[q].size, (name, env, q)
        assert want.any() and (want != want[0]).any(), name          # the case is not vacuous


def test_sharded_nfa_scan_equals_unsharded(gpu):
    from fei_b200 import shard
    from fei_b200.corpus import Corpus
    n = 4100
    pats = ["python", r"\bpython\b.{0,60}\b(rust|django)\b", r"kubernetes.{0,60}docker"]
    prog = content_batch_program([_rx(p) for p in pats])
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA
    whole_c = Corpus().synth(0xFE1, 0, n)
    whole = whole_c.scan_hits(prog, len(pats))
    assert whole_c.timing()["body_kernel"] == NFA_KERNEL
    for world in (2, 4):
        per_rank = [Corpus().synth(0xFE1, a, b - a).scan_hits(prog, len(pats)) for a, b in shard.shard_ranges(n, world)]
        got = shard.concat_in_rank_order(per_rank)
        for q in range(len(pats)):
            assert np.array_equal(got[q], whole[q]), (world, q)


def test_malformed_nfa_section_is_refused(gpu):
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    prog = content_batch_program([_rx(r"kubernetes.{0,60}docker")])
    off = struct.unpack_from("<I", prog, 88)[0]
    c = Corpus().synth(0xFE1, 0, 1000)
    truncated = bytearray(prog[:off + 32])                  # the section's descriptor is cut in half
    struct.pack_into("<I", truncated, 8, len(truncated))
    bad_words = bytearray(prog)
    struct.pack_into("<I", bad_words, off, 3)               # W must be 1, 2, 4 or 8
    bad_class = bytearray(prog)
    off_ascii = struct.unpack_from("<I", prog, off + 32)[0]
    struct.pack_into("<H", bad_class, off_ascii + 2 * ord("k"), 200)     # class id beyond n_classes
    for bad in (truncated, bad_words, bad_class):
        with pytest.raises(_abi.FeiError) as e:
            c.scan_masks(bytes(bad))
        assert e.value.code == _abi.FEI_E_BADARG
    c.scan_masks(prog)                                       # the well-formed program still scans
    assert c.timing()["body_kernel"] == NFA_KERNEL
    c.close()


@pytest.fixture(scope="module")
def api(gpu, tmp_path_factory):
    from tests.memdir_util import build_tree
    base = str(tmp_path_factory.mktemp("memdir_nfa") / "Memdir")
    build_tree(base)
    from fei_b200.memdir_tools import utils as U
    U.set_memdir_base(base)
    return base


def test_proximity_search_and_filters_match_oracle(api):
    from fei_b200.memdir_tools import filter as F
    from fei_b200.memdir_tools.search import parse_search_args, search_memories
    from oracle import memdir_oracle as mo
    from tests.memdir_util import key_of
    base = api
    for text in ("content:/kubernetes.{0,60}docker/ with_content", "content:/kubernetes.{0,60}docker/",
                 r"content:/\bpython\b.{0,60}\b(rust|django)\b/ with_content", "content:/(?:k.{0,20}d|\\A)\\Z/"):
        q = parse_search_args(text)
        with contextlib.redirect_stdout(io.StringIO()):
            res = search_memories(q)
            mems = mo.listing(base, None, None, q.include_content)
        want = [mems[i] for i in mo.run_search(mems, q.conditions)]
        assert [key_of(m) for m in res] == [key_of(m) for m in want], text
    flt = (F.MemoryFilter("Proximity").add_condition("content", r"python.{0,60}(rust|django)")
           .add_action("move", target_folder=".Projects/Python", target_status="cur"))
    neg = F.MemoryFilter("Far").add_condition("content", r"kubernetes.{0,60}docker", negate=True).add_action("flag", flags="F")
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
