"""Head fields whose patterns the DFA refuses, scanned by the position automata of the head kernels, against CPython
re.search(p, value, re.I): masks, ordered hit lists and counts for position vectors of 1, 2, 4 and 8 words; slot modes 0, 1
and 2, empty_if_missing, both header-or-fallback pairs (a `flags` header over the file flags, a `unique_id` header over the
name), negated conditions, flags and name fields; the three ways a corpus' header fields are read; the fused head kernel
and the meta pass + survivor list; the program head in shared memory and in global memory; head and content automata in
one scan; sharded scans; malformed head sections refused; and the public API against the oracle."""
import contextlib
import io
import os
import re
import struct
from datetime import datetime, timezone

import numpy as np
import pytest

from fei_b200 import program as P
from fei_b200 import synth
from fei_b200.program import (C_BODY, C_FLAGS, C_FOLDER_SET, C_NAME, C_SLOT, NAME_DATE_STR, NAME_FILENAME, NAME_HOST, NAME_ID, NAME_TS_STR,
                              VERSION_NFA, Cond, ProgramBuilder)
from fei_b200.regexc import Pattern
from tests.blob_nfa_model import BlobNfa

pytestmark = pytest.mark.gpu

W1, W2, W4, W8 = r"d.{0,16}f", r"deploy.{0,40}fail", r"urgent.{0,90}blocked", r"deploy.{0,200}fail"
TICKET = r"[A-Z]{2,5}-\d{1,6}.{0,20}blocked"
EMPTY_OK = r"deploy.{0,40}fail|^$"              # matches the empty string: the verdict of an absent Status
FLAG_RX = r"p.{0,16}s"
ID_RX = r"a.{0,16}b"
TS_RX = r"0.{0,20}0"
BODY_RX = r"kubernetes.{0,60}docker"
TOKENS = ["deploy", "Deploy", "fail", "FAIL", "urgent", "blocked", "ABC-123", "XY-9", "d", "f", "é", "日本", "Σ", "x" * 30,
          "y" * 60, "-", " ", "release", "kubernetes", "docker"]


def _rx(p):
    return Pattern("regex", p, re.IGNORECASE)


def _text(rng, k):
    """A header value as the headers dict holds it (stripped)."""
    return " ".join(TOKENS[int(i)] for i in rng.integers(0, len(TOKENS), int(rng.integers(0, k)))).strip()


@contextlib.contextmanager
def _env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    os.environ.update(kv)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def _records(n, seed):
    """Synthetic records with generated headers: Subject always; Status, a `flags` header, a `unique_id` header and X-Note
    on some records only."""
    rng = np.random.default_rng(seed)
    recs, heads = [], []
    for i in range(n):
        r = synth.record(0x4EAD, i)
        h = {"Subject": _text(rng, 14)}
        if i % 3:
            h["Status"] = _text(rng, 8)
        if i % 4 == 1:
            h["flags"] = _text(rng, 6)
        if i % 5 == 2:
            h["unique_id"] = _text(rng, 8)
        if i % 2:
            h["X-Note"] = _text(rng, 20)
        r["hdr"] = "".join(f"{k}: {v}\n" for k, v in h.items()).encode()
        r["body"] = _text(rng, 30).encode()
        recs.append(r); heads.append(h)
    return recs, heads


def _arrays(recs, global_base=0):
    """synth.arrays_from_records with the unique_id / hostname spans of each file name ("ts.uid.host:2,flags")."""
    a = synth.arrays_from_records(recs, global_base)
    spans = []
    for r in recs:
        ts, uid, rest = r["filename"].split(".", 2)
        spans += [len(ts) + 1, len(uid), len(ts) + len(uid) + 2, len(rest.split(":2,")[0])]
    a["name_spans"] = np.array(spans, dtype=np.uint16)
    return a


def _value(rec, head, c):
    """The string condition `c` reads for one record (None: header absent)."""
    if c.kind == C_SLOT:
        if c.mode == 2:
            return list(head.values())
        v = head.get(c.field) if c.mode == 1 else next((v for k, v in head.items() if k.lower() == c.field.lower()), None)
        return "" if v is None and c.empty_if_missing else v
    if c.kind == C_FLAGS:
        return rec["flags"]
    if c.kind == C_NAME:
        if c.which == NAME_HOST:                                         # "ts.uid.host:2,flags"
            return rec["filename"].split(".", 2)[2].rsplit(":2,", 1)[0]
        if c.which == NAME_DATE_STR:                                     # str(datetime.fromtimestamp(ts)) of the wall clock
            return str(datetime.fromtimestamp(rec.get("wall", rec["ts"]), timezone.utc).replace(tzinfo=None))
        return {NAME_FILENAME: rec["filename"], NAME_ID: rec["uid"], NAME_TS_STR: str(rec["ts"])}[c.which]
    return rec["body"].decode()


def _want(recs, heads, queries):
    out = np.zeros(len(recs), dtype=np.uint32)
    for i, (rec, head) in enumerate(zip(recs, heads)):
        for q, conds in enumerate(queries):
            ok, k = True, 0
            while ok and k < len(conds):
                c = conds[k]
                if c.kind == C_FOLDER_SET:
                    ok = bool(c.set64 >> rec["folder_id"] & 1)
                    k += 1
                    continue
                v = _value(rec, head, c)
                if v is None and c.if_missing == 2:                  # header absent: the next condition decides
                    k += 1
                    continue
                if v is None:
                    ok = bool(c.if_missing)
                else:
                    vals = v if isinstance(v, list) else [v]
                    ok = any(re.search(c.pattern.text, x, re.IGNORECASE) for x in vals) != c.negate
                k += 2 if c.if_missing == 2 else 1
            out[i] |= np.uint32(ok) << np.uint32(q)
    return out


def _slot(field, p, mode=0, **kw):
    return Cond(C_SLOT, pattern=_rx(p), field=field, mode=mode, **kw)


# name -> queries; each program puts at least one pattern of every listed field into its position automaton
PROGRAMS = {
    # slot modes 0, 1, 2, empty_if_missing, negation; no meta predicate: the fused head kernel
    "slots": [[_slot("subject", W1)], [_slot("Subject", W1), _slot("Subject", "release")], [_slot("Status", EMPTY_OK, 1, empty_if_missing=True)],
              [_slot("Status", EMPTY_OK, 1, empty_if_missing=True, negate=True), _slot("SUBJECT", "deploy")], [_slot("x", W4, 2)],
              [_slot("X-Note", W8, 1)], [_slot("x-note", TICKET, negate=True)],
              [_slot("X-Note", r"^(deploy.{0,40}fail)?$", 1)]],      # a DFA of some 30 KiB: the head outgrows the staging window
    # flags, names and both header-or-fallback pairs; the flags / folder predicates make it a meta pass + survivor list
    "fallbacks": [[_slot("flags", W1, if_missing=2), Cond(C_FLAGS, pattern=_rx(FLAG_RX))],
                  [_slot("unique_id", TICKET, if_missing=2), Cond(C_NAME, which=NAME_ID, pattern=_rx(ID_RX))],
                  [Cond(C_FLAGS, pattern=_rx(FLAG_RX), negate=True)], [Cond(C_NAME, which=NAME_FILENAME, pattern=_rx(ID_RX))],
                  [Cond(C_NAME, which=NAME_TS_STR, pattern=_rx(TS_RX)), _slot("Subject", W2)],
                  [Cond(C_FOLDER_SET, set64=0b1011), _slot("subject", W4)]],
    # head and content automata in one scan
    "head+body": [[_slot("Subject", W2), Cond(C_BODY, pattern=_rx(BODY_RX))], [Cond(C_BODY, pattern=_rx(BODY_RX), negate=True)],
                  [_slot("x", TICKET, 2)]],
}


def _program(queries):
    pb = ProgramBuilder()
    for q in queries:
        pb.add_query(q)
    return pb.build()


def _head_sections(prog):
    """(field, W) of every head position automaton in the program."""
    off_slots, n_slots = struct.unpack_from("<I", prog, 32)[0], struct.unpack_from("<I", prog, 28)[0]
    out = [(f"slot{k}", BlobNfa(prog, struct.unpack_from("<I", prog, off_slots + 16 * k + 12)[0]).W)
           for k in range(n_slots) if struct.unpack_from("<I", prog, off_slots + 16 * k + 12)[0]]
    off = struct.unpack_from("<I", prog, 92)[0]
    if off:
        out += [(f"head{k}", BlobNfa(prog, o).W) for k, o in enumerate(struct.unpack_from("<6I", prog, off)) if o]
    return out


@pytest.fixture(scope="module")
def loads(gpu):
    from fei_b200.corpus import Corpus
    recs, heads = _records(4096 + 300, 20261017)
    out = {"default": Corpus().load(_arrays(recs))}
    for var in ("FEI_HDIR", "FEI_HCOLS"):
        with _env(**{var: "0"}):
            out[var] = Corpus().load(_arrays(recs))
    yield recs, heads, out
    for c in out.values():
        c.close()


@pytest.mark.parametrize("name", list(PROGRAMS))
def test_head_automata_agree_with_cpython(loads, name):
    recs, heads, corpora = loads
    queries = PROGRAMS[name]
    prog = _program(queries)
    assert struct.unpack_from("<I", prog, 4)[0] == VERSION_NFA
    sections = _head_sections(prog)
    assert sections, name                                              # the automaton, not a DFA, carries the patterns
    if name == "slots":
        assert {w for _f, w in sections} == {1, 2, 4, 8} and "slot1" in {f for f, _w in sections}     # slot 1: Status, empty_if_missing
        assert struct.unpack_from("<I", prog, 76)[0] > 32 * 1024     # a head beyond the staging window: read from global memory
    if name == "fallbacks":
        assert {f for f, _w in sections} >= {"head0", "head1", "head2", "head4"}    # flags, filename, unique_id, str(timestamp)
    nq = len(queries)
    want = _want(recs, heads, queries)
    for q in range(nq):                                                # every query hits some records and misses others
        col = want >> np.uint32(q) & 1
        assert col.any() and not col.all(), (name, q)
    in_global = bytearray(prog)
    struct.pack_into("<I", in_global, 76, 0)                           # head_bytes = 0: the head kernels read global memory
    want_lists = [np.nonzero(want >> np.uint32(q) & 1)[0].astype(np.uint64) for q in range(nq)]
    for load, c in corpora.items():
        for leg, p, env in (("smem", prog, {}), ("global", bytes(in_global), {}), ("unfused", prog, {"FEI_HEAD_FUSE": "0"})):
            with _env(**env):
                got = c.scan_masks(p)
                bad = np.nonzero(got != want)[0]
                assert bad.size == 0, (name, load, leg, int(bad[0]), recs[int(bad[0])]["hdr"], int(want[bad[0]]), int(got[bad[0]]))
                hits = c.scan_hits(p, nq)
                counts = c.scan_count(p, nq)
            for q in range(nq):
                assert np.array_equal(hits[q], want_lists[q]), (name, load, leg, q)
                assert int(counts[q]) == want_lists[q].size, (name, load, leg, q)


def test_sharded_head_scan_equals_unsharded(gpu):
    from fei_b200 import shard
    from fei_b200.corpus import Corpus
    recs, _heads = _records(4100, 7)
    queries = PROGRAMS["slots"] + [[Cond(C_FLAGS, pattern=_rx(FLAG_RX))]]
    prog = _program(queries)
    whole_c = Corpus().load(_arrays(recs))
    whole = whole_c.scan_hits(prog, len(queries))
    assert any(len(h) for h in whole)
    for world in (2, 4):
        per_rank = [Corpus().load(_arrays(recs[a:b], a)).scan_hits(prog, len(queries)) for a, b in shard.shard_ranges(len(recs), world)]
        got = shard.concat_in_rank_order(per_rank)
        for q in range(len(queries)):
            assert np.array_equal(got[q], whole[q]), (world, q)


def test_malformed_head_sections_are_refused(gpu):
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    recs, _heads = _records(500, 9)
    c = Corpus().load(_arrays(recs))
    prog = _program([[_slot("Subject", W2)], [Cond(C_FLAGS, pattern=_rx(FLAG_RX))]])
    off_slots = struct.unpack_from("<I", prog, 32)[0]
    off = struct.unpack_from("<I", prog, off_slots + 12)[0]              # slot 0's automaton
    head_nfa = struct.unpack_from("<I", prog, 92)[0]
    head_bytes = struct.unpack_from("<I", prog, 76)[0]
    bad_words = bytearray(prog); struct.pack_into("<I", bad_words, off, 3)                       # W must be 1, 2, 4 or 8
    bad_class = bytearray(prog)
    struct.pack_into("<H", bad_class, struct.unpack_from("<I", prog, off + 32)[0] + 2 * ord("d"), 200)   # class beyond n_classes
    outside = bytearray(prog); struct.pack_into("<I", outside, off_slots + 12, head_bytes)        # a head section behind the head
    bad_table = bytearray(prog); struct.pack_into("<I", bad_table, head_nfa, 8)                  # flags automaton offset misaligned
    version1 = bytearray(prog); struct.pack_into("<I", version1, 4, 1)                           # automata in a version-1 program
    no_part = bytearray(prog); struct.pack_into("<I", no_part, off_slots + 12, 0)                # a slot with neither part
    for what, bad in (("words", bad_words), ("class", bad_class), ("outside", outside), ("table", bad_table), ("version", version1),
                      ("empty slot", no_part)):
        with pytest.raises(_abi.FeiError) as e:
            c.scan_masks(bytes(bad))
        assert e.value.code == _abi.FEI_E_BADARG, what
    assert c.scan_masks(prog).any()                                      # the well-formed program still scans
    c.close()


@pytest.fixture(scope="module")
def api(gpu, tmp_path_factory):
    from tests.memdir_util import build_tree
    from fei_b200.memdir_tools import utils as U
    base = str(tmp_path_factory.mktemp("memdir_head_nfa") / "Memdir")
    build_tree(base)
    U.set_memdir_base(base)
    for k, subj in enumerate(["OPS-4411 deploy blocked", "ABC-12 waiting, still blocked by QA", "XY-7 fine", "deploy then fail soon",
                              "urgent: please release the deploy", "no ticket blocked"]):
        U.save_memory("" if k % 2 else ".Projects/AI", f"body {k}", {"Subject": subj, "Tags": "ops"}, flags="F" if k % 3 else "")
    return base


def test_api_matches_oracle(api):
    from fei_b200.memdir_tools import filter as F
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    from fei_b200.memdir_tools.search import parse_search_args, search_memories
    from oracle import memdir_oracle as mo
    from tests.memdir_util import key_of
    base = api
    for text, p in ((r"subject:/[A-Z]{2,5}-\d{1,6}.{0,20}blocked/", TICKET), (r"filename=/e.{0,30}:2,\w*F/", r"e.{0,30}:2,\w*F"),
                    (r"folder=/p.{0,20}ai/", r"p.{0,20}ai"), (r"subject:/(urgent|asap).{0,30}(deploy|release)/ #ops", r"(urgent|asap).{0,30}(deploy|release)")):
        assert P._route([_rx(p)], P._head_fits)[1] == [0], text        # the position automaton carries the pattern
        q = parse_search_args(text)
        with contextlib.redirect_stdout(io.StringIO()):
            res = search_memories(q)
            mems = mo.listing(base, None, None, q.include_content)
        want = [mems[i] for i in mo.run_search(mems, q.conditions)]
        assert want and len(want) < len(mems), text
        assert [key_of(m) for m in res] == [key_of(m) for m in want], text
    prox = F.MemoryFilter("Blocked").add_condition("Subject", TICKET).add_action("flag", flags="F")
    neg = F.MemoryFilter("NotDeploy").add_condition("Subject", r"deploy.{0,40}(fail|blocked)", negate=True).add_action("flag", flags="S")
    mgr = F.FilterManager()
    mgr.add_filter(prox); mgr.add_filter(neg)
    for statuses in (["new"], ["cur", "new"]):
        with contextlib.redirect_stdout(io.StringIO()):
            stats = mgr.process_memories(statuses=statuses, dry_run=True)
            mems = [m for s in statuses for m in mo.listing(base, None, [s], True)]
        want = mo.run_filters(mems, [{"name": f.name, "conditions": f.conditions, "actions": f.actions} for f in mgr.filters])
        for k in ("total_memories", "filters_applied", "actions_taken", "memories_modified"):
            assert stats[k] == want[k], (statuses, k, stats[k], want[k])
        assert sorted(d["memory_id"] for d in stats["details"]) == sorted(d["memory_id"] for d in want["details"])
    from fei_b200 import packer
    arch = MemoryArchiver()
    crit = {"Subject": TICKET}
    with contextlib.redirect_stdout(io.StringIO()):
        row = arch.match_criteria([crit])[0]
        pm = packer.packed()
        mems = mo.listing(base, None, None, True)
    idx = np.concatenate([np.arange(a, b) for a, b in pm.ranges(None, None)])
    got = [key_of(mems[k]) for k in np.nonzero(row[idx])[0].tolist()]
    want = [key_of(m) for m in mems if mo.matches_criteria(m, crit)]
    assert want and len(want) < len(mems)
    assert got == want
