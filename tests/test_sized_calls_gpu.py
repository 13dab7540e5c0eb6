"""The calls that size variable-length output, place it with offsets and then write it, at their edges: empty inputs and corpora,
a sizing call with null buffers, an exact buffer (FEI_OK) and a buffer one byte or one record short (FEI_E_CAPACITY with the
same needed sizes the exact call reports)."""
import ctypes as C

import numpy as np
import pytest

from fei_b200 import _abi, synth
from fei_b200.program import C_SLOT, Cond, ProgramBuilder
from fei_b200.regexc import Pattern
from oracle import chain_oracle as co
from tests.chain_util import single_block

pytestmark = pytest.mark.gpu

SEED = 0x51ED
FOLDERS = [b"", b".Projects/Python", b".Projects/AI", b".ToDoLater/Learning"]
OK, CAP = _abi.FEI_OK, _abi.FEI_E_CAPACITY


def _p(a):
    return None if a is None else _abi.ptr(a)


def _u64(n, fill=0):
    return np.full(n, fill, dtype=np.uint64)


def _prog(*fields):
    pb = ProgramBuilder()
    pb.add_query([Cond(C_SLOT, pattern=Pattern("regex", "", 0), field=f, mode=1, if_missing=1) for f in fields])
    return pb.build()


@pytest.fixture(scope="module")
def small(gpu):
    """40 synthetic records with their file names ("ts.uid.host:2,flags") and the unique_id / hostname spans in them."""
    from fei_b200.corpus import Corpus
    a = synth.corpus_arrays(SEED, 0, 40)
    spans = []
    for r in a["records"]:
        ts, uid, rest = r["filename"].split(".", 2)
        spans += [len(ts) + 1, len(uid), len(ts) + len(uid) + 2, len(rest.split(":2,")[0])]
    a["name_spans"] = np.array(spans, dtype=np.uint16)
    return Corpus().load(a)


@pytest.fixture(scope="module")
def empty(gpu):
    from fei_b200.corpus import Corpus
    return Corpus().synth(SEED, 0, 0)


def _format(c, idx, fmt, opts, out, cap, off):
    names = np.frombuffer(b"".join(FOLDERS), dtype=np.uint8)
    foff = _u64(len(FOLDERS) + 1)
    foff[1:] = np.cumsum([len(f) for f in FOLDERS])
    return _abi.lib().fei_corpus_format_records(c.handle, _p(idx), idx.size, fmt, opts, _p(names), _p(foff), len(FOLDERS), _p(out), cap,
                                                _p(off), C.byref(C.c_float()))


@pytest.mark.parametrize("opts", [0, _abi.FEI_FMT_CONTENT])
@pytest.mark.parametrize("fmt", [_abi.FEI_FMT_JSON, _abi.FEI_FMT_CSV, _abi.FEI_FMT_COMPACT, _abi.FEI_FMT_TEXT])
def test_format_records_buffer_sizes(small, empty, fmt, opts):
    idx = np.array([3, 0, 17, 3, small.n - 1], dtype=np.uint64)            # any order, repeats allowed
    m = idx.size
    need = _u64(m + 1)
    assert _format(small, idx, fmt, opts, None, 0, need) == CAP
    total = int(need[m])
    assert need[0] == 0 and np.all(need[1:] > need[:-1])
    out, off = np.zeros(total, dtype=np.uint8), _u64(m + 1)
    assert _format(small, idx, fmt, opts, out, total, off) == OK
    assert np.array_equal(off, need)
    for i in range(m):                                                     # each record's text is the one it gets alone
        one, one_off = np.zeros(total, dtype=np.uint8), _u64(2)
        assert _format(small, idx[i:i + 1], fmt, opts, one, total, one_off) == OK
        assert one[:int(one_off[1])].tobytes() == out[int(off[i]):int(off[i + 1])].tobytes()
    short = _u64(m + 1)
    assert _format(small, idx, fmt, opts, out, total - 1, short) == CAP
    assert np.array_equal(short, need)
    for c in (small, empty):
        off0 = _u64(1, 7)
        assert _format(c, idx[:0], fmt, opts, None, 0, off0) == OK and off0[0] == 0


def test_slot_values_buffer_sizes(small, empty):
    lib, prog, n = _abi.lib(), _prog("Tags"), small.n
    present, need = np.zeros(n, dtype=np.uint8), _u64(n + 1)
    assert lib.fei_corpus_slot_values(small.handle, prog, len(prog), _p(present), _p(need), None, 0) == CAP
    total = int(need[n])
    assert total > 0 and present.all()
    blob, off = np.zeros(total, dtype=np.uint8), _u64(n + 1)
    assert lib.fei_corpus_slot_values(small.handle, prog, len(prog), _p(present), _p(off), _p(blob), total) == OK
    assert np.array_equal(off, need)
    want = synth.corpus_arrays(SEED, 0, n)["records"]
    for i, r in enumerate(want):
        tags = next(l for l in r["hdr"].split(b"\n") if l.startswith(b"Tags: "))[6:]
        assert blob[int(off[i]):int(off[i + 1])].tobytes() == tags
    short = _u64(n + 1)
    assert lib.fei_corpus_slot_values(small.handle, prog, len(prog), _p(present), _p(short), _p(blob), total - 1) == CAP
    assert np.array_equal(short, need)
    off0 = _u64(1, 7)
    assert lib.fei_corpus_slot_values(empty.handle, prog, len(prog), _p(np.zeros(1, dtype=np.uint8)), _p(off0), None, 0) == OK
    assert off0[0] == 0


def _tag_edit(c, tags, rec, cap, text, text_cap, off, has):
    prog = _prog("Tags", "Subject")
    src = np.frombuffer(b"".join(tags) or b"\0", dtype=np.uint8)
    toff = _u64(len(tags) + 1)
    toff[1:] = np.cumsum([len(t) for t in tags])
    count = C.c_uint64(7)
    rc = _abi.lib().fei_corpus_tag_edit(c.handle, prog, len(prog), 0, _p(src), _p(toff), len(tags), _p(rec), cap, C.byref(count),
                                        _p(text), text_cap, _p(off), _p(has))
    return rc, count.value


def test_tag_edit_buffer_sizes(small, empty):
    n, tags = small.n, [b"zz-added"]                                       # a new tag changes every record
    need = _u64(1)
    assert _tag_edit(small, tags, None, 0, None, 0, need, None) == (CAP, n)
    total = int(need[0])
    assert total > 0
    rec, text, off, has = _u64(n), np.zeros(total, dtype=np.uint8), _u64(3 * n + 1), np.zeros(n, dtype=np.uint8)
    assert _tag_edit(small, tags, rec, n, text, total, off, has) == (OK, n)
    assert off[3 * n] == total and np.array_equal(rec, np.arange(n, dtype=np.uint64))
    for cap, text_cap in ((n - 1, total), (n, total - 1)):
        short = _u64(1)
        assert _tag_edit(small, tags, rec, cap, text, text_cap, short, has) == (CAP, n)
        assert short[0] == total
    for c, t in ((small, []), (empty, tags)):                              # nothing changes: no buffers needed
        off0 = _u64(1, 7)
        assert _tag_edit(c, t, None, 0, None, 0, off0, None) == (OK, 0) and off0[0] == 0


def _fetch_records(c, idx, hdr, hcap, body, bcap):
    ho, bo = _u64(idx.size + 1, 7), _u64(idx.size + 1, 7)
    rc = _abi.lib().fei_corpus_fetch_records(c.handle, _p(idx), idx.size, _p(hdr), hcap, _p(ho), _p(body), bcap, _p(bo))
    return rc, ho, bo


def test_fetch_records_buffer_sizes(small, empty):
    idx = np.array([5, 5, 0, small.n - 1], dtype=np.uint64)
    m = idx.size
    rc, ho, bo = _fetch_records(small, idx, None, 0, None, 0)
    assert rc == OK
    hb, bb = int(ho[m]), int(bo[m])
    hdr, body = np.zeros(hb, dtype=np.uint8), np.zeros(bb, dtype=np.uint8)
    rc, ho2, bo2 = _fetch_records(small, idx, hdr, hb, body, bb)
    assert rc == OK and np.array_equal(ho2, ho) and np.array_equal(bo2, bo)
    want = synth.corpus_arrays(SEED, 0, small.n)["records"]
    for i, r in enumerate(idx.tolist()):
        assert hdr[int(ho[i]):int(ho[i + 1])].tobytes() == want[r]["hdr"]
        assert body[int(bo[i]):int(bo[i + 1])].tobytes() == want[r]["body"]
    for hcap, bcap in ((hb - 1, bb), (hb, bb - 1)):
        rc, ho3, bo3 = _fetch_records(small, idx, hdr, hcap, body, bcap)
        assert rc == CAP and np.array_equal(ho3, ho) and np.array_equal(bo3, bo)
    for c in (small, empty):
        rc, ho0, bo0 = _fetch_records(c, idx[:0], None, 0, None, 0)
        assert rc == OK and ho0[0] == 0 and bo0[0] == 0


@pytest.mark.parametrize("n", [0, 1])
def test_corpus_synth_tiny(gpu, n):
    from fei_b200.corpus import Corpus
    c = Corpus().synth(SEED, 5, n)
    st = c.stats()
    assert st["n"] == n and st["hdr_bytes"] == (len(synth.record(SEED, 5)["hdr"]) if n else 0)
    got, want = c.fetch(0, n), synth.corpus_arrays(SEED, 5, n)
    for k in ("hdr_off", "body_off", "ts", "wall", "flags8", "fsb"):
        assert np.array_equal(got[k], want[k]), k
    if n:
        assert got["hdr"].tobytes() == want["hdr"][:int(want["hdr_off"][1])].tobytes()
        assert got["body"].tobytes() == want["body"][:int(want["body_off"][1])].tobytes()
    assert c.scan_count(_prog("Tags"), 1).tolist() == [n]


@pytest.mark.parametrize("n", [0, 1])
def test_chain_load_cols_tiny(gpu, chain_golden, n):
    from fei_b200.memdir_tools import memorychain as mc
    blocks = [single_block(chain_golden["single"][0])]
    blocks[0].previous_hash = str(blocks[0].previous_hash)               # the resident column form takes string links only
    cols, stored = mc.chain_columns(blocks)
    hb, ho = mc._str_blob([s if isinstance(s, str) else "" for s in stored])
    lib, h = _abi.lib(), C.c_void_p()
    _abi.check(lib.fei_chain_create(C.byref(h)))
    try:
        _abi.check(lib.fei_chain_load_cols(h, mc._cols_struct(cols), _abi.ptr(hb), _abi.ptr(ho), n, 0))
        dig, fb, kind = np.zeros((1, 32), dtype=np.uint8), C.c_int64(), C.c_int32()
        _abi.check(lib.fei_chain_validate(h, C.byref(fb), C.byref(kind), _abi.ptr(dig), None))
        assert (fb.value, kind.value) == (-1, 0)
        if n:
            off, buf = _u64(2), np.zeros(4096, dtype=np.uint8)
            _abi.check(lib.fei_chain_fetch(h, 0, 1, _abi.ptr(buf), buf.size, _abi.ptr(off), None, None))
            assert buf[:int(off[1])].tobytes() == co.block_text(blocks[0]).encode()
            assert bytes(dig[0]).hex() == co.block_hash(blocks[0])
    finally:
        lib.fei_chain_destroy(h)
