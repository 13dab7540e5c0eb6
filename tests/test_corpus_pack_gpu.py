"""Every way of filling a corpus packs the same records the same way, and both fetches give them back byte for byte.

One record set (odd body lengths around the 16-byte unit and the 4096-byte mark, a body over 64 KiB, non-ASCII text, more
than two 4096-record windows, no '\\r' so that every path yields the same canonical text) is loaded through fei_corpus_load,
fei_corpus_load_raw, fei_corpus_load_raw_spans with permuted gapped spans, and the spans load of a text staged piece by piece;
a snapshot of one of them is restored; fei_corpus_synth is held against the host generator."""
import re

import numpy as np
import pytest

from fei_b200 import synth
from fei_b200.program import content_batch_program
from fei_b200.regexc import Pattern

pytestmark = pytest.mark.gpu

BATCH32 = ["python", "docker|kubernetes", "neural networks", "react", "angular", "rust", "django", "flask", "terraform", "ansible",
           "microservices", "big data", "ci/cd", "git", "aws|azure|gcp", "spring boot", r"vue\.js", r"node\.js", "devops", "security",
           "blockchain", "testing", "databases", "algorithms", "cloud computing", "mobile development", "computer vision",
           "reinforcement learning", "ui/ux", "web development", "data structures", "machine learning"]
WORDS = ["python", "Docker", "kubernetes", "neural networks", "rust", "flask", "machine learning", "ci/cd", "git", "naïve", "café",
         "日本語", "emoji😀", "Straße", "Σίσυφος", "İstanbul", "GIT", "data\nstructures", "node.js", "x"]
N = 2 * 4096 + 700
SPECIAL = {0: 0, 1: 1, 2: 15, 3: 16, 4: 17, 4095: 4095, 4096: 4097, 4097: 4096, 5000: 70001, 8191: 17, 8192: 0, N - 1: 33}
RANGES = [(0, N), (4000, 300), (8100, 200), (N - 1, 1), (5, 0)]


def _body(rng, length):
    """Valid UTF-8 of exactly `length` bytes, no whitespace at either end."""
    if length == 0:
        return b""
    text = ""
    while len(text.encode()) < length:
        text += WORDS[int(rng.integers(len(WORDS)))] + " "
    b = text.encode()[:length].decode("utf-8", "ignore").rstrip().encode()
    return b + b"x" * (length - len(b))


def _records():
    rng = np.random.default_rng(0xC0DE)
    recs = []
    for i in range(N):
        r = synth.record(31, i)
        r["body"] = _body(rng, SPECIAL.get(i, int(rng.integers(0, 400))))
        text = synth.file_text(r)
        r["bits"] = (0 if text.isascii() else 2) | (4 if "Σ" in text else 0) | (8 if "İ" in text else 0)   # what load_raw computes
        recs.append(r)
    return recs


@pytest.fixture(scope="module")
def packs(gpu, tmp_path_factory):
    from fei_b200.corpus import Corpus
    recs = _records()
    a = synth.arrays_from_records(recs)
    assert b"\r" not in a["hdr"].tobytes() + a["body"].tobytes()
    meta = {k: a[k] for k in ("ts", "wall", "flags8", "fsb")}
    raw = [synth.file_text(r).encode() for r in recs]
    lens = np.array([len(p) for p in raw], dtype=np.uint64)
    off = np.zeros(N + 1, dtype=np.uint64); np.cumsum(lens, out=off[1:])
    loads = {"load": Corpus().load(a)}
    loads["load_raw"] = Corpus()
    assert loads["load_raw"].load_raw(dict(meta, n=N, raw=np.frombuffer(b"".join(raw), dtype=np.uint8), raw_off=off)).all()
    rng = np.random.default_rng(7)
    begin = np.zeros(N, dtype=np.uint64)
    pos = 777
    for i in rng.permutation(N).tolist():
        begin[i] = pos; pos += int(lens[i]) + i % 5
    total = pos
    scattered = np.full(total, ord("-"), dtype=np.uint8)
    for i in range(N):
        scattered[int(begin[i]):int(begin[i] + lens[i])] = np.frombuffer(raw[i], dtype=np.uint8)
    spans = dict(meta, n=N, raw_bytes=total, raw_begin=begin, raw_len=lens)
    loads["spans"] = Corpus()
    assert loads["spans"].load_raw(dict(spans, raw=scattered)).all()
    loads["staged"] = Corpus()
    cut = [0, total // 7, total // 3, total // 2, total - 5, total]
    for k in (3, 0, 4, 2, 1):
        loads["staged"].stage_text(total, scattered[cut[k]:cut[k + 1]], cut[k])
    assert loads["staged"].load_raw(dict(spans, raw=None)).all()
    path = str(tmp_path_factory.mktemp("snap") / "corpus.snap")
    loads["spans"].save(path)
    loads["snapshot"] = Corpus()
    loads["snapshot"].load_snapshot(path)
    return a, loads


@pytest.fixture(scope="module")
def synth_pack(gpu):
    from fei_b200.corpus import Corpus
    n = 4096 + 1000
    return synth.corpus_arrays(0x5EED, 123, n), Corpus().synth(0x5EED, 123, n)


def _check_ranges(c, a, ranges):
    for first, cnt in ranges:
        got = c.fetch(first, cnt)
        for k in ("ts", "wall", "flags8", "fsb"):
            assert np.array_equal(got[k], a[k][first:first + cnt]), (k, first, cnt)
        for blob, off in (("hdr", "hdr_off"), ("body", "body_off")):
            o = a[off].astype(np.int64)
            lo, hi = int(o[first]), int(o[first + cnt])
            assert np.array_equal(got[off].astype(np.int64), o[first:first + cnt + 1] - lo), (off, first, cnt)
            assert got[blob][:hi - lo].tobytes() == a[blob][lo:hi].tobytes(), (blob, first, cnt)


def _check_fetch_records(c, n):
    rng = np.random.default_rng(n)
    idx = np.concatenate([rng.integers(0, n, 2500), [n - 1, 0, n - 1, 4096, 4095]]).astype(np.uint64)
    full = c.fetch(0, n)
    hdr, ho, body, bo = c.fetch_records(idx)
    for j, r in enumerate(idx.tolist()):
        for got, off, blob, key in ((hdr, ho, full["hdr"], "hdr_off"), (body, bo, full["body"], "body_off")):
            want = blob[int(full[key][r]):int(full[key][r + 1])].tobytes()
            assert got[int(off[j]):int(off[j + 1])] == want, (key, j, r)


@pytest.mark.parametrize("name", ["load", "load_raw", "spans", "staged", "snapshot"])
def test_fetch_gives_back_the_records(packs, name):
    a, loads = packs
    _check_ranges(loads[name], a, RANGES)
    _check_fetch_records(loads[name], N)


def test_synth_fetch_equals_host_generator(synth_pack):
    a, c = synth_pack
    n = int(a["n"])
    _check_ranges(c, a, [(0, n), (4000, 200), (n - 1, 1), (0, 0)])
    _check_fetch_records(c, n)


def test_load_paths_pack_alike_and_scan_alike(packs):
    a, loads = packs
    keys = ("n", "hdr_bytes", "body_bytes", "tile_bytes", "n_groups")
    stats = {name: {k: c.stats()[k] for k in keys} for name, c in loads.items()}
    assert stats["load"]["hdr_bytes"] == int(a["hdr_off"][-1]) and stats["load"]["body_bytes"] == int(a["body_off"][-1])
    assert stats["load"]["n_groups"] == 3 * 128
    for name in loads:
        assert stats[name] == stats["load"], name
    prog = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in BATCH32])
    want = loads["load"].scan_masks(prog)
    assert np.count_nonzero(want) > N // 4
    for name, c in loads.items():
        assert np.array_equal(c.scan_masks(prog), want), name


def test_fetch_capacity_errors(packs):
    from fei_b200 import _abi
    a, loads = packs
    c, l, p = loads["load_raw"], _abi.lib(), _abi.ptr
    first, cnt = 4090, 20
    need_h = int(a["hdr_off"][first + cnt] - a["hdr_off"][first])
    need_b = int(a["body_off"][first + cnt] - a["body_off"][first])
    assert need_h > 0 and need_b > 0
    hbuf = np.zeros(need_h, dtype=np.uint8); bbuf = np.zeros(need_b, dtype=np.uint8)
    assert l.fei_corpus_fetch(c.handle, first, cnt, p(hbuf), need_h - 1, None, None, 0, None, None, None, None, None) == _abi.FEI_E_CAPACITY
    assert l.fei_corpus_fetch(c.handle, first, cnt, None, 0, None, p(bbuf), need_b - 1, None, None, None, None, None) == _abi.FEI_E_CAPACITY
    assert l.fei_corpus_fetch(c.handle, first, cnt, p(hbuf), need_h, None, p(bbuf), need_b, None, None, None, None, None) == _abi.FEI_OK
    assert bbuf.tobytes() == a["body"][int(a["body_off"][first]):int(a["body_off"][first + cnt])].tobytes()
    idx = np.arange(first, first + cnt, dtype=np.uint64)[::-1].copy()
    for hcap, bcap in ((need_h - 1, need_b), (need_h, need_b - 1)):
        ho = np.zeros(cnt + 1, dtype=np.uint64); bo = np.zeros(cnt + 1, dtype=np.uint64)
        rc = l.fei_corpus_fetch_records(c.handle, p(idx), cnt, p(hbuf), hcap, p(ho), p(bbuf), bcap, p(bo))
        assert rc == _abi.FEI_E_CAPACITY and (int(ho[cnt]), int(bo[cnt])) == (need_h, need_b)
