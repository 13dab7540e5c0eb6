"""GPU parity of the scan kernels through the C ABI against the oracle (record-level restatement
of search.py / filter.py) on seeded synthetic corpora plus adversarial records."""
import contextlib
import os
import re
import struct

import numpy as np
import pytest

from fei_b200 import synth
from fei_b200.program import (C_BODY, C_DATE_CMP, C_FLAGS, C_FOLDER_SET, C_NAME, C_SLOT, C_STATUS_SET, CMP, Cond, ProgramBuilder,
                              content_batch_program, const)
from fei_b200.regexc import Pattern
from oracle import memdir_oracle as mo

pytestmark = pytest.mark.gpu

BATCH32 = ["python", "docker|kubernetes", "neural networks", "react", "angular", "rust", "django", "flask", "terraform", "ansible",
           "microservices", "big data", "ci/cd", "git", "aws|azure|gcp", "spring boot", r"vue\.js", r"node\.js", "devops", "security",
           "blockchain", "testing", "databases", "algorithms", "cloud computing", "mobile development", "computer vision",
           "reinforcement learning", "ui/ux", "web development", "data structures", "machine learning"]


def memories_of(recs):
    return [mo.make_memory(r["filename"], r["folder"], r["status"], synth.file_text(r), True) for r in recs]


@pytest.fixture(scope="module")
def corpus3k(gpu):
    from fei_b200.corpus import Corpus
    n = 3000
    arrays = synth.corpus_arrays(0xFE1, 0, n)
    c = Corpus().load(arrays)
    return c, arrays, memories_of(arrays["records"])


def test_gpu_generator_and_tiler_roundtrip(gpu):
    """fei_corpus_synth (device generator + tiler) == host generator, byte for byte, after un-tiling."""
    from fei_b200.corpus import Corpus
    n = 2500                                            # crosses window boundaries (1024) with a ragged tail
    c = Corpus().synth(0xFE1, 100, n)
    got = c.fetch(0, n)
    want = synth.corpus_arrays(0xFE1, 100, n)
    for k in ("hdr_off", "body_off", "ts", "wall", "flags8", "fsb"):
        assert np.array_equal(got[k], want[k]), k
    assert bytes(got["hdr"][:int(got["hdr_off"][n])]) == bytes(want["hdr"][:int(want["hdr_off"][n])])
    assert bytes(got["body"][:int(got["body_off"][n])]) == bytes(want["body"][:int(want["body_off"][n])])
    st = c.stats()
    assert st["n"] == n and st["tile_bytes"] >= st["body_bytes"] and st["tile_bytes"] <= st["body_bytes"] + 16 * n


def test_load_path_roundtrip_with_odd_lengths(gpu):
    from fei_b200.corpus import Corpus
    recs = []
    for i, ln in enumerate([0, 1, 15, 16, 17, 31, 32, 33, 255, 256, 257, 1000, 5000, 0, 3, 64]):
        r = synth.record(7, i)
        r["body"] = bytes((j * 7 + i) % 251 + 1 for j in range(ln))
        recs.append(r)
    a = synth.arrays_from_records(recs)
    c = Corpus().load(a)
    got = c.fetch(0, len(recs))
    assert np.array_equal(got["body_off"], a["body_off"])
    assert bytes(got["body"][:int(a["body_off"][-1])]) == bytes(a["body"][:int(a["body_off"][-1])])


def test_batch32_content_patterns_match_reference_semantics(corpus3k):
    c, arrays, mems = corpus3k
    prog = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in BATCH32])
    masks = c.scan_masks(prog)
    hits = c.scan_hits(prog, 32)
    for q, p in enumerate(BATCH32):
        want = mo.run_search(mems, [{"field": "content", "operator": "matches", "value": p}])
        got = np.nonzero(masks >> np.uint32(q) & np.uint32(1))[0].tolist()
        assert got == want, p
        assert hits[q].tolist() == want, p


def test_single_regex_with_gaps_and_class_indexed_tables(corpus3k):
    c, arrays, mems = corpus3k
    for p in [r"kubernetes.*docker|docker.*kubernetes", r"react|angular", r"\bgit\b", r"^# (research|book review)", r"(?m)^- clean code$",
              r"\d{3}", r"learning\.$", r"(?s)overview.*summary", r"\w+ design\b", r"[aeiou]{3}"]:
        pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", p, re.IGNORECASE))])
        got = np.nonzero(c.scan_masks(pb.build()))[0].tolist()
        want = mo.run_search(mems, [{"field": "content", "operator": "matches", "value": p}])
        assert got == want, p


def _search_prog(conds):
    """Minimal host compile of reference-style conditions for the fields these tests use."""
    out = []
    for f, op, v in conds:
        fl = f.lower()
        if fl == "content":
            kind = {"matches": "regex", "contains": "contains"}[op]
            out.append(Cond(C_BODY, pattern=Pattern(kind, v if kind == "regex" else v.lower(), re.IGNORECASE if kind == "regex" else 0)))
        elif fl == "flags":
            out.append(Cond(C_FLAGS, pattern=Pattern("exact_contains", v.upper())))
        elif fl == "date":
            import calendar, dateutil.parser
            d = dateutil.parser.parse(v)
            out.append(Cond(C_DATE_CMP, op=CMP[op], i64=calendar.timegm(d.timetuple()) * 1000000 + d.microsecond))
        else:
            kind = {"has_tag": "has_tag", "contains": "contains", "matches": "regex", "=": "equals", "startswith": "startswith", "endswith": "endswith"}[op]
            pat = Pattern(kind, v if kind == "regex" else v.lower(), re.IGNORECASE if kind == "regex" else 0)
            status_hdr = f in ("Status", "status_value", "state")
            out.append(Cond(C_SLOT, pattern=pat, field="Status" if status_hdr else f, mode=1 if status_hdr else 0, empty_if_missing=status_hdr))
    return out


def test_multi_field_filter_cfg2(corpus3k):
    """BASELINE configs[1]: tags + flags + date + body regex (search.py semantics)."""
    c, arrays, mems = corpus3k
    import datetime
    median_ts = int(np.median(arrays["ts"]))
    t = datetime.datetime.fromtimestamp(median_ts, datetime.timezone.utc).strftime("%Y-%m-%d %H:%M:%S")
    cases = [
        [("Tags", "has_tag", "python"), ("flags", "has_flag", "F"), ("date", ">", t), ("content", "matches", r"react|angular")],
        [("Tags", "has_tag", "python")],
        [("flags", "has_flag", "F")],
        [("flags", "has_flag", "FS")],
        [("date", ">", t)], [("date", "<=", t)],
        [("Priority", "=", "HIGH"), ("Status", "=", "active")],
        [("subject", "contains", "review"), ("content", "contains", "review")],
        [("tags", "contains", "rust"), ("Priority", "contains", "i")],
        [("Author", "startswith", "j")], [("Version", "endswith", ".0")], [("nope", "contains", "")], [("Tags", "contains", "")],
        [("state", "matches", "^(active|pending)$")],
    ]
    for conds in cases:
        pb = ProgramBuilder(); pb.add_query(_search_prog(conds))
        got = np.nonzero(c.scan_masks(pb.build()))[0].tolist()
        want = mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in conds])
        assert got == want, conds
    # all of them as one 14-query program: same masks, one pass
    pb = ProgramBuilder()
    for conds in cases:
        pb.add_query(_search_prog(conds))
    masks = c.scan_masks(pb.build())
    for q, conds in enumerate(cases):
        want = mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in conds])
        assert np.nonzero(masks >> np.uint32(q) & np.uint32(1))[0].tolist() == want, conds


ADVERSARIAL = [
    # (header text, body) pairs exercising the parser quirks in SURVEY.md 8(a)
    ("Subject: Beta ", " split here\nTags: x\n---\nbody after second sep"),          # '---' inside a header value
    ("Tags: a,b\ntags: lower,c\nTags: final,python\n", "dup keys"),                      # duplicate-case keys, last value wins
    ("  Subject  :  spaced out  \n\tTags\t:\tpython , rust\t\n", "Ünïcödé K ſ body\nwith KELVIN \u212a and long s \u017f"),
    ("NoColonLine\nTags: python\n: emptykey\nKey:\n", ""),                               # line without colon, empty key, empty value
    ("Tags:\u00a0python\u2003\n", "nbsp and em-space around the tag"),
    ("Tags: " + ",".join(f"tag{i}" for i in range(20)) + ",python, lower\nSubject: " + "long subject " * 8 + "beta\n", "values longer than a column slot (64 bytes): directory walk"),
    ("Subject: x\nStatus: done\nStatus: ACTIVE\n", "status twice"),
    ("", "no headers at all but a body mentioning python and docker then kubernetes"),
    ("Tags: Python,\u212aelvin\nPriority: HIGH\n", "kelvin sign tag"),
    ("Subject: caf\u00e9 R\u00c9SUM\u00c9\n", "caf\u00e9 r\u00e9sum\u00e9 \U0001F409 dragon\nline2 react"),
    ("Tags: a\x0bb,\x1cpython\x1f\n", "odd whitespace controls"),
    ("tags: first\nTAGS: second\ntags: third\nTags: fourth\n", "one key in three spellings: the first one names the dict entry"),
]


@contextlib.contextmanager
def _env0(var):
    os.environ[var] = "0"
    try:
        yield
    finally:
        del os.environ[var]


def _three_loads(recs):
    """The corpus loaded the three ways its header fields can be read: value columns + directory (default), the in-scan
    text parser for every record (FEI_HDIR=0; otherwise only > 64 KiB headers take it), the directory walk for every
    field (FEI_HCOLS=0: no value columns)."""
    from fei_b200.corpus import Corpus
    loads = {"default": Corpus().load(synth.arrays_from_records(recs))}
    for var in ("FEI_HDIR", "FEI_HCOLS"):
        with _env0(var):
            loads[var] = Corpus().load(synth.arrays_from_records(recs))
    return loads


def _scan_legs(c, prog):
    """Masks of one program: as built (automata in the shared-memory copy of the program head), with fei_prog_hdr.head_bytes
    (byte offset 76) set to 0 so that the head kernels read every automaton from global memory, and with the head pass
    split into the meta kernel + work list + parse kernel (FEI_HEAD_FUSE=0)."""
    legs = {"smem": c.scan_masks(prog)}
    in_global = bytearray(prog)
    struct.pack_into("<I", in_global, 76, 0)
    legs["global"] = c.scan_masks(bytes(in_global))
    with _env0("FEI_HEAD_FUSE"):
        legs["unfused"] = c.scan_masks(prog)
    return legs


def _adversarial_records():
    recs = []
    for i, (h, b) in enumerate(ADVERSARIAL):
        r = synth.record(11, i)
        text = h + "---" + b if True else None
        hdr_text, sep, rest = text.partition("---")
        r["hdr"] = hdr_text.encode(); r["body"] = rest.strip().encode(); r["raw_text"] = text
        recs.append(r)
    # a header text longer than 65535 bytes: the header directory (hdir.cu) defers to the in-scan text parser
    big = "Filler: " + "x" * 70000 + "\nTags: python , huge\nsubject:  Big One \nTags: final,python\nKey:\n"
    r = synth.record(11, 98); r["hdr"] = big.encode(); r["body"] = b"big header body"; r["raw_text"] = big + "---\nbig header body"
    recs.append(r)
    # plus one record with no separator at all
    r = synth.record(11, 99); r["hdr"] = b""; r["body"] = "just text: no separator python".encode(); r["raw_text"] = "just text: no separator python"
    r["bits"] = 1
    recs.append(r)
    return recs, [mo.make_memory(r["filename"], r["folder"], r["status"], r["raw_text"], True) for r in recs]


def test_adversarial_records_header_parser_and_unicode(gpu):
    recs, mems = _adversarial_records()
    checks = []                                   # (what, program, oracle's record list)
    cases = [
        [("Tags", "has_tag", "python")], [("tags", "has_tag", "final")], [("Tags", "has_tag", "lower")], [("tags", "contains", "c")],
        [("Subject", "=", "beta")], [("subject", "contains", "spaced out")], [("subject", "=", "spaced out")], [("Key", "=", "")],
        [("Status", "=", "active")], [("state", "=", "done")], [("Tags", "has_tag", "kelvin")], [("Tags", "has_tag", "b")],
        [("content", "matches", r"\bk")], [("content", "matches", "s")], [("content", "contains", "k")], [("content", "contains", "s")],
        [("content", "matches", r"caf. r.sum. \S dragon$")], [("content", "matches", r"(?m)^line2")], [("content", "matches", "^$")],
        [("Subject", "contains", "résumé")], [("Subject", "matches", "RÉSUMÉ$")], [("content", "matches", r"docker.*kubernetes")],
        [("Priority", "=", "high")], [("nokey", "=", "")], [("", "contains", "emptykey")],
        [("Tags", "has_tag", "huge")], [("Subject", "=", "big one")], [("Filler", "startswith", "xxx")], [("filler", "endswith", "xx")],
    ]
    for conds in cases:
        pb = ProgramBuilder(); pb.add_query(_search_prog(conds))
        checks.append((conds, pb.build(), mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in conds])))
    # "any header value" slots (mode 2: the legacy substring search, utils.py:333-336): OR over the values of the headers
    # dict -- a repeated key only counts with its last value -- through the directory walk and the in-scan text parser
    for q in ["python", "a,b", "lower", "final", "big one", "x" * 300, "", "spaced out", "emptykey", "huge"]:
        pb = ProgramBuilder(); pb.add_query([Cond(C_SLOT, pattern=Pattern("contains", q), field="", mode=2)])
        checks.append((q, pb.build(), [i for i, m in enumerate(mems) if any(q in v.lower() for v in m["headers"].values())]))
    for load, c in _three_loads(recs).items():
        for what, prog, want in checks:
            for leg, masks in _scan_legs(c, prog).items():
                assert np.nonzero(masks)[0].tolist() == want, (load, leg, what)


def _dict_value(headers, field, mode):
    """The value of `field` in the headers dict (None: absent): mode 0 the first key whose lower() equals the field
    (oracle.memdir_oracle.lookup without the date parse), mode 1 headers.get(field)."""
    if mode == 1:
        return headers.get(field)
    return next((v for k, v in headers.items() if k.lower() == field.lower()), None)


def test_slot_values_follow_the_headers_dict(gpu):
    """Corpus.slot_values on every way a header can be read, the > 64 KiB header included: fields repeated in several
    spellings, missing, empty and longer than a value column."""
    recs, mems = _adversarial_records()
    for load, c in _three_loads(recs).items():
        for field in ["Tags", "tags", "TAGS", "Subject", "subject", "Status", "Key", "Priority", "Filler", "nokey", ""]:
            for mode in (0, 1):
                pb = ProgramBuilder(); pb.add_query([Cond(C_SLOT, pattern=Pattern("regex", "", 0), field=field, mode=mode)])
                present, off, blob = c.slot_values(pb.build())
                got = [blob[int(off[i]):int(off[i + 1])].tobytes().decode() if present[i] else None for i in range(len(recs))]
                assert got == [_dict_value(m["headers"], field, mode) for m in mems], (load, field, mode)


def test_filter_semantics_negate_and_missing(corpus3k):
    """MemoryFilter.matches: exact-case header keys, negate, missing fields (filter.py:67-109)."""
    c, arrays, mems = corpus3k
    filters = [
        [("Tags", r"python", False), ("content", r"python|django|flask", True)],
        [("Tags", r"ai|machine[- ]learning|neural|llm", False)],
        [("Tags", r"books|reading|learning", False), ("Subject", r"books|read|learning", False)],
        [("Priority", r"high", False)], [("Status", r"completed|done|archived", False)], [("Tags", r"trash|delete|remove", False)],
        [("Nope", r"x", True)], [("Nope", r"x", False)], [("tags", r"python", False)], [("Author", r"^j", True)], [("flags", r"f", False)],
    ]
    pb = ProgramBuilder()
    for conds in filters:
        cl = []
        for f, p, neg in conds:
            pat = Pattern("regex", p, re.IGNORECASE)
            if f == "content":
                cl.append(Cond(C_BODY, pattern=pat, negate=neg))
            elif f == "flags":
                cl.append(Cond(C_SLOT, pattern=pat, negate=neg, field=f, mode=1, if_missing=2))
                cl.append(Cond(C_FLAGS, pattern=pat, negate=neg))
            else:
                cl.append(Cond(C_SLOT, pattern=pat, negate=neg, field=f, mode=1, if_missing=1 if neg else 0))
        pb.add_query(cl)
    masks = c.scan_masks(pb.build())
    for q, conds in enumerate(filters):
        want = [i for i, m in enumerate(mems) if mo.filter_accepts(m, [{"field": f, "pattern": p, "negate": n} for f, p, n in conds])]
        assert np.nonzero(masks >> np.uint32(q) & np.uint32(1))[0].tolist() == want, conds


def test_empty_and_tiny_corpora(gpu):
    """n = 0, n = 1, empty bodies / headers, 32 queries in one program."""
    from fei_b200.corpus import Corpus
    prog = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in BATCH32])
    empty = Corpus().load(synth.arrays_from_records([]))
    assert empty.scan_masks(prog).size == 0
    assert [h.tolist() for h in empty.scan_hits(prog, 32)] == [[]] * 32
    pb = ProgramBuilder(); pb.add_query(_search_prog([("Tags", "has_tag", "python"), ("flags", "has_flag", "F")]))
    assert empty.scan_count(pb.build(), 1).tolist() == [0]
    r = synth.record(3, 0); r["hdr"] = b""; r["body"] = b""
    one = Corpus().load(synth.arrays_from_records([r]))
    pb = ProgramBuilder()
    pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "", re.IGNORECASE))])            # matches the empty body
    pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "x", re.IGNORECASE))])
    pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "^$", re.IGNORECASE))])
    pb.add_query(_search_prog([("Status", "=", "")]))                                     # headers.get("Status", "") == ""
    pb.add_query(_search_prog([("Tags", "contains", "")]))                                # missing header -> None -> False
    pb.add_query([])                                                                       # no conditions: matches everything
    assert int(one.scan_masks(pb.build())[0]) == 0b101101


def test_hits_capacity_error_and_counts(corpus3k):
    from fei_b200 import _abi
    c, arrays, mems = corpus3k
    pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "python", re.IGNORECASE))])
    prog = pb.build()
    n_hits = int(c.scan_count(prog, 1)[0])
    assert n_hits == len(mo.run_search(mems, [{"field": "content", "operator": "matches", "value": "python"}]))
    with pytest.raises(_abi.FeiCapacityError):
        c.scan_hits(prog, 1, cap=10)
    t = c.timing()
    assert t["kernel_launches"] >= 3 and t["total_ms"] > 0


def test_global_base_offsets_hits(gpu):
    """A shard reports GLOBAL record indices (global_base + local index)."""
    from fei_b200.corpus import Corpus
    a = synth.corpus_arrays(0xFE1, 5000, 300)
    c = Corpus().load(a)
    pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "rust", re.IGNORECASE))])
    hits = c.scan_hits(pb.build(), 1)[0]
    mems = memories_of(a["records"])
    assert hits.tolist() == [5000 + i for i in mo.run_search(mems, [{"field": "content", "operator": "matches", "value": "rust"}])]
    c2 = Corpus().synth(0xFE1, 5000, 300)
    assert c2.scan_hits(pb.build(), 1)[0].tolist() == hits.tolist()


def test_raw_ingest_matches_python_text_semantics(gpu):
    """fei_corpus_load_raw: UTF-8 validation, universal newlines, '---' split and .strip() on the GPU must give
    exactly what open(path, "r").read() + parse_memory_content give (utils.py:229-232, :105-120)."""
    from fei_b200.corpus import Corpus
    raws = [
        b"Subject: a\nTags: x\n---\nbody\n",
        b"Subject: crlf\r\nTags: y\r\n---\r\n\r\n  body line 1\r\nline 2\r\n\r\n",
        b"lone\rcarriage\rreturns---\r\rtext\r",
        b"no separator at all \n just text \t\n",
        b"", b"---", b"------", b"a---b---c", b" \n\t ", b"--- \xc2\xa0\xe2\x80\x83 padded \xe3\x80\x80\n",
        "Ünï: cödé\n---\n  日本語 \U0001F409  ".encode(), b"--", b"-\r\n--", b"x\r\n---\r\ny",
        "h---\x1c\x1d body\x1f\x85".encode(), "İstanbul Σ\n---\nς".encode(), b"k: v\n--- \r",
    ]
    bad = [b"bad \xff byte---x", b"trunc \xe2\x82", b"overlong \xc0\xaf", b"surrogate \xed\xa0\x80", b"too big \xf4\x90\x80\x80", b"cont \x80"]
    recs = []
    for i, raw in enumerate(raws + bad):
        r = synth.record(9, i); r["raw"] = raw
        recs.append(r)
    n = len(recs)

    def arrays(rs):
        off = np.zeros(len(rs) + 1, dtype=np.uint64); np.cumsum([len(r["raw"]) for r in rs], out=off[1:])
        base = synth.arrays_from_records(rs)
        return {"n": len(rs), "raw": np.frombuffer(b"".join(r["raw"] for r in rs) or b"\0", dtype=np.uint8).copy(), "raw_off": off,
                "ts": base["ts"], "wall": base["wall"], "flags8": base["flags8"], "fsb": base["fsb"]}
    c = Corpus()
    valid = c.load_raw(arrays(recs))
    assert valid.tolist() == [True] * len(raws) + [False] * len(bad)
    for raw, ok in zip(raws + bad, valid.tolist()):
        try:
            raw.decode("utf-8"); want = True
        except UnicodeDecodeError:
            want = False
        assert ok == want
    good = recs[:len(raws)]
    assert c.load_raw(arrays(good)).all()
    got = c.fetch(0, len(good))
    bits = (got["fsb"] >> 24).tolist()
    for i, raw in enumerate(raws):
        text = raw.decode("utf-8").replace("\r\n", "\n").replace("\r", "\n")
        head, sep, rest = text.partition("---")
        want_h = (head if sep else "").encode(); want_b = (rest if sep else text).strip().encode()
        h = bytes(got["hdr"][int(got["hdr_off"][i]):int(got["hdr_off"][i + 1])])
        b = bytes(got["body"][int(got["body_off"][i]):int(got["body_off"][i + 1])])
        assert (h, b) == (want_h, want_b), raw
        assert bool(bits[i] & 1) == (not sep) and bool(bits[i] & 2) == (not text.isascii()), raw
        assert bool(bits[i] & 4) == ("Σ" in text) and bool(bits[i] & 8) == ("İ" in text), raw


def test_raw_ingest_fuzz_long_records(gpu):
    """Seeded fuzz of the warp-per-file ingest kernels on files long enough to span many 512-byte rows: multi-byte characters,
    separators, "\r\n" pairs and whitespace runs land on every 16-byte / 512-byte boundary; a third of the files are then
    corrupted (one byte overwritten, or cut inside a character) and must be reported exactly as bytes.decode("utf-8") would."""
    import random
    from fei_b200.corpus import Corpus
    rng = random.Random(20260921)
    toks = ["a", "word ", "--", "---", "-", "\r\n", "\r", "\n", " ", "\t", "\u00a0", "\u2003", "\u3000", "\x85", "é", "日本", "\U0001F409", "Σ", "ς", "İ", "x" * 37,
            "Tags: a,b\n", "\r\n\r\n", " \r\n ", "\x1c", "ß", "-\r\n-"]
    raws = []
    for i in range(400):
        target = rng.choice([0, 1, 15, 16, 17, 31, 33, 100, 511, 512, 513, 700, 1500, 3000, 6000])
        parts, size = [], 0
        if rng.random() < 0.3:
            parts.append(rng.choice([" \r\n\t", "\r\n" * rng.randrange(1, 40), "\u2003" * rng.randrange(1, 200)]))
        while size < target:
            t = rng.choice(toks); parts.append(t); size += len(t.encode())
        if rng.random() < 0.3:
            parts.append(rng.choice(["\r\n" * rng.randrange(1, 300), " \u3000\r", "\n"]))
        raw = "".join(parts).encode()
        k = rng.random()
        if raw and k < 0.2:
            j = rng.randrange(len(raw)); raw = raw[:j] + bytes([rng.choice([0x80, 0xBF, 0xC0, 0xC1, 0xE0, 0xED, 0xF0, 0xF4, 0xF5, 0xFF, 0xA0, 0x9F])]) + raw[j + 1:]
        elif raw and k < 0.33:
            raw = raw[:rng.randrange(len(raw))]
        raws.append(raw)
    recs = []
    for i, raw in enumerate(raws):
        r = synth.record(11, i); r["raw"] = raw
        recs.append(r)

    def arrays(rs):
        off = np.zeros(len(rs) + 1, dtype=np.uint64); np.cumsum([len(r["raw"]) for r in rs], out=off[1:])
        base = synth.arrays_from_records(rs)
        return {"n": len(rs), "raw": np.frombuffer(b"".join(r["raw"] for r in rs) or b"\0", dtype=np.uint8).copy(), "raw_off": off,
                "ts": base["ts"], "wall": base["wall"], "flags8": base["flags8"], "fsb": base["fsb"]}

    def decodes(raw):
        try:
            raw.decode("utf-8"); return True
        except UnicodeDecodeError:
            return False
    c = Corpus()
    valid = c.load_raw(arrays(recs)).tolist()
    want_valid = [decodes(r) for r in raws]
    assert valid == want_valid, [i for i in range(len(raws)) if valid[i] != want_valid[i]][:10]
    assert 40 < sum(not v for v in want_valid) < 200
    good = [r for r, v in zip(recs, want_valid) if v]
    assert c.load_raw(arrays(good)).all()
    got = c.fetch(0, len(good))
    bits = (got["fsb"] >> 24).tolist()
    for i, r in enumerate(good):
        text = r["raw"].decode("utf-8").replace("\r\n", "\n").replace("\r", "\n")
        head, sep, rest = text.partition("---")
        want_h = (head if sep else "").encode(); want_b = (rest if sep else text).strip().encode()
        h = bytes(got["hdr"][int(got["hdr_off"][i]):int(got["hdr_off"][i + 1])])
        b = bytes(got["body"][int(got["body_off"][i]):int(got["body_off"][i + 1])])
        assert (h, b) == (want_h, want_b), (i, r["raw"][:80])
        assert bool(bits[i] & 1) == (not sep) and bool(bits[i] & 2) == (not text.isascii()), i
        assert bool(bits[i] & 4) == ("Σ" in text) and bool(bits[i] & 8) == ("İ" in text), i


def test_staged_text_and_spans_load_equal_plain_load(gpu):
    """fei_corpus_stage_text + fei_corpus_load_raw_spans(raw=NULL): the text uploaded in pieces (any order) and files described by
    (begin, len) spans -- with a gap and in shuffled order -- give the same corpus as the plain one-call load; a size mismatch
    between what was staged and what the spans describe is refused."""
    from fei_b200 import _abi
    from fei_b200.corpus import Corpus
    recs = []
    for i in range(300):
        r = synth.record(21, i); r["raw"] = synth.file_text(r).encode()
        recs.append(r)
    base = synth.arrays_from_records(recs)
    meta = {k: base[k] for k in ("ts", "wall", "flags8", "fsb")}
    lens = np.array([len(r["raw"]) for r in recs], dtype=np.uint64)
    off = np.zeros(len(recs) + 1, dtype=np.uint64); np.cumsum(lens, out=off[1:])
    blob = np.frombuffer(b"".join(r["raw"] for r in recs), dtype=np.uint8).copy()
    plain = Corpus()
    assert plain.load_raw(dict(meta, n=len(recs), raw=blob, raw_off=off)).all()
    want = plain.fetch(0, len(recs))
    # spans: file i lives at a shuffled position behind a 1000-byte gap
    rng = np.random.default_rng(5)
    order = rng.permutation(len(recs))
    begin = np.zeros(len(recs), dtype=np.uint64)
    pos = 1000
    for i in order.tolist():
        begin[i] = pos; pos += int(lens[i]) + (int(i) % 3)
    total = pos
    scattered = np.full(total, ord("-"), dtype=np.uint8)                        # the gaps hold dashes: a reader that strays finds separators
    for i in range(len(recs)):
        scattered[int(begin[i]):int(begin[i] + lens[i])] = np.frombuffer(recs[i]["raw"], dtype=np.uint8)
    spans = Corpus()
    assert spans.load_raw(dict(meta, n=len(recs), raw=scattered, raw_bytes=total, raw_begin=begin, raw_len=lens)).all()
    staged = Corpus()
    cut = [0, total // 3, total // 2, total]
    for a, b in reversed(list(zip(cut, cut[1:]))):                             # pieces in reverse order
        staged.stage_text(total, scattered[a:b], a)
    assert staged.load_raw(dict(meta, n=len(recs), raw=None, raw_bytes=total, raw_begin=begin, raw_len=lens)).all()
    for c in (spans, staged):
        got = c.fetch(0, len(recs))
        for k in ("hdr", "hdr_off", "body", "body_off", "ts", "wall", "flags8", "fsb"):
            assert np.array_equal(got[k], want[k]), k
    pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "python|docker", re.IGNORECASE))])
    assert staged.scan_hits(pb.build(), 1)[0].tolist() == plain.scan_hits(pb.build(), 1)[0].tolist() != []
    bad = Corpus()
    bad.stage_text(total + 8, scattered[:100], 0)
    with pytest.raises(_abi.FeiError):
        bad.load_raw(dict(meta, n=len(recs), raw=None, raw_bytes=total, raw_begin=begin, raw_len=lens))
    with pytest.raises(_abi.FeiError):                                         # a span that leaves the buffer
        bad.load_raw(dict(meta, n=len(recs), raw=scattered, raw_bytes=total - 5000, raw_begin=begin, raw_len=lens))


def _random_header_records():
    """Random key spellings, duplicate keys, odd whitespace (incl. multi-byte), missing colons, colons in values, empty keys / values."""
    import random
    rng = random.Random(4242)
    keys = ["Tags", "tags", "TAGS", "Subject", "subject", "Status", "status", "Priority", "X-Note", "", " Tags", "Tags ", "Ta gs", "Täg", "Key"]
    ws = ["", " ", "  ", "\t", " ", " ", "\x0b", "\x1c", " \t "]
    vals = ["python", "Python, rust", "a,b , c", "", "done", "ACTIVE", "high", "x: y: z", "café", "Kelvin,python", "rust ,python", ",", " , ,", "py thon"]
    recs = []
    for i in range(600):
        lines = []
        for _ in range(rng.randint(0, 7)):
            r = rng.random()
            if r < 0.1:
                lines.append(rng.choice(["no colon here", "", "   ", "---x"[:3 * 0] + "plain"]))
            else:
                lines.append(rng.choice(ws) + rng.choice(keys) + rng.choice(ws) + ":" + rng.choice(ws) + rng.choice(vals) + rng.choice(ws))
        hdr = "\n".join(lines) + ("\n" if lines and rng.random() < 0.7 else "")
        if "---" in hdr:
            hdr = hdr.replace("---", "-")
        body = rng.choice(["", "body python", "react here", "x"])
        r = synth.record(77, i)
        r["hdr"] = hdr.encode(); r["body"] = body.encode(); r["raw_text"] = hdr + "---" + body
        if rng.random() < 0.5:
            r["flags"] = "".join(rng.sample("FRSP", rng.randint(0, 4)))
        recs.append(r)
    mems = [mo.make_memory(r["filename"], r["folder"], r["status"], r["raw_text"], True) for r in recs]
    for m, r in zip(mems, recs):
        m["metadata"]["flags"] = list(r["flags"])
    return recs, mems


def test_random_headers_differential(gpu):
    """Seeded fuzz of the device header parser (k_head_meta / k_head_parse) against the oracle."""
    recs, mems = _random_header_records()
    loads = _three_loads(recs)
    c = loads["default"]
    cases = [
        [("Tags", "has_tag", "python")], [("tags", "has_tag", "rust")], [("TAGS", "contains", "b")], [("Tags", "=", "python")], [("Tags", "has_tag", "")],
        [("Status", "=", "done")], [("state", "=", "active")], [("status_value", "contains", "")], [("Subject", "contains", "y:")], [("", "=", "python")],
        [("x-note", "startswith", "py")], [("priority", "endswith", "gh")], [("Tags", "matches", r"^\w+$")], [("Tags", "matches", r",\s*c$")],
        [("täg", "contains", "")], [("key", "contains", "")], [("Tags", "has_tag", "kelvin")], [("Ta gs", "=", "done")], [("Tags", "!=", "python")],
        [("Tags", "has_tag", "python"), ("flags", "has_flag", "F"), ("content", "contains", "python")],
        [("flags", "has_flag", "SP")], [("flags", "=", "f")], [("flags", "contains", "rs")], [("Priority", ">", "h")], [("Priority", "<=", "high")],
    ]
    pb = ProgramBuilder()
    for conds in cases:
        pb.add_query(_search_prog2(conds))
    masks = c.scan_masks(pb.build())
    for q, conds in enumerate(cases):
        want = mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in conds])
        got = np.nonzero(masks >> np.uint32(q) & np.uint32(1))[0].tolist()
        assert got == want, conds
    # every header path (value columns, directory walk, in-scan text parser), automata in shared or global memory, head
    # pass fused or not: the same masks
    for load, c_alt in loads.items():
        for leg, got in _scan_legs(c_alt, pb.build()).items():
            assert np.array_equal(got, masks), (load, leg)


def test_token_histogram_directory_loads_and_text_refusal(gpu):
    """Corpus.token_histogram of the exact "Tags" header (folders.py:286-292) on the default and FEI_HCOLS=0 loads equals a
    Python count; with every header parsed from its text (FEI_HDIR=0) it is refused."""
    recs, mems = _random_header_records()
    want = {}                                    # token -> [count, first record], in first-occurrence order
    for i, m in enumerate(mems):
        if "Tags" in m["headers"]:
            for tag in [t.strip() for t in m["headers"]["Tags"].split(",")]:
                want.setdefault(tag.encode(), [0, i])[0] += 1
    want = [(t, n, first) for t, (n, first) in want.items()]
    pb = ProgramBuilder(); pb.add_query([Cond(C_SLOT, pattern=Pattern("regex", "", 0), field="Tags", mode=1)])
    loads = _three_loads(recs)
    for load in ("default", "FEI_HCOLS"):
        assert loads[load].token_histogram(pb.build(), ",") == want, load
    with pytest.raises(NotImplementedError):
        loads["FEI_HDIR"].token_histogram(pb.build(), ",")


def _search_prog2(conds):
    """Compile through the product's own query compiler (fei_b200.memdir_tools.search.compile_conditions)."""
    from fei_b200.memdir_tools.search import compile_conditions

    class _PM:                       # only what compile_conditions touches for these fields
        folders = [""]
        arrays = {}
    out = compile_conditions([{"field": f, "operator": op, "value": v} for f, op, v in conds], True, _PM())
    assert all(isinstance(x, Cond) for x in out), out
    return out


def test_sharded_scan_equals_unsharded(gpu):
    """1/2/4/8-way range sharding gives byte-identical hit lists: every shard reports global indices and the
    rank-order concatenation is the listing order (the NCCL all-gatherv moves exactly these lists)."""
    from fei_b200 import shard
    from fei_b200.corpus import Corpus
    n = 4100
    prog = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in BATCH32[:8]] + [Pattern("regex", r"kubernetes.*docker", re.IGNORECASE)])
    whole = Corpus().synth(0xFE1, 0, n).scan_hits(prog, 9)
    for world in (2, 4, 8):
        per_rank = []
        for a, b in shard.shard_ranges(n, world):
            per_rank.append(Corpus().synth(0xFE1, a, b - a).scan_hits(prog, 9))
        got = shard.concat_in_rank_order(per_rank)
        for q in range(9):
            assert np.array_equal(got[q], whole[q]), (world, q)


def test_full_size_corpus_sampled_windows_and_invariants(gpu):
    """BASELINE-scale run (2M entries generated and tiled on the GPU): sampled windows must equal the oracle on the same
    records from the host generator; size-independent invariants hold on the whole result (ordering, counts = popcounts,
    hits ⊆ range, union/intersection consistency between a batch and its single-pattern scans)."""
    from fei_b200.corpus import Corpus
    n = 2_000_000
    c = Corpus().synth(0xFE1, 0, n)
    pats = BATCH32[:6] + [r"kubernetes.*docker|docker.*kubernetes", r"quagga"]
    prog = content_batch_program([Pattern("regex", p, re.IGNORECASE) for p in pats])
    masks = c.scan_masks(prog)
    counts = c.scan_count(prog, len(pats))
    for q in range(len(pats)):
        assert int(counts[q]) == int(((masks >> np.uint32(q)) & np.uint32(1)).sum())
    assert int(counts[len(pats) - 1]) == 0
    hits = c.scan_hits(prog, len(pats))
    for q in range(len(pats)):
        h = hits[q]
        assert h.size == int(counts[q]) and (h.size == 0 or (int(h[0]) >= 0 and int(h[-1]) < n and bool(np.all(h[1:] > h[:-1]))))
        assert np.array_equal(np.nonzero((masks >> np.uint32(q)) & np.uint32(1))[0].astype(np.uint64), h)
    # single-pattern (sticky kernel variant) == its bit in the batch (multi-output variant)
    for q in (0, 6):
        pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", pats[q], re.IGNORECASE))])
        assert np.array_equal(c.scan_hits(pb.build(), 1)[0], hits[q])
    # selective header predicates + one content pattern: few records reach the body pass (k_live_list + k_body_gather, one
    # thread per surviving record); it must equal the intersection of the header-only and the content-only scans (other kernels)
    head_conds = [("Tags", "has_tag", "python"), ("flags", "has_flag", "F")]
    body_cond = ("content", "matches", r"react|angular")
    pb = ProgramBuilder(); pb.add_query(_search_prog(head_conds)); m_head = c.scan_masks(pb.build()) & np.uint32(1)
    pb = ProgramBuilder(); pb.add_query(_search_prog([body_cond])); m_body = c.scan_masks(pb.build()) & np.uint32(1)
    pb = ProgramBuilder(); pb.add_query(_search_prog(head_conds + [body_cond])); m_both = c.scan_masks(pb.build()) & np.uint32(1)
    assert 0 < int(m_head.sum()) < n // 16                              # sparse enough for the gather path
    assert np.array_equal(m_both, m_head & m_body)
    for first in (0, 777_777, n - 1500):
        k = 1500
        recs = [synth.record(0xFE1, first + i) for i in range(k)]
        mems = memories_of(recs)
        for q, p in enumerate(pats):
            want = mo.run_search(mems, [{"field": "content", "operator": "matches", "value": p}])
            got = np.nonzero((masks[first:first + k] >> np.uint32(q)) & np.uint32(1))[0].tolist()
            assert got == want, (first, p)
        want = mo.run_search(mems, [{"field": f, "operator": op, "value": v} for f, op, v in head_conds + [body_cond]])
        assert np.nonzero(m_both[first:first + k])[0].tolist() == want, first


def test_single_pattern_kernel_shapes(gpu):
    """k_body_sticky's code paths: full rows through the TMA ring (pairs of groups, then one group), the joint ragged tail,
    early stop of one / both groups, window boundary (4096), needles at row and chunk edges, NUL bytes and bytes whose
    stored form differs (the tile byte substitution), empty bodies."""
    from fei_b200.corpus import Corpus
    rng = np.random.default_rng(20260921)
    words = [b"alpha", b"Beta", b"GAMMA", b"delta", b" ", b"\n", b"_", b"@", b"`", b"{", b"\x00", "é".encode(), "Ω".encode(), b"1234", b"~"]

    def filler(n):
        out = bytearray()
        while len(out) < n:
            out += words[int(rng.integers(len(words)))]
        return bytes(out[:n]).decode("utf-8", "ignore").encode()     # keep it valid UTF-8 after the cut

    recs = []
    n = 4096 + 70                                                     # second window: 70 records, 3 groups, padded lanes
    for i in range(n):
        r = synth.record(11, i)
        kind = i % 8
        if kind == 0:
            ln = 1024                                                 # equal lengths, multiples of 16: no ragged rows at all
        elif kind == 1:
            ln = 0
        elif kind == 2:
            ln = int(rng.integers(1, 48))                             # shorter than one chunk: tail loop only
        else:
            ln = int(rng.integers(900, 1400))
        body = bytearray(filler(ln))
        ln = len(body)
        where = i % 11
        needle = b"NeEdLe"
        pos = None
        if ln >= 16 and where < 8:                                    # 3 of 11 records carry no needle
            pos = [0, ln - len(needle), 10, 16 - 3, 512 - 2, 1024 - 6 if ln >= 1024 else ln // 2, ln // 2, ln // 3][where]
            pos = max(0, min(pos, ln - len(needle)))
            body[pos:pos + len(needle)] = needle
        try:
            body.decode("utf-8")
        except UnicodeDecodeError:                                    # the needle cut a multi-byte character: repair the neighbours
            body = bytearray(bytes(body).decode("utf-8", "replace").replace("�", "?").encode())
        if body and body[:1] in (b" ", b"\n"):                        # bodies are stored stripped (utils.py:120)
            body[0:1] = b"x"
        if body and body[-1:] in (b" ", b"\n"):
            body[-1:] = b"x"
        r["body"] = bytes(body)
        recs.append(r)
    # one group where every record matches in its first row (both groups of a pair stop at once)
    for i in range(64):
        recs[2048 + i]["body"] = b"needle " + filler(1100).rstrip() + b"."
    a = synth.arrays_from_records(recs)
    c = Corpus().load(a)
    mems = memories_of(recs)
    got = c.fetch(0, n)
    assert bytes(got["body"][:int(a["body_off"][-1])]) == bytes(a["body"][:int(a["body_off"][-1])])
    for p in ["needle", r"^needle", r"needle\Z", r"alpha.*needle|needle.*delta", "absent-everywhere", r"\x00", "é", r"[`{@~_]needle", "(?s).", r"\Aalpha"]:
        pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", p, re.IGNORECASE))])
        want = mo.run_search(mems, [{"field": "content", "operator": "matches", "value": p}])
        assert c.scan_hits(pb.build(), 1)[0].tolist() == want, p
    pb = ProgramBuilder(); pb.add_query([Cond(C_BODY, pattern=Pattern("regex", "NeEdLe", 0))])      # case-sensitive: upper/lower columns differ
    want = [i for i, m in enumerate(mems) if re.search("NeEdLe", m["content"])]
    assert c.scan_hits(pb.build(), 1)[0].tolist() == want
