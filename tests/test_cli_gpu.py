"""The Memdir command line on the GPU (fei_b200.memdir_tools.cli, search.main, Corpus.format_records) against the reference
goldens (tests/golden/cli_golden.json) and against tests/cli_expect.py's formatting of the oracle's dicts: every golden argv
replayed on a fresh golden tree gives the same stdout bytes and the same tree afterwards; seeded random records with awkward
text format byte-exactly in all four formats; a base corpus with a delta formats in listing order across several device calls;
a record with an 8 MiB body is viewed whole."""
import base64
import contextlib
import io
import os
import random
import sys

import numpy as np
import pytest

from tests import cli_expect as X
from tests.conftest import load_golden
from tests.memdir_util import build_tree

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return load_golden("cli_golden.json")


@pytest.fixture
def fresh(gpu, tmp_path, monkeypatch):
    from fei_b200 import packer
    from fei_b200.memdir_tools import utils as U
    bases = []

    def make(name, build=build_tree):
        base = str(tmp_path / name / "Memdir")
        build(base)
        monkeypatch.setattr(U, "MEMDIR_BASE", base)
        bases.append(base)
        return base
    yield make
    for b in bases:
        packer.drop(b)


def run_main(fn, argv, encoding="utf-8", errors="surrogateescape"):
    buf = io.BytesIO()
    out = io.TextIOWrapper(buf, encoding=encoding, errors=errors, newline="\n", write_through=True)
    old = sys.argv
    sys.argv = argv
    exc = None
    try:
        with contextlib.redirect_stdout(out):
            fn()
    except Exception as e:
        exc = e
    finally:
        sys.argv = old
    out.flush()
    return buf.getvalue(), exc


@pytest.mark.parametrize("k", range(51))
def test_cli_replays_reference_goldens(golden, fresh, k):
    from fei_b200.memdir_tools import cli, search
    from fei_b200.memdir_tools import utils as U
    case = golden["cases"][k]
    base = fresh(f"case{k}")
    U.ensure_memdir_structure()
    same_ties = X.tie_groups(base) == golden["ties"]
    before = X.tree_files(base)
    got, exc = run_main(cli.main if case["kind"] == "cli" else search.main, [case["kind"]] + case["argv"])
    assert (type(exc).__name__ if exc else None) == case["exception"], exc
    if "stdout" in case and same_ties:
        assert got == base64.b64decode(case["stdout"])
    d = X.digest(got)
    assert d["bytes"] == case["bytes"]
    if same_ties:
        assert d["sha256"] == case["sha256"]
    else:                                   # records with equal timestamps listed in another os.listdir order on this file system
        assert d["sha256_lines"] == case["sha256_lines"]
    if "tree" in case:
        assert X.tree_change(before, X.tree_files(base)) == case["tree"]
    if case["argv"][0] in ("list", "view") and case["kind"] == "cli":
        assert got == (X.list_cmd if case["argv"][0] == "list" else X.view_cmd)(base, case["argv"])


# ----------------------------------------------------------------------------- seeded random records
_PIECES = ["plain", "é ü", "\U0001F409", " x", "tab\there", 'q"uo\\te', "\x01\x1f\x7f", " padded ", "", "İΣ", "日本"]


def _rand_text(rng, n=3):
    return "".join(rng.choice(_PIECES) for _ in range(rng.randint(0, n)))


def _random_tree(base, seed, n=300):
    rng = random.Random(seed)
    folders = ["", ".Projects/AI", ".Archive"]
    for f in folders:
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(base, f, st), exist_ok=True)
    for i in range(n):
        lines = []
        for _ in range(rng.randint(0, 6)):
            key = rng.choice(["Subject", "Tags", "Priority", "Status", " Subject ", "subject", "X-" + _rand_text(rng, 1), ""])
            lines.append(rng.choice([f"{key}: {_rand_text(rng)}", f"{key}:{_rand_text(rng)}", _rand_text(rng), f"{key}:"]))
        head = "\n".join(lines)
        body = _rand_text(rng, 6) + "\nline two " + _rand_text(rng)
        text = rng.choice([f"{head}\n---\n{body}", body, f"{head}\n---\n{body}".replace("\n", "\r\n")])
        flags = "".join(rng.sample("FPRS", rng.randint(0, 4))) + rng.choice(["", "", "ABC"])
        host = rng.choice([b"hostA", b"h\xc3\xa9st", b"bad\xffhost", b"h\xed\xa0\x80x"])
        name = b"%d.r%07d." % (1700000000 + rng.randint(0, 10 ** 6), i) + host + b":2," + flags.encode()
        d = os.path.join(base, rng.choice(folders), rng.choice(["cur", "new", "tmp"]))
        with open(os.path.join(os.fsencode(d), name), "wb") as fh:
            fh.write(text.encode("utf-8"))


def _with_content(m, content):
    return m if content else {k: v for k, v in m.items() if k != "content"}


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_format_records_matches_oracle_dicts(fresh, seed):
    from fei_b200 import _abi, packer
    base = fresh(f"rand{seed}", lambda b: _random_tree(b, seed))
    pm = packer.packed(base)
    with pm.lock, contextlib.redirect_stdout(io.StringIO()):
        positions = np.arange(pm.n)
        mems = {}
        for (f, st), (a, b) in pm.segments.items():
            for p, m in zip(range(a, b), X.mo.read_folder(base, f, st, True)):
                mems[p] = m
        rng = np.random.default_rng(seed)
        order = rng.permutation(positions)
        for fmt, code in (("json", _abi.FEI_FMT_JSON), ("csv", _abi.FEI_FMT_CSV), ("compact", _abi.FEI_FMT_COMPACT), ("text", _abi.FEI_FMT_TEXT)):
            for content in (False, True):
                opts = _abi.FEI_FMT_CONTENT if content else 0
                got = b"".join(d for d, _ in pm.format_records(order, code, opts))
                want = b"".join(X.record(_with_content(mems[int(p)], content), fmt, content) for p in order)
                assert got == want, (fmt, content)
        # JSON items against json.dumps of the dicts pm.materialize builds, dates converted as the reference does
        items = []
        for d, off in pm.format_records(order, _abi.FEI_FMT_JSON, _abi.FEI_FMT_CONTENT):
            items += [d[off[k]:off[k + 1]] for k in range(len(off) - 1)]
        assert items == X.json_items(pm.materialize(order, True))


def test_text_raises_where_print_raises_on_a_strict_stream(fresh):
    from fei_b200.memdir_tools import cli
    base = fresh("strict", lambda b: _random_tree(b, 7, 40))
    name = next(n for n in os.listdir(os.path.join(os.fsencode(base), b"cur")) if b"\xff" in n)
    mid = name.split(b".")[1].decode()
    got, exc = run_main(cli.main, ["cli", "view", mid], encoding="ascii", errors="strict")
    assert isinstance(exc, UnicodeEncodeError)
    assert got == X.enc(X.colorize(f"Memory ID: {mid}", "bold") + "\n")     # the line before File:, nothing of File:


def test_delta_corpus_and_small_chunks(fresh, monkeypatch):
    """Files added and renamed after the first pack land in the delta corpus: listings interleave base and delta records, and
    with the chunk budget lowered one listing takes several device calls and the capacity path."""
    from fei_b200 import _abi, packer
    from fei_b200.memdir_tools import cli
    base = fresh("delta", lambda b: _random_tree(b, 11, 400))
    pm = packer.packed(base)
    cur = os.path.join(os.fsencode(base), b"cur")
    names = sorted(os.listdir(cur))
    for n in names[:20:2]:                                           # renames and new files after the first pack
        os.rename(os.path.join(cur, n), os.path.join(cur, n.replace(b".r", b".z", 1)))
    for k in range(15):
        with open(os.path.join(cur, b"%d.n%07d.hostA:2," % (1700400000 + 37 * k, k)), "w") as fh:
            fh.write(f"Subject: new {k}\n---\nbody {k}")
    pm = packer.packed(base)
    assert pm.delta is not None and pm.delta.n > 0
    calls = []
    real = type(pm.corpus).format_records

    def spy(self, idx, fmt, opts, names, cap=None):
        data, off = real(self, idx, fmt, opts, names, cap)
        calls.append(data is None)
        return data, off
    monkeypatch.setattr(type(pm.corpus), "format_records", spy)
    monkeypatch.setattr(packer, "FORMAT_CHUNK_BYTES", 4096)
    got, exc = run_main(cli.main, ["cli", "list", "-c", "--json"])
    assert exc is None
    assert got == X.list_cmd(base, ["list", "-c", "--json"])
    assert len(calls) > 4 and any(calls)


def test_view_of_an_8_mib_body(fresh):
    from fei_b200.memdir_tools import cli

    def build(b):
        for st in ("cur", "new", "tmp"):
            os.makedirs(os.path.join(b, st))
        rng = random.Random(5)
        body = "".join(rng.choice(["word ", "ü", "\"q\"\n", "\U0001F409"]) for _ in range(3 << 20))[: 8 << 20]
        with open(os.path.join(b, "cur", "1700000000.big00001.hostA:2,F"), "w") as fh:
            fh.write("Subject: big\n---\n" + body)
    base = fresh("big", build)
    got, exc = run_main(cli.main, ["cli", "view", "big00001"])
    assert exc is None and len(got) > 8 << 20
    assert got == X.view_cmd(base, ["view", "big00001"])
