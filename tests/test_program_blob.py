"""The content automaton as a program blob carries it (CPU suite): serialize_dfa renumbers the states so that accepting ones
come first, permutes the columns (or the class table) by the tile byte substitution, pads the rows and writes the sticky
marker.  A model of the scan kernels' stepping (tests/blob_model.py) run over that blob must agree with CPython's re,
for byte-indexed and class-indexed tables alike."""
import random
import re

import pytest

from fei_b200.program import SMEM_TABLE_LIMIT, serialize_dfa
from fei_b200.regexc import Pattern, PatternTooLarge, compile_patterns
from tests.blob_model import BlobDfa
from tests.test_regexc_fuzz import ALPHABET, rand_regex

TEXT_ALPHABET = ALPHABET + ["Σ", "σ", "ς", "İ", "@", "`", "[", "{", "\0", "Z"]


def _layouts(pats):
    d = compile_patterns([Pattern("regex", p, re.IGNORECASE) for p in pats], sticky=True)
    models = []
    for limit in (SMEM_TABLE_LIMIT, 0):
        blob = bytearray(b"\0" * 32)                              # a descriptor never sits at offset 0 of a program
        off = serialize_dfa(d, blob, limit, tile_bytes=True)
        models.append(BlobDfa(bytes(blob), off))
    return models


@pytest.mark.parametrize("seed", range(2))
def test_serialized_automaton_agrees_with_re(seed):
    rng = random.Random(1000 + seed)
    layouts = set()
    checked = 0
    for _ in range(40):
        k = rng.choice([1, 3, 6])
        pats = []
        while len(pats) < k:
            p = rand_regex(rng)
            try:
                re.compile(p, re.IGNORECASE)
                pats.append(p)
            except re.error:
                pass
        try:
            models = _layouts(pats)
        except PatternTooLarge:
            continue
        assert models[1].n_cols < 256
        for m in models:
            assert m.sticky != 0 if k == 1 else m.sticky == 0
            assert m.n_patterns == k
            layouts.add((m.direct, k == 1))
        for _ in range(30):
            t = "".join(rng.choice(TEXT_ALPHABET) for _ in range(rng.randint(0, 16)))
            raw = t.encode("utf-8")
            want = sum(1 << j for j, p in enumerate(pats) if re.search(p, t, re.IGNORECASE))
            for m in models:
                assert m.run(raw) == want, (pats, t, m.direct)
                checked += 1
    assert layouts == {(True, True), (False, True), (True, False), (False, False)}
    assert checked > 1500
