"""The oracle's search on the fuzz tree (tests/search_fuzz.py) against the reference-generated golden
(tests/golden/search_fuzz_golden.json), without a GPU: the same result keys in the same order, the same "Unable to sort"
warning, or the same exception type and message.  Both read the tree with sorted directory listings."""
import pytest

from tests import search_fuzz as F
from tests.conftest import load_golden
from tests.golden.make_golden_search_fuzz import SEED, sample


@pytest.fixture(scope="module")
def fuzz(tmp_path_factory):
    base = str(tmp_path_factory.mktemp("search_fuzz") / "Memdir")
    F.build_fuzz_tree(base)
    return base, load_golden("search_fuzz_golden.json")


def test_golden_covers_the_generated_sample(fuzz):
    _base, g = fuzz
    assert (g["seed"], g["tree_seed"]) == (SEED, F.SEED)
    assert [w["query"] for w in g["queries"]] == [repr(q) for q in sample()]
    kinds = [("raises" in w, bool(w.get("keys")), w.get("unable_to_sort", False)) for w in g["queries"]]
    assert any(k[0] for k in kinds) and any(k[1] for k in kinds) and any(k[2] for k in kinds)
    assert any(w.get("raises", [None])[0] == "OverflowError" for w in g["queries"])


def test_oracle_search_matches_reference(fuzz):
    base, g = fuzz
    cache, bad = {}, []
    with F.sorted_fs():
        for q, want in zip(sample(), g["queries"]):
            got = F.oracle_search(base, q, cache)
            want = {k: v for k, v in want.items() if k != "query"}
            if got != want:
                bad.append((q, got, want))
    assert not bad, "\n".join(f"query={q!r}\n  oracle={got}\n  reference={want}" for q, got, want in bad[:10])
