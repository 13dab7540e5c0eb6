"""The maintenance methods of MemoryArchiver have the reference's signatures (recorded in the goldens), without a GPU."""
import inspect

from tests import maintenance_tree as T
from tests.conftest import load_golden


def test_signatures_match_reference():
    from fei_b200.memdir_tools.archiver import MemoryArchiver
    want = load_golden("maintenance_golden.json")["signatures"]
    assert set(want) == set(T.METHODS)
    for name, sig in want.items():
        assert str(inspect.signature(getattr(MemoryArchiver, name), eval_str=True)) == sig, name
