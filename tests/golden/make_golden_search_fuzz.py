"""Write tests/golden/search_fuzz_golden.json from the reference's search_memories (memdir_tools/search.py).

Run on a machine that has the reference project:  python tests/golden/make_golden_search_fuzz.py /path/to/reference

The tree is tests/search_fuzz.py's fuzz tree; the queries are the first N_QUERIES of search_fuzz.random_query's stream (seed SEED)
whose outcome does not depend on today's date (search_fuzz.depends_on_today).  For each the golden records the query's repr and
either the result keys and whether "Unable to sort" was printed, or the exception type and message.  The reference reads the tree
with os.walk / os.listdir sorted (search_fuzz.sorted_fs), so the listing order, and with it the record that raises first, does not
depend on the file system.  One query per line."""
import contextlib
import io
import json
import os
import random
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
os.environ["TZ"] = "UTC"
time.tzset()

from tests import search_fuzz as F          # noqa: E402

SEED = 0x60DE
N_QUERIES = 300


def sample():
    """The golden's queries: the first N_QUERIES today-independent queries of the seeded stream."""
    rng, vocab, out = random.Random(SEED), F.tree_vocab(), []
    while len(out) < N_QUERIES:
        q = F.random_query(rng, vocab)
        if not F.depends_on_today(q):
            out.append(q)
    return out


def main(reference: str) -> None:
    sys.path.insert(0, reference)
    import memdir_tools.search as rs
    import memdir_tools.utils as ru
    assert rs.__file__.startswith(os.path.abspath(reference)), rs.__file__
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        base = os.path.join(tmp, "Memdir")
        F.build_fuzz_tree(base)
        ru.MEMDIR_BASE = base
        for q in sample():
            conds, include_content, folders, statuses, sort, reverse, limit, offset = q
            sq = rs.SearchQuery()
            for f, op, v in conds:
                sq.add_condition(f, op, v)
            sq.with_content(include_content)
            if sort:
                sq.set_sort(sort, reverse)
            sq.set_pagination(limit, offset)

            def run():
                buf = io.StringIO()
                with contextlib.redirect_stdout(buf), F.sorted_fs():
                    res = rs.search_memories(sq, folders, statuses)
                return res, buf.getvalue()
            lines.append(json.dumps({"query": repr(q), **F.outcome(run)}, ensure_ascii=False))
    with open(os.path.join(HERE, "search_fuzz_golden.json"), "w") as f:
        f.write('{"seed": %d, "tree_seed": %d, "queries": [\n' % (SEED, F.SEED) + ",\n".join(lines) + "\n]}\n")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_search_fuzz.py <directory holding the reference's memdir_tools package>")
    main(sys.argv[1])
