"""Model of the row kernel's key path (DESIGN.md 3.1, step 3): B' columns renumbered by (colB, column id), the exact
k-th-smallest-key cut, the key-valued dominance frontier with first_key_of_cb, the A'^T A' diagonal, and rows that fall
back to the colB path.  It must return exactly the brute-force top-k, and evaluate no more cells than the colB cut."""
import os
import random
import sys

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools", "proto"))


def test_column_order_and_first_key_table():
    import cut_model
    rng = random.Random(1)
    marg = {b: rng.choice([1, 1, 2, 3, 7, 7, 7, 40]) for b in rng.sample(range(1000), 300)}
    key_of_col, col_of_key, marg_key, first = cut_model.column_order(marg)
    assert [key_of_col[b] for b in col_of_key] == list(range(len(marg)))
    assert all((marg_key[i], col_of_key[i]) < (marg_key[i + 1], col_of_key[i + 1]) for i in range(len(marg) - 1))
    for c in range(max(marg.values()) + 2):
        for key in range(len(marg)):
            assert (key >= first[c]) == (marg_key[key] >= c)


def test_key_path_model_is_exact(orc):
    import cut_model
    import select_model
    rng = random.Random(5)
    stats_key, stats_cut = {}, {}
    for t in range(600):
        cells, ra, n = (cut_model.tied_row if t % 2 else select_model.random_row)(rng)
        k = rng.choice([1, 5, 50, 200])
        min_llr = rng.choice([None, None, 0.5])
        item, self_ = rng.randrange(0, 5000), rng.random() < 0.3
        want = select_model.brute(cells, ra, n, k, min_llr, item, self_)
        assert cut_model.key_path(cells, ra, n, k, min_llr, item, self_, stats=stats_key) == want, t
        assert cut_model.level1_cut(cells, ra, n, k, min_llr, item, self_, stats=stats_cut) == want, t
    assert stats_key["keyed"] > 100 and stats_key["fallback"] > 100
    assert stats_key["evals"] <= stats_cut["evals"]
