"""Sorted rows of `k_rows` (DESIGN.md 3.1): warp-owned hashed bins whose rows are all keyed with an exact cut gather a
row's keys, radix-sort them in the warp and read the counts, the compacted cells and the level-1 key cut off the runs of
equal keys.  Each case is checked bit for bit against the brute force of tests/rowref.py and against the oracle, and
asserts through `sorted_bins` (a restatement of `use_sorted` and its caller in cco_api.cu) which rows took the path."""
import numpy as np
import pytest

import row_paths
import rowref
from test_gpu_bitmap_rows import ramp, run, shaped, singles_row

pytestmark = pytest.mark.gpu
M_ALL = 10 ** 9
N_COLS = 70_001          # 17-bit keys: two 9-bit digits


def sort_digits(n_cols_b: int):
    """(passes, histogram words per digit): cco_kernels.cuh sort_digits."""
    kb = 32 - row_paths.count_bits(n_cols_b)
    passes = (kb + 8) // 9
    dbits = max(-(-kb // passes), 6)
    return passes, 1 << (dbits - 1)


def sorted_bins(top_k: int, n_cols_b: int, max_marg_a: int, max_marg_b: int, n_users: int) -> set:
    """Bins that run sorted rows (cco_api.cu: `bitmap_ok` in enqueue_indicator, then `use_sorted` per bin)."""
    if not (row_paths.cut_exact(n_users, max_marg_a, max_marg_b) and 2 * max_marg_a * max_marg_b < n_users):
        return set()
    cfgs, h_thr = row_paths.bins(top_k, n_cols_b)
    passes, hwords = sort_digits(n_cols_b)
    out = set()
    for b in range(1, len(cfgs)):
        f, max_w = cfgs[b], h_thr[b - 1]
        if f.dense or f.group != 32 or max_w > 1024 or max(2 * max_w - 320, max_w) > f.slots:
            continue
        if passes * hwords <= 4 * f.cbuf:                                        # digit histograms in the candidates
            out.add(b)
    return out


def sorted_rows(e: rowref.Expected) -> list:
    """Per output row: True (sorted row), False (another path) or None (no work)."""
    bins = sorted_bins(e.top_k, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users)
    return [None if p is None else p.bin in bins for p in e.paths()]


def test_warp_bins_are_sorted_at_c3_and_c4_widths():
    # 100 K columns (two 9-bit digits) and 1 M columns (three 7-bit digits) at top_k 50, as in the C3 and C4 workloads
    assert sort_digits(100_000) == (2, 256) and sort_digits(1_000_000) == (3, 64)
    for n_cols in (100_000, 1_000_000):
        assert sorted_bins(50, n_cols, 600, 600, 10 ** 6) == {5, 6, 7}
    assert sorted_bins(50, 100_000, 600, 600, 700_000) == set()                  # 2 rowA colB >= N: not keyed
    assert sorted_bins(50, 300, 600, 600, 10 ** 6) == set()                      # dense warp bins


def test_row_sizes(orc, ctx):
    from test_gpu_row_paths import work_rows
    works = [1, 31, 32, 33, 256, 257, 512, 513, 1024]
    mats = work_rows(works, N_COLS, True, seed=21)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "row sizes")
    assert sorted_rows(exp[1]) == [True] * len(works)
    assert [p.bin for p in exp[1].paths()] == [7, 7, 7, 7, 7, 6, 6, 5, 5]


def test_every_product_on_one_key(orc, ctx):
    # one cell per row: k11 = w (1, 33, 256, 1024 products), at the smallest key, a digit edge and the largest key
    items = [{0: 1}, {511: 33}, {512: 256}, {N_COLS - 1: 1024}]
    colb = np.ones(N_COLS, dtype=np.int64)
    colb[[511, 512, N_COLS - 1]] = [33, 256, 1024]
    mats = shaped(items, N_COLS, colb, n_users=3_000_000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "one key")
    assert sorted_rows(exp[1]) == [True] * 4
    assert exp[1].count.tolist() == [1, 33, 256, 1024]


def test_all_keys_distinct(orc, ctx):
    # every cell k11 = 1: 1000, 300 and 40 singles (the last fewer than top_k)
    rng = np.random.default_rng(4)
    items = [{int(c): 1 for c in rng.choice(N_COLS, n, replace=False)} for n in (1000, 300, 40)]
    mats = shaped(items, N_COLS, ramp(N_COLS, 3, 12), n_users=1000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "distinct")
    assert sorted_rows(exp[1]) == [True] * 3
    assert np.diff(exp[1].row_ptr).tolist() == [50, 50, 40]


@pytest.mark.parametrize("n_singles", [49, 50, 51])
def test_singles_around_top_k(orc, ctx, n_singles):
    # fewer than, exactly and one more than top_k singles, below repeated cells of a larger colB
    items = [singles_row(range(100, 100 + n_singles), w, 20_000) for w in (1000, 200)]
    colb = ramp(N_COLS, 2, 3)
    colb[20_000:] = 150
    mats = shaped(items, N_COLS, colb, n_users=1000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, f"{n_singles} singles")
    e = exp[1]
    assert sorted_rows(e) == [True] * 2
    for r in range(2):
        got = e.col[e.row_ptr[r]:e.row_ptr[r + 1]]
        assert got[:min(n_singles, 50)].tolist() == list(range(100, 100 + min(n_singles, 50)))


@pytest.mark.parametrize("kth", [255, 256, 511, 512])
def test_top_k_th_single_at_a_digit_edge(orc, ctx, kth):
    # the 50th smallest single key at the last / first key of a radix digit (8-bit and 9-bit edges); the repeated
    # cells (colB 150) rank below every kept single, so the kept cells are exactly the 50 smallest singles
    first = kth - 49
    singles = list(range(first, kth + 1)) + list(range(kth + 300, kth + 600))
    items = [singles_row(singles, 1000, 60_000), singles_row(singles[:200], 500, 60_000)]
    colb = ramp(N_COLS, 2, 3)
    colb[60_000:] = 150
    mats = shaped(items, N_COLS, colb, n_users=1000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, f"kth single {kth}")
    e = exp[1]
    assert sorted_rows(e) == [True, True]
    for r in range(2):
        assert e.col[e.row_ptr[r]:e.row_ptr[r + 1]].tolist() == list(range(first, kth + 1))


def test_colb_ties_straddle_the_cut(orc, ctx):
    # colB runs of 40 equal values that fall as the column id rises; the 50th single sits inside a run
    colb = np.minimum(2 + (N_COLS - 1 - np.arange(N_COLS)) // 40, 12)
    colb[1000:6000] = 150
    tail = np.arange(N_COLS - 400, N_COLS)
    items = [singles_row(tail.tolist(), 1000, 1000), singles_row(tail[::2].tolist(), 600, 1000)]
    mats = shaped(items, N_COLS, colb, n_users=1000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "colB ties")
    e = exp[1]
    assert sorted_rows(e) == [True, True]
    assert e.col[e.row_ptr[0]:e.row_ptr[1]].tolist() == list(range(N_COLS - 40, N_COLS)) + \
        list(range(N_COLS - 80, N_COLS - 70))


def test_self_diagonal_as_single_and_as_repeat(orc, ctx):
    # A'^T A': users 0 and 1 buy 400 items each, 100 in common.  A common item's row has 800 products and its diagonal
    # k11 = 2; an item of one user has 400 products, all k11 = 1, its diagonal a single
    from test_gpu_row_paths import csr
    rng = np.random.default_rng(5)
    items = rng.permutation(N_COLS)[:700]
    common, own0, own1 = items[:100], items[100:400], items[400:700]
    rows = [sorted(np.concatenate([common, own0]).tolist()), sorted(np.concatenate([common, own1]).tolist())]
    m = csr(rows, N_COLS, 1000)
    exp, got = run(orc, ctx, [m, m], [(M_ALL, 50, None), (M_ALL, 50, None)], "self diagonal")
    for e in exp:
        sr = sorted_rows(e)
        assert all(sr[i] for i in common) and all(sr[i] for i in own0)
    for i in (int(common[0]), int(own0[0])):
        kept = got[0][4][exp[0].row_ptr[i]:exp[0].row_ptr[i + 1]]
        assert i not in kept.tolist() and len(kept) == 50


def test_min_llr(orc, ctx):
    items = [singles_row(list(range(0, 900, 3)), 1000, 10_000), singles_row(list(range(5, 400, 2)), 300, 10_000)]
    mats = shaped(items, N_COLS, ramp(N_COLS, 4, 12), n_users=1000)
    base = rowref.expected(ctx, mats, [(M_ALL, 50, None)] * 2, 1)[1]
    for row, rank in ((0, 30), (1, 49)):
        t = float(base.llr[base.row_ptr[row] + rank])
        exp, got = run(orc, ctx, mats, [(M_ALL, 50, t)] * 2, f"minLLR={t!r}")
        assert sorted_rows(exp[1]) == [True, True]
        assert (got[1][5] >= t).all() and (got[1][5] == t).any()


def test_three_digit_keys(orc, ctx):
    # 300 000 columns: 19-bit keys, three 7-bit digits (as at C4's 1 M columns)
    from test_gpu_row_paths import work_rows
    works = [40, 300, 700, 1024]
    mats = work_rows(works, 300_000, True, seed=8)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "three digits")
    assert sort_digits(300_000) == (3, 64)
    assert sorted_rows(exp[1]) == [True] * 4


@pytest.mark.parametrize("shape", ["colB-scored", "dense", "top_k"])
def test_ineligible_shapes_fall_back(orc, ctx, shape):
    # colB-scored: 2 max rowA max colB >= N, so not every row is keyed; dense: 300 columns fit every warp table;
    # top_k 230: no warp-owned bins at all
    from test_gpu_row_paths import work_rows
    works = [100, 600, 1000]
    top_k = 230 if shape == "top_k" else 50
    mats = work_rows(works, 300 if shape == "dense" else N_COLS, shape != "colB-scored", seed=6)
    exp, _ = run(orc, ctx, mats, [(M_ALL, top_k, None)] * 2, f"fallback {shape}")
    e = exp[1]
    assert sorted_bins(top_k, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users) == set()
    assert not any(sorted_rows(e))
