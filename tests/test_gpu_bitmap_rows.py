"""Bitmap rows of `k_rows` (DESIGN.md 3.1): CTA-owned hashed bins whose rows are all keyed with an exact cut count each
cell's first product into a bitmap over the keys, hash only the repeated products, and list the k11 = 1 cells up to the
key cut from the bitmap.  Each case is checked bit for bit against the brute force of tests/rowref.py and against the
oracle, and asserts through `bitmap_bins` (a restatement of `use_bitmap` and its caller in cco_api.cu) which rows took
the bitmap path."""
import numpy as np
import pytest

import row_paths
import rowref
from test_gpu_parity import assert_indicators_equal, oracle_train

pytestmark = pytest.mark.gpu
M_ALL = 10 ** 9
N_COLS = 70_001          # hashed in every CTA bin, bitmap in the 512- and 256-thread bins; not a multiple of 32


def bitmap_bins(top_k: int, n_cols_b: int, max_marg_a: int, max_marg_b: int, n_users: int) -> set:
    """Bins that run bitmap rows (cco_api.cu: `bitmap_ok` in enqueue_indicator, then `use_bitmap` per bin)."""
    if not (row_paths.cut_exact(n_users, max_marg_a, max_marg_b) and 2 * max_marg_a * max_marg_b < n_users):
        return set()
    cfgs, h_thr = row_paths.bins(top_k, n_cols_b)
    out = set()
    for b in range(1, len(cfgs)):
        f = cfgs[b]
        if f.dense or f.group not in (512, 256):                                # `f.dense || (group != 512 && != 256)`
            continue
        rep = -(-max(h_thr[b - 1], 64) // f.group) * f.group                     # `rep`: max_w rounded to 32 NW
        if rep + -(-n_cols_b // 32) + top_k <= f.slots:                          # `rep + bm + top_k > f.slots`
            out.add(b)
    return out


def bitmap_rows(e: rowref.Expected) -> list:
    """Per output row: True (bitmap row), False (another path) or None (no work)."""
    bins = bitmap_bins(e.top_k, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users)
    return [None if p is None else p.bin in bins for p in e.paths()]


def run(orc, ctx, mats, params, tag):
    got = ctx.train_csr(mats, params, seed=1)
    exp = rowref.expected(ctx, mats, params, 1)
    rowref.assert_matches(exp, got, tag)
    assert_indicators_equal(oracle_train(orc, mats, params, 1, 0), got, mats[0][0], tag)
    assert ctx.last_stats.distinct_cells == [e.distinct for e in exp]   # popcount of the bitmap + the repeated cells
    return exp, got


def shaped(items, n_cols, colb, n_users=0):
    """Cross indicator A'^T B' with given cells: items[i] = {column: k11}.  Item i gets max(k11) users, user t buying the
    columns with k11 > t; users outside A' then raise every column's colB to colb[j] (they add no products).  With colb
    non-decreasing in the column id, key = id.  N makes every row keyed (2 rowA colB < N)."""
    a_rows, b_rows = [], []
    for i, cells in enumerate(items):
        for t in range(max(cells.values())):
            a_rows.append([i])
            b_rows.append(sorted(c for c, k in cells.items() if k > t))
    used = np.bincount(np.concatenate([np.asarray(r, dtype=np.int64) for r in b_rows]), minlength=n_cols)
    deficit = np.asarray(colb, dtype=np.int64) - used
    assert (deficit >= 0).all()
    for f in range(int(deficit.max(initial=0))):
        b_rows.append(np.nonzero(deficit > f)[0].tolist())
    max_ra = max(max(c.values()) for c in items)
    n = max(len(b_rows), 2 * max_ra * int(max(colb)) + 1, n_users)
    from test_gpu_row_paths import csr
    return [csr(a_rows, len(items), n), csr(b_rows, n_cols, n)]


def ramp(n_cols, lo=2, hi=12):
    """colB non-decreasing in the column id (so key = id)."""
    return lo + (np.arange(n_cols, dtype=np.int64) * (hi - lo + 1)) // n_cols


def singles_row(single_keys, w, rep_from, k11=2, rng=None):
    """{column: k11}: k11 = 1 at single_keys, then repeated cells (k11) from column rep_from up until w products."""
    cells = {int(c): 1 for c in single_keys}
    c = rep_from
    while sum(cells.values()) < w:
        if c not in cells:
            cells[c] = k11
        c += 1
    return cells


def test_rows_in_each_bitmap_bin(orc, ctx):
    # random rows around the bin edges: 512-thread bin (4096 < w <= 8192), 256 (2048 < w <= 4096), and the 128-thread
    # and 1024-thread bins next to them, which keep the hashed path
    from test_gpu_row_paths import work_rows
    works = [2048, 2049, 3000, 4096, 4097, 6000, 8192, 8193]
    mats = work_rows(works, N_COLS, True, seed=11)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "bitmap bins")
    e = exp[1]
    assert bitmap_bins(50, N_COLS, e.max_marg_a, e.max_marg_b, e.n_users) == {2, 3}
    assert bitmap_rows(e) == [False, True, True, True, True, True, True, False]


def test_keys_at_word_edges_and_fewer_singles_than_top_k(orc, ctx):
    # keys 0, 31, 32 and n_cols - 1 (the last, partial bitmap word) as the only k11 = 1 cells of a row (fewer than top_k:
    # all listed), and as singles below the cut of a row with 5000 more singles
    last = N_COLS - 1
    items = [singles_row([0, 31, 32, last], 5000, 1000),
             singles_row([0, 31, 32, last], 3000, 1000, k11=3),
             singles_row([0, 31, 32, last] + list(range(100, 5100)), 6000, 20_000)]
    colb = np.where(np.arange(N_COLS) < 1000, 3, 150)   # non-decreasing: key = id; repeated cells all have colB 150
    mats = shaped(items, N_COLS, colb, n_users=1000)
    exp, got = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "word edges")
    e = exp[1]
    assert bitmap_rows(e) == [True, True, True]
    # the third row keeps its strongest singles: the smallest keys, word edges included
    assert {0, 31, 32} <= set(e.col[e.row_ptr[2]:e.row_ptr[3]].tolist())


@pytest.mark.parametrize("kth", [63, 64, 159, 160, 287, 288])
def test_top_k_th_single_at_a_word_edge(orc, ctx, kth):
    # the 50th smallest single key at the last / first bit of a bitmap word, and at the edge of a thread's word range
    # (5 words per thread in the 512-thread bin at 70 001 columns, 9 in the 256-thread bin).  Every single has colB 2 and
    # the repeated cells colB 150, so the 50 kept cells are exactly the 50 smallest singles.
    first = kth - 49
    singles = list(range(first, kth + 1)) + list(range(kth + 500, kth + 500 + 4300))
    items = [singles_row(singles[:50 + 4300], 6000, 60_000), singles_row(singles[:50 + 2400], 3000, 60_000)]
    colb = ramp(N_COLS, 2, 3)
    colb[60_000:] = 150
    mats = shaped(items, N_COLS, colb, n_users=1000)
    exp, got = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, f"kth single {kth}")
    e = exp[1]
    assert bitmap_rows(e) == [True, True]
    for r in range(2):
        assert e.col[e.row_ptr[r]:e.row_ptr[r + 1]].tolist() == list(range(first, kth + 1))


def test_every_cell_repeated(orc, ctx):
    # no k11 = 1 cell at all: the bitmap empties completely after the repeats leave it
    items = [{c: 2 + c % 3 for c in range(7, 2007)}, {c: 2 for c in range(30_000, 31_500)}]
    mats = shaped(items, N_COLS, ramp(N_COLS, 5, 9), n_users=1000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "all repeated")
    assert bitmap_rows(exp[1]) == [True, True]
    assert not (exp[1].count == 1).any()


def test_colb_ties_straddle_the_cut(orc, ctx):
    # colB runs of 40 equal values that fall as the column id rises: key order and id order disagree across runs, agree
    # inside one; the 50th single sits inside a run.  The repeated cells (colB 150) rank below every kept single.
    colb = np.minimum(2 + (N_COLS - 1 - np.arange(N_COLS)) // 40, 12)
    colb[1000:6000] = 150
    tail = np.arange(N_COLS - 400, N_COLS)
    items = [singles_row(tail.tolist(), 5000, 1000), singles_row(tail[::2].tolist(), 3000, 1000)]
    mats = shaped(items, N_COLS, colb, n_users=1000)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, "colB ties")
    e = exp[1]
    assert bitmap_rows(e) == [True, True]
    # row 0 keeps the 40 singles of colB 2 and the first 10 (by id) of the 40 of colB 3
    assert e.col[e.row_ptr[0]:e.row_ptr[1]].tolist() == list(range(N_COLS - 40, N_COLS)) + \
        list(range(N_COLS - 80, N_COLS - 70))


def test_self_diagonal_as_single_and_as_repeat(orc, ctx):
    # A'^T A' over 70 001 items: users 0 and 1 buy 3000 items each, 1000 of them in common.  A common item's row has
    # 6000 products and its diagonal k11 = 2 (a repeat); an item of one user has 3000 products, all k11 = 1, its diagonal
    # a single with one of the smallest keys.
    from test_gpu_row_paths import csr
    rng = np.random.default_rng(3)
    items = rng.permutation(N_COLS)[:5000]
    common, own0, own1 = items[:1000], items[1000:3000], items[3000:5000]
    n = 1000   # users without items keep every row keyed (2 rowA colB < N)
    rows = [sorted(np.concatenate([common, own0]).tolist()), sorted(np.concatenate([common, own1]).tolist())]
    m = csr(rows, N_COLS, n)
    exp, got = run(orc, ctx, [m, m], [(M_ALL, 50, None), (M_ALL, 50, None)], "self diagonal")
    for e in exp:
        br = bitmap_rows(e)
        assert all(br[i] for i in common) and all(br[i] for i in own0)
    assert bitmap_bins(50, N_COLS, exp[0].max_marg_a, exp[0].max_marg_b, n) == {2, 3}
    for i in (int(common[0]), int(own0[0])):
        kept = got[0][4][exp[0].row_ptr[i]:exp[0].row_ptr[i + 1]]
        assert i not in kept.tolist() and len(kept) == 50


def test_min_llr(orc, ctx):
    items = [singles_row(list(range(0, 4500, 3)), 6000, 10_000), singles_row(list(range(5, 2000, 2)), 3000, 10_000)]
    mats = shaped(items, N_COLS, ramp(N_COLS, 4, 12), n_users=1000)
    base = rowref.expected(ctx, mats, [(M_ALL, 50, None)] * 2, 1)[1]
    for row, rank in ((0, 30), (1, 49)):
        t = float(base.llr[base.row_ptr[row] + rank])
        exp, got = run(orc, ctx, mats, [(M_ALL, 50, t)] * 2, f"minLLR={t!r}")
        assert bitmap_rows(exp[1]) == [True, True]
        assert (got[1][5] >= t).all() and (got[1][5] == t).any()


@pytest.mark.parametrize("shape", ["wide", "colB-scored"])
def test_ineligible_shapes_fall_back(orc, ctx, shape):
    # 300 000 columns: the bitmap does not fit the 512- or 256-thread bin's table.  colB-scored: 2 max rowA max colB >= N,
    # so not every row is keyed and no bin runs bitmap rows
    from test_gpu_row_paths import work_rows
    works = [3000, 6000]
    if shape == "wide":
        mats = work_rows(works, 300_000, True, seed=5)
    else:
        mats = work_rows(works, N_COLS, False, seed=5)
    exp, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, f"fallback {shape}")
    e = exp[1]
    if shape == "colB-scored":
        assert 2 * e.max_marg_a * e.max_marg_b >= e.n_users
    assert bitmap_bins(50, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users) == set()
    assert [p.group for p in e.paths()] == [256, 512]
