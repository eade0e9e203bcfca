"""The device LLR against exact arithmetic: the fp64 error bound eps(N) = 2^-47 N ln N (cco_api.cu llr_error_bound)
that the row kernel's level-1 cut and dominance filter rely on, checked on the device's own values (DESIGN.md 3.1).

  * llr_cells (ctx.debug_llr) within eps of the real value on the edge grid of tests/llr_exact.py, both entropy orders;
  * computed k11 = 1 LLRs strictly decreasing in colB wherever row_paths.cut_exact admits the cut;
  * the dominance property dev(k', c') <= dev(k, c) + 2 eps on pairs biased toward independence;
  * the kernel's hoisted LLR (x11tab, x12tab, ColTerm.x_cbm1, row_e) at its table edges, on every owner path;
  * the cut decision at its boundary, end to end."""
import numpy as np
import pytest

import llr_exact as lx
import row_paths
import synth
import universal_recommender_b200 as ur
from test_gpu_bitmap_rows import bitmap_bins
from test_gpu_row_paths import csr, run
from test_gpu_sorted_rows import sorted_bins

pytestmark = pytest.mark.gpu
M_ALL = 10 ** 9
ORDERS = [0, ur.FLAG_ENTROPY_VARARGS]
ORDER_IDS = ["left-to-right", "varargs"]


def k1_llr(ctx, n, ra, cb, flags=0):
    """Device LLR of the k11 = 1 cells of rowA = ra at every colB of cb"""
    cb = np.asarray(cb, dtype=np.int64)
    one = np.ones_like(cb)
    return ctx.debug_llr(one, one * (ra - 1), cb - 1, n - ra - cb + 1, flags)


# ---- a. llr_cells against the real value -----------------------------------------------------------------------------
@pytest.mark.parametrize("flags", ORDERS, ids=ORDER_IDS)
def test_device_llr_within_eps_of_the_real_value(orc, ctx, request, flags):
    lines = []
    for n in lx.GRID_N:
        cells = lx.grid(n)
        real = lx.llr_longdouble(*cells)
        dev = ctx.debug_llr(*cells, flags)
        worst = lx.check_against_real(dev, real, n, f"device N={n} flags={flags}")
        ref = lx.oracle_llr(orc, cells, flags)
        gap = np.abs(dev - ref)
        bad = np.nonzero(gap > 2 * lx.eps(n))[0]
        assert not len(bad), f"N={n}: device {dev[bad[0]]!r} vs oracle {ref[bad[0]]!r} at cell " \
                             f"{tuple(int(x[bad[0]]) for x in cells)}"
        lines.append(f"N = {n:>10}: {worst:.4f} eps ({len(real)} cells, {int((dev != ref).sum())} differ from glibc)")
    lx.report(request, f"device llr_cells ({ORDER_IDS[ORDERS.index(flags)]}): largest |computed - real| / eps per N",
              lines)


# ---- b. monotone in colB wherever the cut is admitted -----------------------------------------------------------------
@pytest.mark.parametrize("n", [10 ** 5, 10 ** 6, 10 ** 7, 5 * 10 ** 7, 2 * 10 ** 8, 2 ** 31 - 1])
def test_device_k1_llr_strictly_decreasing_where_the_cut_is_admitted(ctx, n):
    for ra in (1, 2, 7, 60, 600):
        c = lx.cut_c_max(n, ra)
        assert 2 * ra * c < n and (c == (n - 1) // (2 * ra) - 1 or not row_paths.cut_exact(n, ra, c + 1))
        # the bound turns the cut off once max colB nears 1 / eps, so c_max stays below 10^6 for every N here (873 164 at
        # N = 1e7, rowA = 1; 3 049 at N = 2^31 - 1): every colB of 1..c_max is evaluated
        assert c < 1_000_000
        cb = np.arange(1, c + 1)
        for flags in ORDERS:
            v = k1_llr(ctx, n, ra, cb, flags)
            up = np.nonzero(np.diff(v) >= 0)[0]
            assert not len(up), f"N={n} rowA={ra} flags={flags} (c_max {c}): colB {cb[up[0]]} -> {cb[up[0]] + 1} " \
                                f"computes {v[up[0]]!r} -> {v[up[0] + 1]!r}"


def test_documented_fp64_defects_on_device_values(ctx):
    # N = 2e7, rowA = 1: colB 9 271 424 and 9 271 425 compute to the same LLR; cut_exact refuses that max colB
    n = 20_000_000
    v = k1_llr(ctx, n, 1, [9_271_424, 9_271_425])
    assert v[0] == v[1], f"no fp64 tie on this device: {v[0]!r} (colB 9271424) vs {v[1]!r} (colB 9271425)"
    assert lx.llr_exact(n, 1, 9_271_424) > lx.llr_exact(n, 1, 9_271_425)
    assert not row_paths.cut_exact(n, 1, 9_271_425)
    # N = 5e7, rowA = 1: computed values increase somewhere above colB 1.5e7, while the real ones decrease
    n = 50_000_000
    seen = []
    for lo in (15_000_000, 20_000_000):
        cb = np.arange(lo, lo + 4000)
        v = k1_llr(ctx, n, 1, cb)
        seen += [int(cb[i]) for i in np.nonzero(np.diff(v) > 0)[0]]
    assert seen, "no increase of the computed k11 = 1 LLR above colB 1.5e7 at N = 5e7 on this device"
    real = lx.llr_longdouble(1, 0, np.array(seen) - 1, n - np.array(seen))
    real_next = lx.llr_longdouble(1, 0, np.array(seen), n - np.array(seen) - 1)
    assert (real_next < real).all()
    assert not row_paths.cut_exact(n, 1, 15_000_000)


# ---- c. the dominance property ----------------------------------------------------------------------------------------
def dominance_pairs(n, rng, count):
    """(rowA, k, c, k', c') with k' <= k, c' >= c, (k', c') on the positive side (rowA c' < k' N); half of them with c'
    just below the independence point of k' (rowA c' ~ k' N), where the fp64 LLR is cancellation-limited"""
    ra = np.choose(rng.integers(0, 5, count), [rng.integers(1, 601, count), np.full(count, 20), np.full(count, 2),
                                                rng.integers(1, max(n // 4, 1) + 1, count), rng.integers(30, 35, count)])
    ra = np.clip(ra, 1, max(n // 2, 1)).astype(np.int64)
    near = rng.random(count) < 0.5
    # near independence: k' small, c' the largest colB with rowA c' < k' N (minus 0..3)
    kp_near = np.minimum(rng.integers(1, 41, count), ra)
    cp_near = (kp_near * n - 1) // ra - rng.integers(0, 4, count)
    # random: c' anywhere, k' from the first positive count up to its limit
    cp_rand = rng.integers(1, n - ra + 1)
    kmin = ra * cp_rand // n + 1
    kp_rand = kmin + (rng.random(count) * (np.minimum(ra, cp_rand) - kmin + 1)).astype(np.int64)
    kp = np.where(near, kp_near, kp_rand)
    cp = np.minimum(np.where(near, cp_near, cp_rand), n - ra + kp)
    cp = np.maximum(cp, kp)
    k = np.minimum(kp + rng.integers(0, 3, count), np.minimum(ra, cp))
    c = np.maximum(cp - rng.integers(0, 6, count), k)
    keep = ra * cp < kp * n
    return ra[keep], k[keep], c[keep], kp[keep], cp[keep]


@pytest.mark.parametrize("flags", ORDERS, ids=ORDER_IDS)
def test_dominance_property_on_device_values(ctx, request, flags):
    lines, total = [], 0
    for n in (10 ** 3, 10 ** 5, 10 ** 6, 10 ** 7, 2 * 10 ** 7, 10 ** 8, 2 ** 31 - 1):
        ra, k, c, kp, cp = dominance_pairs(n, np.random.default_rng(7 + n), 160_000)
        if n == 10 ** 6:      # the documented crossing: rowA = 20, k11 = 3, colB 149 995 -> 149 996
            ra, k, c, kp, cp = (np.append(x, y) for x, y in zip((ra, k, c, kp, cp), (20, 3, 149_995, 3, 149_996)))
        assert (kp <= k).all() and (cp >= c).all() and (k <= np.minimum(ra, c)).all() and (n - ra - cp + kp >= 0).all()
        hi = ctx.debug_llr(k, ra - k, c - k, n - ra - c + k, flags)
        lo = ctx.debug_llr(kp, ra - kp, cp - kp, n - ra - cp + kp, flags)
        e = lx.eps(n)
        over = lo - hi
        bad = np.nonzero(over > 2 * e)[0]
        assert not len(bad), f"N={n}: dominated cell (k'={kp[bad[0]]}, c'={cp[bad[0]]}) computes {lo[bad[0]]!r}, above " \
                             f"(k={k[bad[0]]}, c={c[bad[0]]}) {hi[bad[0]]!r} + 2 eps (rowA {ra[bad[0]]})"
        total += len(ra)
        lines.append(f"N = {n:>10}: {len(ra)} pairs, {int((over > 0).sum())} dominated cells compute higher, largest "
                     f"excess {max(float(over.max()), 0.0) / e:.4f} eps")
    assert total >= 1_000_000
    lx.report(request, f"dominance on device values ({ORDER_IDS[ORDERS.index(flags)]})", lines)


# ---- d. the kernel's hoisted LLR at its table edges -------------------------------------------------------------------
def rows_with_cells(items, n_cols, rng):
    """items: [(rowA, {column: k11})] -> [A', B'].  Item i gets rowA users of its own, user t buying the columns with
    k11 > t; users outside A' then raise each used column's colB by 0..20.  N makes every row keyed (2 rowA colB < N)."""
    a_rows, b_rows = [], []
    for i, (ra, cells) in enumerate(items):
        assert max(cells.values()) <= ra
        for t in range(ra):
            a_rows.append([i])
            b_rows.append(sorted(c for c, k in cells.items() if k > t))
    used = np.bincount(np.concatenate([np.asarray(r, dtype=np.int64) for r in b_rows]), minlength=n_cols)
    extra = np.where(used > 0, rng.integers(0, 21, n_cols), 0)
    for f in range(int(extra.max())):
        b_rows.append(np.nonzero(extra > f)[0].tolist())
    n = max(len(b_rows), 2 * max(ra for ra, _ in items) * int((used + extra).max()) + 1)
    return [csr(a_rows, len(items), n), csr(b_rows, n_cols, n)]


def edge_row(ra, work, cols):
    """{column: k11}: k11 = 1..min(40, rowA) (x11tab ends at 32, x12tab at 31), then cells of k11 = rowA (rowA - k11 =
    0) until the row has `work` products"""
    ks = list(range(1, min(40, ra) + 1))
    while sum(ks) < work:
        ks.append(ra)
    assert len(ks) <= len(cols)
    return {int(c): k for c, k in zip(cols, ks)}


EDGE_RA = [30, 31, 32, 33, 600]
TOP_K = 200          # above every row's cell count, and warp-owned rows still exist (top_k + 32 <= 256)


@pytest.mark.parametrize("flags", ORDERS, ids=ORDER_IDS)
@pytest.mark.parametrize("table", ["dense", "hashed"])
def test_hoisted_llr_at_the_table_edges(orc, ctx, table, flags):
    # dense (128 columns): warp-owned rows (work <= 1024) and 128-thread rows (1025..2048);
    # hashed (70 001 columns): sorted warp rows, 128-thread rows and bitmap rows (256 threads, 2049..4096)
    rng = np.random.default_rng(40 + len(table))
    n_cols = 128 if table == "dense" else 70_001
    kinds = [("warp", 0), ("cta", 1100)] if table == "dense" else [("sorted", 0), ("cta", 1100), ("bitmap", 2600)]
    items, kind_of = [], []
    for kind, work in kinds:
        for ra in EDGE_RA:
            cols = rng.permutation(n_cols)[:TOP_K]
            items.append((ra, edge_row(ra, work, cols)))
            kind_of.append(kind)
    mats = rows_with_cells(items, n_cols, rng)
    exp, paths, got = run(orc, ctx, mats, [(M_ALL, TOP_K, None)] * 2, flags=flags, tag=f"table edges {table}")
    e = exp[1]
    bm = bitmap_bins(TOP_K, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users)
    so = sorted_bins(TOP_K, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users)
    for i, (p, kind) in enumerate(zip(paths[1], kind_of)):
        assert p is not None and p.keyed and p.cut and p.dense == (table == "dense"), (i, p)
        want = {"warp": p.group == 32, "sorted": p.group == 32 and p.bin in so,
                "cta": p.group == 128 and p.bin not in bm, "bitmap": p.group in (256, 512) and p.bin in bm}[kind]
        assert want, (kind, items[i][0], int(e.work[i]), p)
    # every cell is kept (all are positive, fewer than top_k per row), k11 = 31 on every row with rowA >= 31
    _, _, _, rp, ci, ll, cn = got[1]
    assert np.diff(rp).tolist() == [len(c) for _, c in items]
    row = np.repeat(np.arange(len(items)), np.diff(rp))
    for i, (ra, _) in enumerate(items):
        if ra >= 31:
            assert 31 in cn[rp[i]:rp[i + 1]].tolist(), i
    # every kept LLR within eps of the real value (rowref.assert_matches in run: bit-equal to llr_cells)
    n = e.n_users
    ra = e.ra[row].astype(np.int64)
    cb = np.bincount(mats[1][3], minlength=n_cols)[ci].astype(np.int64)
    k11 = cn.astype(np.int64)
    for r, (_, cells) in enumerate(items):
        assert {int(c): int(k) for c, k in zip(ci[rp[r]:rp[r + 1]], cn[rp[r]:rp[r + 1]])} == cells
    real = lx.llr_longdouble(k11, ra - k11, cb - k11, n - ra - cb + k11)
    lx.check_against_real(np.asarray(ll, dtype=np.float64), real, n, f"kept LLRs, {table}")


# ---- e. the cut decision at its boundary, end to end -------------------------------------------------------------------
@pytest.mark.parametrize("top_colb,cut", [(418_581, True), (418_582, False)], ids=["cut-on", "cut-off"])
def test_cut_at_its_boundary_end_to_end(orc, ctx, top_colb, cut):
    # N = 2e7, one item bought by user 0 (rowA = 1).  User 0 also buys 12 columns of B' whose colB are top_colb,
    # top_colb - 1, ..., top_colb - 11: twelve k11 = 1 cells at adjacent colB, top_k = 4.  cut_exact admits max colB
    # 418 581 at R = 1 and refuses 418 582, far below the strongly positive cap (~1e7).
    n, n_cells, top_k, n_cols = 20_000_000, 12, 4, 70_001
    assert row_paths.cut_exact(n, 1, top_colb) == cut and 2 * top_colb < n
    cols = np.arange(n_cells) * 5_000 + 17                     # colB top_colb - j on column cols[j]
    colb = top_colb - np.arange(n_cells)
    users = np.concatenate([np.zeros(n_cells, np.int64)] + [np.arange(1, b, dtype=np.int64) for b in colb])
    items = np.concatenate([cols] + [np.full(b - 1, c, np.int64) for c, b in zip(cols, colb)])
    rp, ci = synth.to_binary_csr(users, items, n, n_cols)
    a = csr([[0]], 1, n)
    mats = [a, (n, n_cols, rp, ci)]
    v = k1_llr(ctx, n, 1, colb[::-1])
    if cut:
        assert (np.diff(v) < 0).all(), v                         # the cut's premise on the device's values
    exp, paths, got = run(orc, ctx, mats, [(M_ALL, top_k, None)] * 2, tag=f"cut boundary {top_colb}")
    e = exp[1]
    assert e.max_marg_b == top_colb and e.max_marg_a == 1
    p = paths[1][0]
    so = sorted_bins(top_k, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users)
    bm = bitmap_bins(top_k, e.n_cols_b, e.max_marg_a, e.max_marg_b, e.n_users)
    assert p.keyed and p.group == 32 and not p.dense and p.cut == cut
    if cut:
        assert p.bin in so                                       # a sorted row: its key cut runs on the sorted runs
    else:
        assert not so and not bm                                 # neither sorted nor bitmap rows without the cut
    # the four lowest colB win: columns of colB top_colb - 11 .. top_colb - 8
    assert got[1][4].tolist() == cols[::-1][:top_k].tolist()
    # what the device decided (the kept set is the same either way): with the cut, the k11 = 1 cells past the top_k-th
    # key are dropped before they are evaluated; without it every cell is evaluated
    st = ctx.last_stats
    assert st.distinct_cells[1] == n_cells
    if cut:
        assert top_k <= st.llr_evaluated[1] < n_cells, st.llr_evaluated
    else:
        assert st.llr_evaluated[1] == n_cells, st.llr_evaluated
