"""The train's preparation stage on the device, bit for bit, on directed shapes (tests/sampler_shapes.py):
canonicalisation (canonicalize_device), raw column counts (count_raw_columns: k_check_row_ptr, k_col_histogram_flat,
k_sum_copies), sampleDownAndBinarize per chunk (k_sample_count + the compaction), one rank's user block
(cco_debug_downsample_block: row_base != 0, absolute entry offsets), the transpose and the kept-count scan (through the
train's `products`).  Every case is compared with tests/sampler_ref.py (numpy, written from the header's Sampler) and
with the C oracle."""
import numpy as np
import pytest

import rowref
import sampler_ref as sr
import sampler_shapes as shp
import universal_recommender_b200 as ur

pytestmark = pytest.mark.gpu

SHAPES = shp.shapes()
IDS = [s[0] for s in SHAPES]
BIG = 2 ** 31 - 1


def reference(orc, mat, m, seed, flags):
    """sampler_ref's preparation of a (possibly messy) matrix, checked against the oracle's"""
    nr, nc, rp, ci = mat
    s = sr.prepare(nr, nc, rp, ci, m, seed, flags)
    d, raw, new = orc.downsample(orc.canonicalize(orc.Csr(nr, nc, rp, ci)), m, seed, flags & 3)
    assert np.array_equal(s.row_ptr, d.row_ptr) and np.array_equal(s.col_idx, d.col_idx)
    assert np.array_equal(s.raw, raw) and np.array_equal(s.new, new)
    return s


def assert_downsample(ctx, orc, mat, m, seed, flags, tag):
    nr, nc, rp, ci = mat
    want = reference(orc, mat, m, seed, flags)
    grp, gci, graw, gnew = ctx.debug_downsample(nr, nc, rp, ci, m, seed, flags)
    assert np.array_equal(graw, want.raw), f"{tag}: raw column counts differ at {np.flatnonzero(graw != want.raw)[:8]}"
    bad = np.flatnonzero(np.diff(grp) != want.kept)
    assert not len(bad), f"{tag}: kept per row differs at rows {bad[:8]}: {np.diff(grp)[bad[:8]]} vs {want.kept[bad[:8]]}"
    assert np.array_equal(gci, want.col_idx), f"{tag}: kept columns differ"
    assert np.array_equal(gnew, want.new), f"{tag}: post-sample column counts differ"
    return want


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_downsample_directed_shapes(ctx, orc, name, mat, m):
    for i, (mm, seed, flags) in enumerate(shp.settings(m)):
        # half the settings as a caller-promised canonical matrix: the in-train verdict path of count_raw_columns
        f = flags | (ur.FLAG_ASSUME_CANONICAL if i % 2 else 0)
        assert_downsample(ctx, orc, mat, mm, seed, f, f"{name} m={mm} seed={seed} flags={f}")


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_canonicalisation_of_messy_input(ctx, orc, name, mat, m):
    """shuffled, duplicated, all-duplicate and heavy unsorted rows, at n_rows, 2^k and 2^k + 1 (the top bit of the
    (row << 32 | col) sort key)"""
    nr, nc, rp, ci = mat
    k = max(nr - 1, 1).bit_length()
    for n_rows in (nr, 1 << k, (1 << k) + 1):
        x = shp.messy(mat, 5, n_rows)
        want_rp, want_ci = sr.canonicalize(n_rows, x[2], x[3])
        grp, gci, _, _ = ctx.debug_downsample(*x, BIG, 1, 0)           # m = 2^31 - 1: the identity sample
        assert np.array_equal(grp, want_rp) and np.array_equal(gci, want_ci), f"{name} n_rows={n_rows}: canonical form"
        if n_rows == nr:
            assert np.array_equal(grp, rp) and np.array_equal(gci, ci)
        assert_downsample(ctx, orc, x, m, 13, 0, f"{name} messy n_rows={n_rows}")


def cuts(name, mat):
    """block boundaries beyond the ranks' even split: inside runs of empty rows, at and next to the long rows"""
    nr, _, rp, _ = mat
    d = np.diff(rp)
    out = set()
    if name == "empty_runs":
        zero = np.flatnonzero(d == 0)
        out.update(int(zero[i]) for i in (0, 17, len(zero) // 3, len(zero) // 2, len(zero) - 500))
    if name in ("row_lengths", "short_rows"):
        long_rows = np.flatnonzero(d >= 256)
        out.update(int(r) for r in long_rows[::5])
        out.update(int(r) + 1 for r in long_rows[1::5])
    out.update((1, nr - 1, nr // 2))
    return sorted(r for r in out if 0 < r < nr)


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_user_blocks_as_their_ranks_sample_them(ctx, orc, name, mat, m):
    """users cut into rank blocks as on W GPUs, each sampled with row_base != 0: the blocks' kept counts, columns laid end
    to end and summed post-sample counts are the whole-matrix sample"""
    nr, nc, rp, ci = mat
    for (mm, seed, flags) in ((m, 29, 0), (m, -1, ur.FLAG_ROWRATE_INTDIV), (1, 2 ** 31 - 1, 0)):
        whole = assert_downsample(ctx, orc, mat, mm, seed, flags, f"{name} whole")
        splits = [shp.user_blocks(nr, w) for w in (2, 3, 7)]
        c = cuts(name, mat)
        splits.append(list(zip([0] + c, c + [nr])))
        for blocks in splits:
            kept = np.zeros(nr, np.int64)
            cols, new = [], np.zeros(nc, np.int64)
            for lo, hi in blocks:
                tag = f"{name} m={mm} seed={seed} block [{lo}, {hi}) of {len(blocks)}"
                want = sr.downsample_block(nr, nc, rp, ci, lo, hi, whole.raw, mm, seed, flags)
                gk, gc, gn = ctx.debug_downsample_block(nr, nc, rp, ci, lo, hi, whole.raw, mm, seed,
                                                        flags | ur.FLAG_ASSUME_CANONICAL)
                outside = np.concatenate((gk[:lo], gk[hi:]))
                assert not outside.any(), f"{tag}: kept counts written outside the block"
                bad = np.flatnonzero(gk[lo:hi] != want.kept)
                assert not len(bad), f"{tag}: kept per row differs at rows {lo + bad[:8]}"
                assert np.array_equal(gc, want.col_idx), f"{tag}: kept columns differ"
                assert np.array_equal(gn, want.new), f"{tag}: post-sample column counts differ"
                kept[lo:hi] = gk[lo:hi]
                cols.append(gc)
                new += gn
            assert np.array_equal(kept, whole.kept) and np.array_equal(np.concatenate(cols), whole.col_idx)
            assert np.array_equal(new, whole.new)


def second_matrix(mat):
    """a B of the same users: every row's columns shifted, a few rows emptied"""
    nr, nc, rp, ci = mat
    rows = [sorted({(int(c) * 7 + 3) % nc for c in ci[rp[r]:rp[r + 1]]}) if r % 11 != 5 else [] for r in range(nr)]
    return shp.csr(rows, nc)


def assert_train(ctx, orc, mats, params, seed, flags, tag):
    sampler = sr.csr_sampler(orc.Csr)
    got = ctx.train_csr(mats, params, seed=seed, flags=flags)
    st = ctx.last_stats
    exp = rowref.expected(ctx, mats, params, seed, flags, sampler=sampler)
    rowref.assert_matches(exp, got, tag)
    sm = [sampler(orc.Csr(*x), p[0], seed, flags & 3)[0] for x, p in zip(mats, params)]
    assert st.nnz_downsampled == [int(s.row_ptr[-1]) for s in sm], f"{tag}: nnz_downsampled"
    a = sm[0]
    want_p = [sr.products(a.row_ptr, s.row_ptr) for s in sm]
    assert want_p == [sr.products_by_transpose(a.n_rows, a.n_cols, a.row_ptr, a.col_idx, s.row_ptr) for s in sm]
    assert st.products == want_p, f"{tag}: products"
    assert st.distinct_cells == [e.distinct for e in exp], f"{tag}: distinct cells"


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_train_on_directed_shapes(ctx, orc, name, mat, m):
    """the whole train with the sampler active and top_k = 2048 (every positive cell written), once on the canonical
    matrices under FLAG_ASSUME_CANONICAL and once on messy copies (canonicalised on the device) at 2^k and 2^k + 1 rows"""
    nr = mat[0]
    mats = [mat, second_matrix(mat)]
    params = [(m, 2048, None), (max(m // 2, 1), 2048, None)]
    assert_train(ctx, orc, mats, params, 42, ur.FLAG_ASSUME_CANONICAL, f"{name} canonical")
    k = max(nr - 1, 1).bit_length()
    for n_rows in (1 << k, (1 << k) + 1):
        messy = [shp.messy(x, 7 + i, n_rows) for i, x in enumerate(mats)]
        assert_train(ctx, orc, messy, params, -1, ur.FLAG_ROWRATE_INTDIV if n_rows & 1 else 0, f"{name} messy n_rows={n_rows}")
