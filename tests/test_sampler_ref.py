"""The C oracle's canonicalisation and sampler (orc.canonicalize, orc.downsample) against tests/sampler_ref.py, an
independent numpy reading of include/cco_b200.h "Sampler", on the directed shapes of tests/sampler_shapes.py and on
synth "tiny" and "small".  Runs on every CPU box: the oracle the GPU tests trust is pinned here."""
import numpy as np
import pytest

import sampler_ref as sr
import sampler_shapes as shp
import synth

SHAPES = shp.shapes()
IDS = [s[0] for s in SHAPES]


def assert_same(orc, mat, m, seed, flags, tag):
    nr, nc, rp, ci = mat
    d, raw, new = orc.downsample(orc.Csr(nr, nc, rp, ci), m, seed, flags)
    s = sr.downsample(nr, nc, rp, ci, m, seed, flags)
    assert np.array_equal(s.raw, raw), f"{tag}: raw column counts"
    assert np.array_equal(s.row_ptr, d.row_ptr), f"{tag}: kept per row"
    assert np.array_equal(s.col_idx, d.col_idx), f"{tag}: kept columns"
    assert np.array_equal(s.new, new), f"{tag}: post-sample column counts"
    return s


def test_hash_and_u01_match_the_oracle(orc):
    rng = np.random.default_rng(0)
    u = rng.integers(0, 2 ** 31 - 1, 200)
    j = rng.integers(0, 2 ** 31 - 1, 200)
    for seed in (0, 1, -1, 2 ** 31 - 1, -2 ** 31):
        h = sr.hash64(seed, u, j)
        assert [int(x) for x in h] == [orc.hash64(seed, int(a), int(b)) for a, b in zip(u, j)]
        assert np.array_equal(sr.u01(h), [orc.u01(int(x)) for x in h])


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_directed_shapes_match_the_oracle(orc, name, mat, m):
    kept_any = dropped_any = False
    for (mm, seed, flags) in shp.settings(m):
        s = assert_same(orc, mat, mm, seed, flags, f"{name} m={mm} seed={seed} flags={flags}")
        kept_any |= bool(s.keep.any())
        dropped_any |= bool((~s.keep).any())
    assert kept_any and dropped_any or len(mat[3]) < 2, f"{name}: the sampler must both keep and drop"


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_shape_reaches_its_edges(name, mat, m):
    """the directed shapes really hold what their names promise"""
    nr, nc, rp, ci = mat
    d = np.diff(rp)
    assert (ci >= 0).all() and (ci < nc).all()
    assert all((np.diff(ci[rp[r]:rp[r + 1]]) > 0).all() for r in range(nr))          # canonical
    c = np.bincount(ci, minlength=nc)
    if name == "row_lengths":
        for length in (0, 1, 31, 32, 33, 255, 256, 257, 5000):
            starts = rp[:-1][d == length]
            for modulus in (shp.CHUNK, shp.BATCH):
                assert {0, 1, modulus - 1} <= set((starts % modulus).tolist()), (length, modulus)
    if name == "empty_runs":
        runs = np.diff(np.flatnonzero(np.concatenate(([1], d != 0, [1])))) - 1
        assert {31, 32, 33, 64, 1000} <= set(runs.tolist())
        assert d[:33].sum() == 0 and d[-1000:].sum() == 0
    if name.startswith("thresholds"):
        assert {m, m + 1} <= set(d.tolist()) and c[0] == m and c[1] == m + 1
    if name == "one_column":
        assert nc == 1 and len(ci) % 32 and len(ci) > 16 * shp.CHUNK
    if name == "last_column":
        assert c[nc - 1] > m
    if name.startswith("rows"):
        assert nr == int(name[4:name.index("_")]) and len(ci) == int(name[name.index("nnz") + 3:])


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_user_blocks_add_up_to_the_whole_matrix(name, mat, m):
    """a block sampled with the whole matrix's raw counts and global user ids: blocks laid end to end are the whole"""
    nr, nc, rp, ci = mat
    whole = sr.downsample(nr, nc, rp, ci, m, 11, 0)
    for world in (2, 3, 7):
        kept = np.zeros(nr, np.int64)
        cols, new = [], np.zeros(nc, np.int64)
        for lo, hi in shp.user_blocks(nr, world):
            s = sr.downsample_block(nr, nc, rp, ci, lo, hi, whole.raw, m, 11, 0)
            assert np.array_equal(s.keep, whole.keep[rp[lo]:rp[hi]])
            kept[lo:hi] = s.kept
            cols.append(s.col_idx)
            new += s.new
        assert np.array_equal(kept, whole.kept) and np.array_equal(np.concatenate(cols), whole.col_idx)
        assert np.array_equal(new, whole.new)


@pytest.mark.parametrize("name,mat,m", SHAPES, ids=IDS)
def test_canonicalisation_matches_the_oracle(orc, name, mat, m):
    nr, nc, rp, ci = mat
    for n_rows in (nr, 1 << max(nr - 1, 1).bit_length(), (1 << max(nr - 1, 1).bit_length()) + 1):
        x = shp.messy(mat, 5, n_rows)
        want = orc.canonicalize(orc.Csr(*x))
        got_rp, got_ci = sr.canonicalize(x[0], x[2], x[3])
        assert np.array_equal(got_rp, want.row_ptr) and np.array_equal(got_ci, want.col_idx), (name, n_rows)
        if n_rows == nr:
            assert np.array_equal(got_rp, rp) and np.array_equal(got_ci, ci)
        # the whole preparation of the messy input equals the oracle's
        s = sr.prepare(x[0], nc, x[2], x[3], m, 9, 0)
        d, raw, new = orc.downsample(want, m, 9, 0)
        assert np.array_equal(s.row_ptr, d.row_ptr) and np.array_equal(s.col_idx, d.col_idx)
        assert np.array_equal(s.raw, raw) and np.array_equal(s.new, new)


@pytest.mark.parametrize("name", ["tiny", "small"])
def test_synth_matches_the_oracle_and_its_products(orc, name):
    w = synth.make(name)
    for i, (nr, nc, rp, ci) in enumerate(w.mats):
        for (m, seed, flags) in ((w.max_interactions, 42, 0), (40, -1, 0), (40, 2 ** 31 - 1, sr.FLAG_ROWRATE_INTDIV)):
            assert_same(orc, (nr, nc, rp, ci), m, seed, flags, f"{name} matrix {i} m={m} seed={seed}")
    # P = sum_u deg_A'(u) deg_B'(u), which the train reports as `products`, and nnz of the sampled matrices
    params = [(40, 50, None)] * len(w.mats)
    ref = orc.train([orc.Csr(*x) for x in w.mats], [orc.Params(*p) for p in params], 42)
    sm = [sr.prepare(nr, nc, rp, ci, 40, 42, 0) for (nr, nc, rp, ci) in w.mats]
    a = sm[0]
    for i, (s, r) in enumerate(zip(sm, ref)):
        assert sr.products(a.row_ptr, s.row_ptr) == r.products, i
        assert sr.products_by_transpose(w.n_users, w.mats[0][1], a.row_ptr, a.col_idx, s.row_ptr) == r.products, i
        assert int(s.row_ptr[-1]) == r.nnz_b, i


def test_transpose_is_the_transpose():
    nr, nc, rp, ci = shp.empty_runs()
    ptr, users = sr.transpose(nr, nc, rp, ci)
    dense = np.zeros((nr, nc), bool)
    dense[np.repeat(np.arange(nr), np.diff(rp)), ci] = True
    for j in range(nc):
        assert np.array_equal(users[ptr[j]:ptr[j + 1]], np.flatnonzero(dense[:, j]))
