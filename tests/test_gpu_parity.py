"""Parity tests proper: the sm_90a path, called through the C ABI, against the oracle on the same seeded inputs,
against the committed golden fixtures, and -- at BASELINE.json's C3 size -- through size-independent properties.

Bars: co-occurrence counts, kept columns and row lengths bit-exact; LLR within 2 eps(N) of the oracle's, eps(N) =
2^-47 N ln N being the bound on |computed - real| of one fp64 LLR that the row kernel's cut and dominance filter rely on
(cco_api.cu llr_error_bound; tests/test_gpu_llr_exact.py checks it against exact values)."""
import numpy as np
import pytest

import rowref
import row_paths
import synth
import universal_recommender_b200 as ur
from conftest import load_golden, prepared_from_fixture

pytestmark = pytest.mark.gpu
LLR_RTOL = 1e-6         # the reference's golden fixtures


def llr_bar(n_users):
    """Largest |device - oracle| of one LLR at N = n_users: each is within eps(N) of the real value"""
    return 2.0 * row_paths.llr_error_bound(int(n_users))


def assert_llr_close(got, want, n_users, tag=""):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, f"{tag}: LLR shapes differ"
    bar = llr_bar(n_users)
    bad = np.nonzero(~(np.abs(got - want) <= bar))[0]
    assert not len(bad), f"{tag}: LLR beyond 2 eps(N) = {bar!r} (N = {n_users}) at {len(bad)} cells, first {bad[0]}: " \
                         f"{got[bad[0]]!r} vs {want[bad[0]]!r}"


def assert_indicators_equal(ref, got, n_users, tag=""):
    """n_users: N of the train, the row count of its matrices"""
    assert len(ref) == len(got)
    for i, (r, g) in enumerate(zip(ref, got)):
        rb, re_, nc, rp, ci, ll, cn = g
        assert (rb, re_, nc) == (0, r.n_rows, r.n_cols), f"{tag} indicator {i}: shape"
        assert np.array_equal(rp, r.row_ptr), f"{tag} indicator {i}: row lengths differ"
        assert np.array_equal(ci, r.col_idx), f"{tag} indicator {i}: kept columns differ"
        assert np.array_equal(cn, r.count), f"{tag} indicator {i}: co-occurrence counts differ"
        assert_llr_close(ll, r.llr, n_users, f"{tag} indicator {i}")


def oracle_train(orc, mats, params, seed, flags=0):
    return orc.train([orc.Csr(*m) for m in mats], [orc.Params(*p) for p in params], seed, flags)


# ---- synthetic workloads (sizes the oracle finishes in seconds) -------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny", "small", "C2", "C3-tenth"])
def test_synthetic_parity(orc, ctx, name):
    w = synth.make(name, ctx=ctx)                 # generated + ingested on the device (cco_synth_ingest)
    got = ctx.train_csr(w.mats, w.params, seed=42)
    ref = oracle_train(orc, w.mats, w.params, 42)
    assert_indicators_equal(ref, got, w.mats[0][0], name)
    st = ctx.last_stats
    assert st.products == [r.products for r in ref]
    assert st.distinct_cells == [r.distinct_cells for r in ref]
    assert st.nnz_downsampled == [r.nnz_b for r in ref]
    assert st.n_kernel_launches > 0


@pytest.mark.parametrize("flags", [ur.FLAG_ROWRATE_INTDIV, ur.FLAG_ENTROPY_VARARGS, ur.FLAG_ASSUME_CANONICAL])
def test_flags_parity(orc, ctx, flags):
    w = synth.make("small")
    got = ctx.train_csr(w.mats, w.params, seed=9, flags=flags)
    ref = oracle_train(orc, w.mats, w.params, 9, flags & 3)
    assert_indicators_equal(ref, got, w.mats[0][0], f"flags={flags}")


def test_per_indicator_params_and_min_llr(orc, ctx):
    w = synth.make("small")
    params = [(50, 10, None), (500, 3, 2.0), (20, 64, 0.25)]
    got = ctx.train_csr(w.mats, params, seed=3)
    ref = oracle_train(orc, w.mats, params, 3)
    assert_indicators_equal(ref, got, w.mats[0][0])
    assert (got[1][5] >= 2.0).all()


@pytest.mark.parametrize("k", [1, 97, 300, 2048])
def test_top_k_extremes(orc, ctx, k):
    # k > 224 switches the small rows from warp-owned to CTA-owned groups; k > n_cols keeps every positive cell
    w = synth.make("tiny")
    params = [(500, k, None)] * 3
    assert_indicators_equal(oracle_train(orc, w.mats, params, 5), ctx.train_csr(w.mats, params, seed=5), w.mats[0][0], f"k={k}")


def test_unsorted_duplicated_input_is_canonicalised(orc, ctx):
    rng = np.random.default_rng(4)
    w = synth.make("tiny")
    messy = []
    for (nr, nc, rp, ci) in w.mats:
        rows = [list(ci[rp[r]:rp[r + 1]]) for r in range(nr)]
        rows = [list(rng.permutation(r + r[: len(r) // 2])) for r in rows]       # duplicates + shuffled
        nrp = np.zeros(nr + 1, dtype=np.int64)
        np.cumsum([len(r) for r in rows], out=nrp[1:])
        messy.append((nr, nc, nrp, np.array([c for r in rows for c in r], dtype=np.int32)))
    assert_indicators_equal(oracle_train(orc, w.mats, w.params, 8), ctx.train_csr(messy, w.params, seed=8), w.mats[0][0])


# ---- golden fixtures of the reference ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["handmade.json", "item_sets.json", "movielens_sample.json"])
def test_golden_fixtures_through_reference_interface(ctx, name):
    fx = load_golden(name)
    prepared = prepared_from_fixture(fx)
    ds = [ur.DownsamplableCrossOccurrenceDataset(d, p[0], p[1], p[2]) for (_, d), p in zip(prepared, fx["params"])]
    out = ur.SimilarityAnalysis.crossOccurrenceDownsampled(ds, randomSeed=1, ctx=ctx)
    want = fx["oracle"]["indicators"]
    a_items = prepared[0][1].column_ids.inverse
    for (ev, d), ind in zip(prepared, out):
        assert ind.row_ids is prepared[0][1].column_ids and ind.column_ids is d.column_ids     # A.create(drm, A.columnIDs, B.columnIDs)
        cols = d.column_ids.inverse
        for row, item in enumerate(a_items):
            c, v = ind.row(row)
            assert [cols[int(x)] for x in c] == [r[0] for r in want[ev][item]], (ev, item)
            assert np.allclose(v, [r[1] for r in want[ev][item]], rtol=LLR_RTOL, atol=0)
        # the consumer's view (package.scala:82-110): ordered id lists
        sm = ind.to_string_map(ev)
        for item in a_items:
            assert sm[item][ev] == [r[0] for r in want[ev][item]]


def test_handmade_expected_file_constraints(ctx):
    fx = load_golden("handmade.json")
    prepared = prepared_from_fixture(fx)
    out = ur.SimilarityAnalysis.cooccurrencesIDSs([d for _, d in prepared], randomSeed=1, ctx=ctx)
    for (ev, _), ind in zip(prepared, out):
        sm = ind.to_string_map(ev)
        assert sm["Galaxy"][ev] == [] and sm["Iphone 5"][ev] == []        # integration-test-expected.txt:48-50
        assert "Surface" not in sm                                           # :52-54


# ---- debug entries: every stage against the oracle ------------------------------------------------------------------------
def test_device_llr_known_answers_and_oracle(orc, ctx):
    kats = load_golden("llr_kats.json")["kats"]
    k = np.array([x[:4] for x in kats], dtype=np.int64)
    got = ctx.debug_llr(k[:, 0], k[:, 1], k[:, 2], k[:, 3])
    assert np.allclose(got, [x[4] for x in kats], rtol=5e-7)
    rng = np.random.default_rng(0)
    n = 20000
    N = rng.integers(10, 10 ** 7, n)
    ra = (rng.random(n) * np.minimum(N, 600)).astype(np.int64) + 1
    cb = (rng.random(n) * np.minimum(N, 600)).astype(np.int64) + 1
    k11 = (rng.random(n) * np.minimum(ra, cb)).astype(np.int64)
    k12, k21 = ra - k11, cb - k11
    k22 = np.maximum(N - ra - cb + k11, 0)
    for flags in (0, ur.FLAG_ENTROPY_VARARGS):
        dev = ctx.debug_llr(k11, k12, k21, k22, flags)
        ref = np.array([orc.llr(*map(int, t), flags) for t in zip(k11, k12, k21, k22)])
        # 2 eps(N) of each cell's own N, the cancellation-limited cells (SURVEY.md 7 "fp64 cancellation") included
        bar = np.array([llr_bar(x) for x in k11 + k12 + k21 + k22])
        worst = np.argmax(np.abs(dev - ref) / bar)
        assert (np.abs(dev - ref) <= bar).all(), (flags, k11[worst], k12[worst], k21[worst], k22[worst], dev[worst], ref[worst])
    with pytest.raises(ur.CcoInvalidArgument):
        ctx.debug_llr([-1], [1], [1], [1])                            # Preconditions.checkArgument(k >= 0)


def test_device_downsample_bit_exact(orc, ctx):
    w = synth.make("small")
    nr, nc, rp, ci = w.mats[1]
    for m, flags in ((500, 0), (40, 0), (40, ur.FLAG_ROWRATE_INTDIV), (10 ** 9, 0)):
        d, raw, new = orc.downsample(orc.Csr(nr, nc, rp, ci), min(m, 2 ** 31 - 1), 77, flags)
        grp, gci, graw, gnew = ctx.debug_downsample(nr, nc, rp, ci, min(m, 2 ** 31 - 1), 77, flags)
        assert np.array_equal(grp, d.row_ptr) and np.array_equal(gci, d.col_idx)
        assert np.array_equal(graw, raw) and np.array_equal(gnew, new)


def test_device_cooccurrence_counts_bit_exact(orc, ctx):
    w = synth.make("tiny")
    a, b = w.mats[0], w.mats[1]
    for x, y in ((a, b), (a, a)):
        rp, ci, cn = ctx.debug_cooccurrence(x, y)
        orp, oci, ocn = orc.cooccurrence(orc.Csr(*x), orc.Csr(*y))
        assert np.array_equal(rp, orp) and np.array_equal(ci, oci) and np.array_equal(cn, ocn)


# ---- accumulator variants -----------------------------------------------------------------------------------------------------
def test_dense_and_hashed_tables_agree_with_oracle(orc, ctx):
    # n_cols = 300 -> direct-indexed (dense) tables in every bin; n_cols = 70000 -> hashed tables in every bin
    rng = np.random.default_rng(12)
    for n_items in (300, 70_000):
        nu = 4000
        mats = []
        for t in range(2):
            u = rng.integers(0, nu, 60_000)
            i = (rng.zipf(1.3, 60_000) - 1) % n_items
            rp, ci = synth.to_binary_csr(u.astype(np.int64), i.astype(np.int64), nu, n_items)
            mats.append((nu, n_items, rp, ci))
        params = [(500, 20, None)] * 2
        assert_indicators_equal(oracle_train(orc, mats, params, 1), ctx.train_csr(mats, params, seed=1), mats[0][0], f"n_items={n_items}")


def test_multi_pass_rows(orc, ctx):
    # one primary item whose row touches more distinct columns than a shared-memory table holds -> hash-partition passes
    rng = np.random.default_rng(13)
    nu, ia, ib = 400, 3, 200_000
    a_rows = [[0] if u < 300 else [1] for u in range(nu)]
    b_rows = [sorted(set(rng.integers(0, ib, 400).tolist())) for _ in range(nu)]
    def csr(rows, nc):
        rp = np.zeros(len(rows) + 1, dtype=np.int64)
        np.cumsum([len(r) for r in rows], out=rp[1:])
        return (len(rows), nc, rp, np.array([c for r in rows for c in r], dtype=np.int32))
    mats = [csr(a_rows, ia), csr(b_rows, ib)]
    params = [(10 ** 6, 50, None), (10 ** 6, 50, None)]
    ref = oracle_train(orc, mats, params, 2)
    assert ref[1].distinct_cells > 100_000
    assert_indicators_equal(ref, ctx.train_csr(mats, params, seed=2), mats[0][0], "multi-pass")
    rp, ci, cn = ctx.debug_cooccurrence(mats[0], mats[1])
    orp, oci, ocn = orc.cooccurrence(orc.Csr(*mats[0]), orc.Csr(*mats[1]))
    assert np.array_equal(rp, orp) and np.array_equal(ci, oci) and np.array_equal(cn, ocn)


# ---- edge cases ---------------------------------------------------------------------------------------------------------------------
def test_empty_and_degenerate_inputs(orc, ctx):
    z = lambda nr, nc: (nr, nc, np.zeros(nr + 1, dtype=np.int64), np.zeros(0, dtype=np.int32))
    for mats in ([z(5, 4)], [z(5, 4), z(5, 0)], [z(0, 3)], [z(0, 0)]):
        params = [(500, 50, None)] * len(mats)
        assert_indicators_equal(oracle_train(orc, mats, params, 1), ctx.train_csr(mats, params, seed=1), mats[0][0])
    # one user, one item; an item everybody bought (LLR == 0 everywhere -> empty indicators)
    one = (1, 1, np.array([0, 1], dtype=np.int64), np.array([0], dtype=np.int32))
    assert_indicators_equal(oracle_train(orc, [one], [(500, 50, None)], 1), ctx.train_csr([one], [(500, 50, None)], seed=1), one[0])
    full = (6, 2, np.arange(0, 13, 2, dtype=np.int64), np.tile(np.array([0, 1], dtype=np.int32), 6))
    got = ctx.train_csr([full], [(500, 50, None)], seed=1)
    assert got[0][3][-1] == 0
    rowref.assert_matches(rowref.expected(ctx, [full], [(500, 50, None)], 1), got, "item everybody bought")


def test_error_behaviour(ctx):
    ok = (3, 3, np.array([0, 1, 2, 3], dtype=np.int64), np.array([0, 1, 2], dtype=np.int32))
    with pytest.raises(ur.CcoInvalidArgument):      # rows must be shared (Preparator.scala:47-77)
        ctx.train_csr([ok, (4, 3, np.array([0, 1, 2, 3, 3], dtype=np.int64), np.array([0, 1, 2], dtype=np.int32))], [(500, 50, None)] * 2, 1)
    with pytest.raises(ur.CcoInvalidArgument):      # column out of range
        ctx.train_csr([(3, 3, np.array([0, 1, 2, 3], dtype=np.int64), np.array([0, 1, 5], dtype=np.int32))], [(500, 50, None)], 1)
    with pytest.raises(ur.CcoInvalidArgument):      # row_ptr not monotone
        ctx.train_csr([(3, 3, np.array([0, 2, 1, 3], dtype=np.int64), np.array([0, 1, 2], dtype=np.int32))], [(500, 50, None)], 1)
    with pytest.raises(ur.CcoInvalidArgument):      # k >= 1, m >= 1
        ctx.train_csr([ok], [(500, 0, None)], 1)
    with pytest.raises(ur.CcoInvalidArgument):
        ctx.train_csr([ok], [(0, 5, None)], 1)
    with pytest.raises(ur.CcoError) as e:           # documented limit
        ctx.train_csr([ok], [(500, 5000, None)], 1)
    assert e.value.status == -6
    # the context stays usable after errors
    assert len(ctx.train_csr([ok], [(500, 50, None)], 1)) == 1


def test_determinism_and_seed_sensitivity(ctx):
    w = synth.make("small")
    a = ctx.train_csr(w.mats, w.params, seed=11)
    b = ctx.train_csr(w.mats, w.params, seed=11)
    c = ctx.train_csr(w.mats, w.params, seed=12)
    for x, y in zip(a, b):
        assert all(np.array_equal(p, q) for p, q in zip(x[3:], y[3:]))
    assert any(not np.array_equal(x[4], y[4]) for x, y in zip(a, c))      # downsampling is active in 'small'


def test_dataset_api_matches_one_shot(ctx):
    w = synth.make("small")
    one = ctx.train_csr(w.mats, w.params, seed=4)
    ds = ctx.upload(w.mats)
    two = ctx.train_dataset(ds, w.params, seed=4)
    three = ctx.train_dataset(ds, [(100, 7, None)] * 3, seed=4)
    ctx.free_dataset(ds)
    for x, y in zip(one, two):
        assert all(np.array_equal(p, q) for p, q in zip(x[3:], y[3:]))
    assert max(np.diff(three[0][3])) <= 7


# ---- full size: BASELINE.json configs[2] (C3) against the oracle, plus size-independent properties -----------------------------------
def test_c3_full_size_against_oracle(orc, ctx):
    from oracle import parity as par
    w = synth.make("C3", ctx=ctx)
    res = ctx.train_csr(w.mats, w.params, seed=42, flags=ur.FLAG_ASSUME_CANONICAL)
    st = ctx.last_stats
    ref = oracle_train(orc, w.mats, w.params, 42)
    par.assert_ok(par.compare(ref, res, w.n_users), "C3 full size")
    assert st.products == [r.products for r in ref] and st.distinct_cells == [r.distinct_cells for r in ref]
    n_items = w.n_items
    for i, (rb, re_, nc, rp, ci, ll, cn) in enumerate(res):
        assert (rb, re_, nc) == (0, n_items, n_items)
        lens = np.diff(rp)
        assert lens.max() <= 50 and rp[-1] == len(ci) == len(ll) == len(cn)
        assert (ll > 0).all() and (cn >= 1).all() and (ci >= 0).all() and (ci < n_items).all()
        # rows sorted by (llr desc, col asc): inside a row llr never increases, ties have ascending columns
        same_row = np.repeat(np.arange(n_items), lens)
        inner = same_row[1:] == same_row[:-1]
        assert (ll[1:][inner] <= ll[:-1][inner]).all()
        tie = inner & (ll[1:] == ll[:-1])
        assert (ci[1:][tie] > ci[:-1][tie]).all()
        if i == 0:
            assert (ci != same_row).all()                       # A'^T A': the diagonal is excluded
    # idempotence
    again = ctx.train_csr(w.mats, w.params, seed=42, flags=ur.FLAG_ASSUME_CANONICAL)
    for x, y in zip(res, again):
        assert all(np.array_equal(p, q) for p, q in zip(x[3:], y[3:]))


def test_downsampling_dominated_million_column_shape(orc, ctx):
    """BASELINE.json configs[3] (C4) at a tenth of the users and events: 1M-column item space (hashed tables in every bin,
    12 count bits), Zipf-hot columns far above m = 500 (column downsampling removes most of their entries), users above m,
    minEventsPerUser = 3 applied when the CSR is built -- against the oracle, bit for bit."""
    from oracle import parity as par
    w = synth.make("C4-tenth", ctx=ctx)
    assert w.n_users < 1_000_000                                  # the duplicate-counting minEventsPerUser filter bit
    raw_col = np.bincount(w.mats[0][3], minlength=w.n_items)
    assert raw_col.max() > 50 * 500 and (raw_col > 500).sum() > 1000
    res = ctx.train_csr(w.mats, w.params, seed=42, flags=ur.FLAG_ASSUME_CANONICAL)
    st = ctx.last_stats
    ref = oracle_train(orc, w.mats, w.params, 42)
    par.assert_ok(par.compare(ref, res, w.n_users), "C4-tenth")
    assert st.nnz_downsampled == [r.nnz_b for r in ref]
    assert st.nnz_downsampled[0] < 0.8 * len(w.mats[0][3])       # downsampling really dominates
    # intdiv row rate (the literal Mahout recall) on the same shape
    got = ctx.train_csr(w.mats, w.params, seed=42, flags=ur.FLAG_ASSUME_CANONICAL | ur.FLAG_ROWRATE_INTDIV)
    par.assert_ok(par.compare(oracle_train(orc, w.mats, w.params, 42, ur.FLAG_ROWRATE_INTDIV), got, w.n_users), "C4-tenth intdiv")


# ---- documented limits (include/cco_b200.h "Limits"): clean errors, never wrong results -------------------------------------------
def _csr_from_rows(rows, nc):
    rp = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=rp[1:])
    return (len(rows), nc, rp, np.array([c for r in rows for c in r], dtype=np.int32))


def test_packed_word_limit_is_a_clean_error_and_downsampling_lifts_it(orc, ctx):
    # 3M columns leave 10 count bits in the packed (key, count) word.  One (a, b) pair co-occurs 3000 times: without
    # downsampling that count does not fit -> CCO_E_UNSUPPORTED with a message that names the remedy; with the reference's
    # default m = 500 every marginal (hence every count) is <= ~560 and the same matrices train and match the oracle.
    rng = np.random.default_rng(21)
    nu, ia, ib = 5000, 40, 3_000_000
    hot_b = [7, 2_999_999, 1_500_001]
    a_rows, b_rows = [], []
    for u in range(nu):
        a = set(rng.integers(1, ia, 2).tolist())
        b = set(rng.integers(0, ib, 6).tolist())
        if u < 3000:
            a.add(0)
            b.update(hot_b)
        a_rows.append(sorted(a))
        b_rows.append(sorted(b))
    mats = [_csr_from_rows(a_rows, ia), _csr_from_rows(b_rows, ib)]
    with pytest.raises(ur.CcoError) as e:
        ctx.train_csr(mats, [(10 ** 6, 50, None)] * 2, seed=2)
    assert e.value.status == -6 and "maxItemsPerUser" in str(e.value)
    params = [(500, 50, None), (500, 50, None)]
    assert_indicators_equal(oracle_train(orc, mats, params, 2), ctx.train_csr(mats, params, seed=2), mats[0][0], "3M columns, m=500")
