"""Indicators trained in key ranges (include/cco_b200.h CCO_FLAG_KEY_RANGES, DESIGN.md 3.1 "key ranges"), bit for bit:
columns, counts and LLR bit patterns against the brute-force reference of tests/rowref.py, the oracle and the unsplit
run.  Past the packed-word limit the flag trains what is otherwise refused; where the word fits, the debug cap
(cco_debug_key_range_cap) forces ranges through every row path, and the flag alone changes nothing.  The device's
last_key_ranges equal the host restatement of the plan (tests/key_ranges_ref.py) in every case."""
import json

import numpy as np
import pytest

import key_ranges_ref as kr
import row_paths
import rowref
import synth
import universal_recommender_b200 as ur
from conftest import load_golden, prepared_from_fixture
from test_gpu_parity import assert_indicators_equal, oracle_train

pytestmark = pytest.mark.gpu
M_ALL = 10 ** 6


@pytest.fixture
def capped(ctx):
    """ctx with a debug key-range cap set by the test; the cap is off again afterwards (ctx is shared)."""
    yield ctx
    ctx.debug_key_range_cap(0)


def csr_from_pairs(users, items, nu, ni):
    rp, ci = synth.to_binary_csr(np.asarray(users, np.int64), np.asarray(items, np.int64), nu, ni)
    return (nu, ni, rp, ci)


def expected_ranges(mats, params, seed, flags=0, cap=0):
    sm = rowref.sampled(mats, params, seed, flags)
    max_a = int(sm[0][1].max(initial=0))
    return [kr.n_ranges(marg, max_a, cap) for _, marg in sm]


def same_arrays(x, y, tag):
    assert len(x) == len(y), tag
    for i, (p, q) in enumerate(zip(x, y)):
        assert p[:3] == q[:3], f"{tag} indicator {i}: shape"
        for name, a, b in (("row_ptr", p[3], q[3]), ("columns", p[4], q[4]), ("counts", p[6], q[6]),
                           ("LLR bits", np.asarray(p[5]).view(np.uint64), np.asarray(q[5]).view(np.uint64))):
            assert np.array_equal(a, b), f"{tag} indicator {i}: {name} differ"


def split_vs_unsplit(ctx, mats, params, cap, seed=1, flags=0, tag=""):
    """The same train unsplit and capped: identical arrays and products / distinct cells, the reference bit for bit,
    and the plan the host restatement cuts."""
    ctx.debug_key_range_cap(0)
    whole = ctx.train_csr(mats, params, seed=seed, flags=flags)
    st0 = ctx.last_stats
    assert ctx.last_key_ranges == [1] * len(mats)
    ctx.debug_key_range_cap(cap)
    got = ctx.train_csr(mats, params, seed=seed, flags=flags)
    st1 = ctx.last_stats
    same_arrays(whole, got, f"{tag} cap={cap}")
    assert st1.products == st0.products and st1.distinct_cells == st0.distinct_cells, tag
    assert ctx.last_key_ranges == expected_ranges(mats, params, seed, flags, cap), tag
    if not flags & (ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR):
        rowref.assert_matches(rowref.expected(ctx, mats, params, seed, flags), got, f"{tag} cap={cap}")
    return got


# ---- forced ranges where the word fits -----------------------------------------------------------------------------------
def _dense_hashed(n_items, seed):
    rng = np.random.default_rng(seed)
    nu = 4000
    mats = []
    for _ in range(2):
        u = rng.integers(0, nu, 60_000)
        i = (rng.zipf(1.3, 60_000) - 1) % n_items
        mats.append(csr_from_pairs(u, i, nu, n_items))
    return mats


def _multi_pass():
    # one primary item whose row touches more distinct columns than a shared-memory table holds
    rng = np.random.default_rng(13)
    nu, ia, ib = 400, 3, 200_000
    ua = np.arange(nu)
    a = csr_from_pairs(ua, np.where(ua < 300, 0, 1), nu, ia)
    ub = np.repeat(np.arange(nu), 400)
    b = csr_from_pairs(ub, rng.integers(0, ib, len(ub)), nu, ib)
    return [a, b]


SHAPES = {
    "tiny": (lambda: synth.make("tiny").mats, [1, 2, 31, 32, 33]),
    "small": (lambda: synth.make("small").mats, [31, 33, 1700]),
    "C2": (lambda: synth.make("C2").mats, [32, 1333]),
    "dense300": (lambda: _dense_hashed(300, 12), [1, 2, 31, 32, 33]),
    "hashed70k": (lambda: _dense_hashed(70_000, 12), [33, 23_334]),
    "multi-pass": (lambda: _multi_pass(), [66_667]),
}


@pytest.mark.parametrize("shape", list(SHAPES))
def test_forced_ranges_equal_the_unsplit_run(capped, shape):
    make, caps = SHAPES[shape]
    mats = make()
    for m in (500, M_ALL):
        params = [(m, 20, None)] * len(mats)
        for cap in caps:
            split_vs_unsplit(capped, mats, params, cap, tag=f"{shape} m={m}")


@pytest.mark.parametrize("params,flags", [
    ([(500, 1, None)] * 3, 0),
    ([(500, 2048, None)] * 3, 0),
    ([(500, 10, None), (500, 3, 2.0), (20, 64, 0.25)], 0),
    ([(500, 20, None)] * 3, ur.FLAG_ENTROPY_VARARGS),
    ([(40, 20, None)] * 3, ur.FLAG_ROWRATE_INTDIV),
    ([(500, 20, None)] * 3, ur.FLAG_RESULT_NO_COUNT),
    ([(500, 20, None)] * 3, ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR),
], ids=["k1", "k2048", "min_llr", "varargs", "intdiv", "no_count", "no_llr"])
def test_forced_ranges_params_and_flags(capped, params, flags):
    mats = synth.make("small").mats
    for cap in (33, 1024):
        split_vs_unsplit(capped, mats, params, cap, seed=9, flags=flags, tag=f"flags={flags}")


def test_cap_splits_a_run_of_equal_colb_with_the_cut_on_a_tie(capped, orc):
    # columns 0..11 share colB = 5 and co-occur once with item 0: twelve cells of one LLR.  top_k = 6 cuts inside the
    # tie and the caps split the run across ranges: the kept cells must be the six lowest column ids
    nu, ia, ib = 400, 4, 40
    us, bs = [], []
    for j in range(12):
        for u in (j, 100 + j, 120 + j, 140 + j, 160 + j):
            us.append(u)
            bs.append(j)
    for j in range(12, ib):     # other colB values around the run
        for u in range(200 + j, 200 + j + (j % 7) + 1):
            us.append(u)
            bs.append(j)
    b = csr_from_pairs(us, bs, nu, ib)
    a = csr_from_pairs(list(range(12)) + list(range(200, 260)), [0] * 12 + [1 + (u % 3) for u in range(200, 260)], nu, ia)
    params = [(M_ALL, 6, None), (M_ALL, 6, None)]
    for cap in (1, 2, 4, 5, 7):
        got = split_vs_unsplit(capped, [a, b], params, cap, tag="tie run")
        _, _, _, rp, ci, ll, _ = got[1]
        assert list(ci[rp[0]:rp[1]]) == [0, 1, 2, 3, 4, 5]
        assert len(set(ll[rp[0]:rp[1]].tolist())) == 1
    assert_indicators_equal(oracle_train(orc, [a, b], params, 1), got, a[0], "tie run")


def test_forced_ranges_golden_fixtures(capped):
    for name in ("handmade.json", "item_sets.json", "movielens_sample.json"):
        fx = load_golden(name)
        prepared = prepared_from_fixture(fx)
        ds = [ur.DownsamplableCrossOccurrenceDataset(d, p[0], p[1], p[2]) for (_, d), p in zip(prepared, fx["params"])]
        capped.debug_key_range_cap(0)
        whole = ur.SimilarityAnalysis.crossOccurrenceDownsampled(ds, randomSeed=1, ctx=capped)
        mats = [(d.iD.n_rows, d.iD.n_cols, d.iD.row_ptr, d.iD.col_idx) for d in ds]
        params = [(d.maxElementsPerRow, d.maxInterestingElements, d.minLLROpt) for d in ds]
        for cap in (1, 2, 3):
            capped.debug_key_range_cap(cap)
            split = ur.SimilarityAnalysis.crossOccurrenceDownsampled(ds, randomSeed=1, ctx=capped)
            assert capped.last_key_ranges == expected_ranges(mats, params, 1, 0, cap), (name, cap)
            for x, y in zip(whole, split):
                for r in range(len(x.row_ids)):
                    (c0, v0), (c1, v1) = x.row(r), y.row(r)
                    assert np.array_equal(c0, c1) and np.array_equal(np.asarray(v0).view(np.uint64), np.asarray(v1).view(np.uint64)), \
                        (name, cap, r)


def test_forced_ranges_debug_cooccurrence_emit_all(capped, orc):
    w = synth.make("tiny")
    a, b = w.mats[0], w.mats[1]
    for x, y in ((a, b), (a, a)):
        orp, oci, ocn = orc.cooccurrence(orc.Csr(*x), orc.Csr(*y))
        for cap in (1, 2, 31, 32, 33):
            capped.debug_key_range_cap(cap)
            rp, ci, cn = capped.debug_cooccurrence(x, y)
            assert np.array_equal(rp, orp) and np.array_equal(ci, oci) and np.array_equal(cn, ocn), cap


def test_forced_ranges_train_dataset_and_group_context(capped):
    w = synth.make("small")
    capped.debug_key_range_cap(0)
    one = capped.train_csr(w.mats, w.params, seed=4)
    capped.debug_key_range_cap(64)
    ds = capped.upload(w.mats)
    try:
        two = capped.train_dataset(ds, w.params, seed=4)
    finally:
        capped.free_dataset(ds)
    same_arrays(one, two, "train_dataset")
    assert capped.last_key_ranges == expected_ranges(w.mats, w.params, 4, 0, 64)
    g = ur.CcoContext(devices=[0])
    try:
        g.debug_key_range_cap(64)
        three = g.train_csr(w.mats, w.params, seed=4)
        assert g.last_key_ranges == expected_ranges(w.mats, w.params, 4, 0, 64)
    finally:
        g.close()
    same_arrays(one, three, "group context")


# ---- the flag where the word fits: nothing changes ----------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny", "small"])
def test_flag_where_the_word_fits_changes_nothing(ctx, name):
    w = synth.make(name)
    off = ctx.train_csr(w.mats, w.params, seed=3)
    n_off = ctx.last_stats.n_kernel_launches
    on = ctx.train_csr(w.mats, w.params, seed=3, flags=ur.FLAG_KEY_RANGES)
    assert ctx.last_stats.n_kernel_launches == n_off
    assert ctx.last_key_ranges == [1] * len(w.mats)
    same_arrays(off, on, name)


# ---- past the packed-word limit --------------------------------------------------------------------------------------------
def _limit_test_matrices():
    # test_gpu_parity's packed-word limit shape: 3M columns, one (a, b) pair co-occurring 3000 times
    rng = np.random.default_rng(21)
    nu, ia, ib = 5000, 40, 3_000_000
    hot_b = [7, 2_999_999, 1_500_001]
    us, as_, ub, bs = [], [], [], []
    for u in range(nu):
        a = set(rng.integers(1, ia, 2).tolist())
        b = set(rng.integers(0, ib, 6).tolist())
        if u < 3000:
            a.add(0)
            b.update(hot_b)
        us += [u] * len(a)
        as_ += sorted(a)
        ub += [u] * len(b)
        bs += sorted(b)
    return [csr_from_pairs(us, as_, nu, ia), csr_from_pairs(ub, bs, nu, ib)]


def _check_past_limit(orc, ctx, mats, params, seed, want_ranges, tag, brute=True):
    """brute=False: the oracle's train only (the brute-force reference scans every column per primary item)."""
    with pytest.raises(ur.CcoError) as e:
        ctx.train_csr(mats, params, seed=seed)
    assert e.value.status == -6 and "maxItemsPerUser" in str(e.value) and "CCO_FLAG_KEY_RANGES" in str(e.value)
    got = ctx.train_csr(mats, params, seed=seed, flags=ur.FLAG_KEY_RANGES)
    assert ctx.last_key_ranges == expected_ranges(mats, params, seed)
    assert ctx.last_key_ranges == want_ranges, tag
    if brute:
        rowref.assert_matches(rowref.expected(ctx, mats, params, seed), got, tag)
    ref = oracle_train(orc, mats, params, seed)
    assert_indicators_equal(ref, got, mats[0][0], tag)
    assert ctx.last_stats.products == [r.products for r in ref] and ctx.last_stats.distinct_cells == [r.distinct_cells for r in ref]
    return got


def test_limit_test_matrices_train_with_the_flag(orc, ctx):
    _check_past_limit(orc, ctx, _limit_test_matrices(), [(M_ALL, 50, None)] * 2, 2, [1, 2], "3M columns, m=10^6")


def test_16m_column_secondary_at_default_m(orc, ctx):
    # 16M-column secondary, m = 500: 40 hot columns (~2400 raw users each) sample to marginals around 500, some >= 512,
    # and so does the primary's largest marginal; 16M columns take 25 key bits and leave 7 count bits
    rng = np.random.default_rng(31)
    nu, ia, ib, n_hot = 24_000, 30, 16_777_216, 40
    users = np.arange(nu)
    a = csr_from_pairs(np.repeat(users, 3), rng.integers(0, ia, nu * 3), nu, ia)
    hot = (rng.integers(0, n_hot, nu * 4) * 400_009) % ib
    cold = rng.integers(0, ib, nu * 8)
    b = csr_from_pairs(np.concatenate([np.repeat(users, 4), np.repeat(users, 8)]), np.concatenate([hot, cold]), nu, ib)
    mats, params = [a, b], [(500, 50, None)] * 2
    sm = rowref.sampled(mats, params, 2)
    assert sm[0][1].max() >= 512 and sm[1][1].max() >= 512
    _check_past_limit(orc, ctx, mats, params, 2, [1, 2], "16M columns, m=500")


def test_self_indicator_past_the_limit(orc, ctx):
    # a 5M-column primary whose hot columns are bought by 600 users each: 23 key bits leave 9 count bits, so A'^T A'
    # runs in ranges; the diagonal (each key's own column, in whichever range holds it) is never kept
    rng = np.random.default_rng(5)
    nu, ia, n_hot = 1000, 5_000_000, 12
    users = np.arange(nu)
    hot = rng.choice(ia, n_hot, replace=False)
    pu = np.concatenate([users, np.repeat(users[:600], n_hot)])
    pi = np.concatenate([rng.integers(0, ia, nu), np.tile(hot, 600)])
    a = csr_from_pairs(pu, pi, nu, ia)
    got = _check_past_limit(orc, ctx, [a], [(M_ALL, 5, None)], 3, [2], "self, 5M columns", brute=False)
    _, _, _, rp, ci, _, _ = got[0]
    rows = np.repeat(np.arange(ia), np.diff(rp))
    assert len(ci) > 0 and (ci != rows).all()


# ---- directed row-kernel shapes, split: every bin, dense and hashed tables, bitmap and sorted rows, multi-pass -------------
def range_views(mats, params, cap, seed=1):
    """[(n_r, max colB of the range, per-item work over B'_r)] of indicator 1 as the device splits it (the plan of
    key_ranges_ref over the key order (colB ascending, column id ascending))"""
    sm = rowref.sampled(mats, params, seed)
    (a, marg_a), (b, marg_b) = sm[0], sm[1]
    key_col = np.lexsort((np.arange(len(marg_b)), marg_b))       # key -> column
    key_of_col = np.empty_like(key_col)
    key_of_col[key_col] = np.arange(len(key_col))
    mk = marg_b[key_col]
    b_users = np.repeat(np.arange(b.n_rows), np.diff(b.row_ptr))
    b_keys = key_of_col[b.col_idx]
    a_users = np.repeat(np.arange(a.n_rows), np.diff(a.row_ptr))
    out = []
    for k0, k1 in kr.plan(mk, int(marg_a.max()), cap):
        inr = (b_keys >= k0) & (b_keys < k1)
        deg = np.bincount(b_users[inr], minlength=b.n_rows)
        work = np.bincount(a.col_idx, weights=deg[a_users], minlength=a.n_cols).astype(np.int64)
        out.append((k1 - k0, int(mk[k1 - 1]), work))
    return out, int(marg_a.max()), marg_a[:a.n_cols], int(a.n_rows)


def range_paths(mats, params, cap):
    """Per range: the set of (bin, group, table, score path, cut, passes, bitmap, sorted) the rows with work take there
    (row_paths.row_path and the bitmap / sorted bin restatements of their test modules, on the range's view)"""
    from test_gpu_bitmap_rows import bitmap_bins
    from test_gpu_sorted_rows import sorted_bins
    views, max_a, ra, n = range_views(mats, params, cap)
    top_k = params[1][1]
    out = []
    for n_r, mm, work in views:
        bm = bitmap_bins(top_k, n_r, max_a, mm, n)
        so = sorted_bins(top_k, n_r, max_a, mm, n)
        cells = set()
        for w, r in zip(work, ra):
            p = row_paths.row_path(int(w), int(r), n_r, max_a, mm, n, top_k)
            if p is not None:
                cells.add(p.cell() + (p.bin in bm, p.bin in so))
        out.append(cells)
    return out


@pytest.mark.parametrize("case", ["bins-hashed", "bins-dense", "bitmap", "sorted"])
def test_forced_ranges_directed_row_paths(capped, case):
    from test_gpu_row_paths import BOUNDARIES, CAP, work_rows
    # caps chosen so that both ranges hold columns with products (the colB = 0 keys come first) and stay wide enough for
    # the path named: hashed tables need more keys than the bin's table, bitmap rows a hashed 256- or 512-thread bin
    if case == "bins-hashed":     # every bin hashed, the 1024-thread bin multi-pass: two ranges of 70 000 keys
        mats, cap = work_rows(BOUNDARIES + [CAP, CAP + 1, 30_000, 50_000], 140_000, True, seed=11), 70_000
    elif case == "bins-dense":    # dense tables in every bin on 150-key ranges
        mats, cap = work_rows(BOUNDARIES, 300, True, seed=12), 150
    elif case == "bitmap":        # bitmap rows in both ranges
        mats, cap = work_rows([2048, 2049, 3000, 4096, 4097, 6000, 8192, 8193], 70_001, True, seed=11), 55_000
    else:                         # the warp bins' sorted rows in both ranges
        mats, cap = work_rows([1, 31, 32, 33, 256, 257, 512, 513, 1024], 70_001, True, seed=21), 67_500
    params = [(10 ** 9, 50, None)] * 2
    split_vs_unsplit(capped, mats, params, cap, tag=case)
    per_range = range_paths(mats, params, cap)
    assert len(per_range) == 2
    cells = set().union(*per_range)
    groups = {c[0] for c in cells}
    if case == "bins-hashed":
        assert all({c[0] for c in r} == {32, 128, 256, 512, 1024} for r in per_range)
        assert {c[1] for c in cells} == {"hash"} and any(c[4] == "multi" for c in cells)
    elif case == "bins-dense":
        assert groups == {32, 128, 256, 512, 1024} and {c[1] for c in cells} == {"dense"}
    elif case == "bitmap":
        assert all(any(c[5] for c in r) for r in per_range)      # bitmap rows in both ranges
    else:
        assert all(any(c[6] for c in r) for r in per_range)      # sorted rows in both ranges


# ---- end to end: a PredictionIO export whose item space passes the limit ---------------------------------------------------
def test_calc_all_from_events_passes_the_flag(ctx):
    # 32 768 users each buy the two hot items and two cold ones, 1 000 more users one cold item each (so that the hot
    # pair is not bought by everybody): 66 538 items take 17 key bits and leave 15 count bits, and the hot pair
    # co-occurs 32 768 times -- past the word at maxEventsPerEventType = 10^6
    n, extra = 32_768, 1_000
    t0 = b'"eventTime":"2020-01-01T00:00:00Z"'
    line = b'{"event":"buy","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"%s",%s}'
    lines = []
    for u in range(n):
        for it in (b"h0", b"h1", b"c%d" % (2 * u), b"c%d" % (2 * u + 1)):
            lines.append(line % (u, it, t0))
    for u in range(n, n + extra):
        lines.append(line % (u, b"c%d" % (n + u), t0))
    data = b"\n".join(lines) + b"\n"
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy"], "seed": 1, "recsModel": "collabFiltering",
                                                "maxEventsPerEventType": 10 ** 6, "maxCorrelatorsPerEventType": 20})
    with pytest.raises(ur.CcoError) as e:
        ur.calc_all_from_events(data, ap, 0, now_ms=10 ** 12, ctx=ctx)
    assert e.value.status == -6 and "CCO_FLAG_KEY_RANGES" in str(e.value)
    body = ur.calc_all_from_events(data, ap, 0, now_ms=10 ** 12, ctx=ctx, flags=ur.FLAG_KEY_RANGES)
    got = {}
    for line in body.decode().splitlines()[1::2]:
        d = json.loads(line)
        if d.get("buy"):
            got[d["id"]] = d["buy"]
    # the same CSR through train_csr
    log = ctx.read_events(data)
    try:
        ds, _, items = ctx.ingest_event_log(log, ["buy"], 0)
        try:
            mat = ctx.dataset_to_host(ds, 0, pinned=False)
        finally:
            ctx.free_dataset(ds)
    finally:
        log.free()
    from universal_recommender_b200 import ur_algorithm as ua
    seed, flags = ua._seed_and_flags(ap, ur.FLAG_KEY_RANGES)
    res = ctx.train_csr([mat], ua._indicator_params(ap, ["buy"]), seed=seed, flags=flags)
    assert ctx.last_key_ranges == [2]
    _, _, _, rp, ci, _, _ = res[0]
    ids = items[0]
    want = {ids[r]: [ids[c] for c in ci[rp[r]:rp[r + 1]]] for r in range(len(ids)) if rp[r + 1] > rp[r]}
    assert got == want
    assert got["h0"][0] == "h1" and got["h1"][0] == "h0"
