"""Directed row-kernel cases: hand-made inputs that put rows on each path of `k_rows` (bin and owner, dense or hashed
table, passes, keyed or colB scoring, key-cut depth or no cut, single-warp or CTA-wide select, top_k splits), each checked
bit for bit against the brute-force reference of tests/rowref.py and against the oracle.  Every case asserts, through
the path model of tests/row_paths.py, that it reaches the path it names; the last test checks and prints which
(owner x table x score path x cut x passes) cells the module covered."""
import numpy as np
import pytest

import row_paths
import rowref
import universal_recommender_b200 as ur
from test_gpu_parity import assert_indicators_equal, oracle_train

pytestmark = pytest.mark.gpu
M_ALL = 10 ** 9          # max_interactions above every row and column count: downsampling is the identity
COVERED = set()     # RowPath.cell() of every row a directed case ran
RAN = set()         # node ids of the tests of this module that have run


@pytest.fixture(autouse=True)
def _record_ran(request):
    yield
    RAN.add(request.node.nodeid)


def csr(rows, nc, n_rows=None):
    n_rows = len(rows) if n_rows is None else n_rows
    rp = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows] + [0] * (n_rows - len(rows)), out=rp[1:])
    ci = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows]) if rows else np.zeros(0, np.int32)
    return (n_rows, nc, rp, ci.astype(np.int32))


def run(orc, ctx, mats, params, seed=1, flags=0, tag=""):
    """Train on the device; check against the reference (bit for bit) and the oracle; record the paths taken."""
    got = ctx.train_csr(mats, params, seed=seed, flags=flags)
    exp = rowref.expected(ctx, mats, params, seed, flags)
    rowref.assert_matches(exp, got, tag)
    assert_indicators_equal(oracle_train(orc, mats, params, seed, flags & 3), got, mats[0][0], tag)
    assert ctx.last_stats.distinct_cells == [e.distinct for e in exp]
    paths = [e.paths() for e in exp]
    for ps in paths:
        COVERED.update(p.cell() for p in ps if p is not None)
    return exp, paths, got


def pick(rng, n, d):
    if n <= 4096:
        return np.sort(rng.permutation(n)[:d])
    s = rng.permutation(np.unique(rng.integers(0, n, 3 * d)))[:d]
    assert len(s) == d
    return np.sort(s)


def work_rows(works, n_cols_b, keyed, seed, dmax=64):
    """Primary item i gets its own users; their B' rows (distinct random columns, <= dmax each) sum to works[i]
    products.  keyed: empty users are appended until 2 rowA max colB < N holds for every row."""
    rng = np.random.default_rng(seed)
    a_rows, b_rows = [], []
    for item, w in enumerate(works):
        d = min(dmax, n_cols_b)
        ra = -(-w // d)
        for i in range(ra):
            a_rows.append([item])
            b_rows.append(pick(rng, n_cols_b, w // ra + (1 if i < w % ra else 0)))
    n = len(a_rows)
    if keyed:
        max_cb = np.bincount(np.concatenate(b_rows), minlength=n_cols_b).max()
        max_ra = max(-(-w // min(dmax, n_cols_b)) for w in works)
        n = max(n, 2 * max_ra * int(max_cb) + 1)
    return [csr(a_rows, len(works), n), csr(b_rows, n_cols_b, n)]


CAP = row_paths.bins(50, 70_000)[0][1].cap      # hashed capacity of the 1024-thread bin at top_k 50 on an H100
BOUNDARIES = [256, 257, 512, 513, 1024, 1025, 2048, 2049, 4096, 4097, 8192, 8193, 20_000, 70_000]


@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "colB"])
@pytest.mark.parametrize("n_cols_b", [300, 70_000], ids=["dense", "hashed"])
def test_bin_boundaries(orc, ctx, n_cols_b, keyed):
    works = BOUNDARIES + ([CAP, CAP + 1, 30_000, 50_000] if n_cols_b > 45_056 else [])
    mats = work_rows(works, n_cols_b, keyed, seed=len(works) + n_cols_b)
    params = [(M_ALL, 50, None)] * 2
    exp, paths, _ = run(orc, ctx, mats, params, tag=f"bins {n_cols_b} keyed={keyed}")
    ps = paths[1]
    assert [int(w) for w in exp[1].work] == works
    _, h_thr = row_paths.bins(50, n_cols_b)
    for w, p in zip(works, ps):
        assert p.dense == (n_cols_b == 300)
        assert p.cut == (w < 65_536)
        if keyed:
            assert p.keyed
        b = row_paths.bin_of(w, h_thr)
        assert b == p.bin and (b == 0 or w <= h_thr[b - 1]) and w > h_thr[b]
    groups = {w: p.group for w, p in zip(works, ps)}
    assert [groups[w] for w in (256, 257, 512, 513, 1024, 1025, 2048, 2049, 4096, 4097, 8192, 8193)] == \
        [32, 32, 32, 32, 32, 128, 128, 256, 256, 512, 512, 1024]
    if n_cols_b > 45_056:
        passes = {w: p.n_pass for w, p in zip(works, ps)}
        assert passes[CAP] == 1 and passes[CAP + 1] == 2 and passes[30_000] == 2 and passes[50_000] == 3
    if not keyed:
        assert any(not p.keyed for p in ps)


@pytest.mark.parametrize("top_k", [64, 65, 128, 129, 224, 225, 400, 2048])
def test_top_k_splits(orc, ctx, top_k):
    # warp_ok ends at 224; next_pow2 of the candidate buffer / final select changes at 64/65 and 128/129; 400 makes
    # CTA-owned rows prune and finish with more than 512 candidates (CTA-wide radix select); 2048 exceeds every row
    works = [200, 257, 700, 1025, 3000, 9000, 30_000]
    mats = work_rows(works, 70_000, True, seed=top_k)
    exp, paths, _ = run(orc, ctx, mats, [(M_ALL, top_k, None)] * 2, tag=f"top_k={top_k}")
    groups = {p.group for p in paths[1]}
    assert (32 in groups) == (top_k <= 224)
    cfgs, _ = row_paths.bins(top_k, 70_000)
    if top_k == 400:
        assert any(c.group > 32 and c.cbuf - c.group > 512 for c in cfgs)   # prunes see > 512 candidates
    if top_k == 2048:
        assert np.diff(exp[1].row_ptr)[0] <= 200                           # a row keeps every positive cell


def test_count_phase_windows(orc, ctx):
    # CTA-owned rows whose users are mostly zero-degree: one user holds all of a window's products, windows with T = 0,
    # and user counts that are not multiples of 32
    rng = np.random.default_rng(5)
    a_rows, b_rows = [], []
    for item, (ra, heavy) in enumerate([(1000, [1500]), (2001, [2500, 2000]), (3003, [9000]), (333, [1100]), (77, [4500])]):
        for i in range(ra):
            a_rows.append([item])
            b_rows.append(pick(rng, 70_000, heavy[i]) if i < len(heavy) else [])
    n = 20_000_000 // 1000
    mats = [csr(a_rows, 5, n), csr(b_rows, 70_000, n)]
    _, paths, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, tag="count windows")
    assert [p.group for p in paths[1]] == [128, 512, 1024, 128, 512]


@pytest.mark.parametrize("n_cols_b", [300, 512, 513, 5000, 2 ** 18, 2 ** 18 + 1, 300_000])
@pytest.mark.parametrize("offset", [0, -1], ids=["bin-start", "bin-end"])
def test_key_cut_depths(orc, ctx, n_cols_b, offset):
    # One row, one user buying the last n_cells columns of B' (colB 1; every other column has colB 0, so the cells hold
    # the top keys).  n_cells puts the 50th smallest cell key on the first (offset 0) or the last (offset -1) key of a
    # level-1 cut bin (bins of 2^shift keys).
    s = 1 << row_paths.key_shift(n_cols_b)
    n_cells = (n_cols_b + 49 - offset) % s
    while n_cells < 100:
        n_cells += s
    n_cells = min(n_cells, n_cols_b)
    kth_key = n_cols_b - n_cells + 49
    assert s == 1 or kth_key % s == offset % s
    mats = [csr([[0]], 1, 10), csr([list(range(n_cols_b - n_cells, n_cols_b))], n_cols_b, 10)]
    exp, paths, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, tag=f"key cut {n_cols_b}")
    p = paths[1][0]
    assert p.keyed and p.cut and p.levels == row_paths.key_levels(n_cols_b)
    assert exp[1].col.tolist() == list(range(n_cols_b - n_cells, n_cols_b - n_cells + 50))


def test_colb_ties_straddle_the_cut_and_the_diagonal(orc, ctx):
    # 200 items bought by one user; item j also by (199 - j) // 40 more users, so colB runs of 40 equal values
    # straddle the k-th cell and column ids run against key order across runs.  In A'^T A' (k = 20) the row whose
    # diagonal is the 20th smallest key (item 179) cuts one key further.
    n_items = 200
    extra = [(n_items - 1 - j) // 40 for j in range(n_items)]
    rows = [list(range(n_items))] + [[j for j in range(n_items) if extra[j] > f] for f in range(max(extra))]
    n = 2 * (max(extra) + 1) * (max(extra) + 2) + 10
    m = csr(rows, n_items, n)
    params = [(M_ALL, 20, None), (M_ALL, 50, None)]
    exp, paths, _ = run(orc, ctx, [m, m], params, tag="ties")
    assert all(p.keyed and p.cut and p.group == 32 for ps in paths for p in ps if p is not None)
    # item 179: colA = 1, key 19 (keys 0..39 are items 160..199)
    assert exp[0].ra[179] == 1 and list(exp[0].col[exp[0].row_ptr[179]:exp[0].row_ptr[180]]) == \
        [j for j in range(160, 181) if j != 179]


def test_mixed_keyed_and_colb_rows_and_colb_cut_at_511_512(orc, ctx):
    # max colB 2100 in N = 8000: rows with rowA = 1 are keyed, rowA = 2 are not.  The colB rows have 60 k11 = 1 cells
    # with colB 462 + i (resp. 463 + i): their 50th is at colB 511 (last cut bin) resp. 512 (outside the bins: no cut)
    n = 8000
    b_rows = [[] for _ in range(n)]
    target = {}
    for j in range(60):
        target[j] = 462 + j
        target[60 + j] = 463 + j
    for j in range(120, 170):
        target[j] = 3 + j % 7
    target[170] = 2100
    buyers = {0: range(0, 60), 2: range(60, 120), 4: range(120, 170)}
    for u, cs in buyers.items():
        b_rows[u].extend(cs)
    for j, cb in target.items():
        have = sum(1 for cs in buyers.values() if j in cs)
        for f in range(cb - have):
            b_rows[10 + f].append(j)
    b_rows = [sorted(r) for r in b_rows]
    a_rows = [[] for _ in range(n)]
    a_rows[0], a_rows[1], a_rows[2], a_rows[3], a_rows[4] = [0], [0], [1], [1], [2]
    mats = [csr(a_rows, 3, n), csr(b_rows, 171, n)]
    exp, paths, _ = run(orc, ctx, mats, [(M_ALL, 50, None)] * 2, tag="mixed")
    p0, p1, p2 = paths[1]
    assert not p0.keyed and not p1.keyed and p2.keyed and p0.cut and p1.cut
    cb = np.bincount(mats[1][3], minlength=171)
    kept0 = exp[1].col[exp[1].row_ptr[0]:exp[1].row_ptr[1]]
    assert len(kept0) == 50 and cb[kept0].max() == 511
    kept1 = exp[1].col[exp[1].row_ptr[1]:exp[1].row_ptr[2]]
    assert len(kept1) == 50 and cb[kept1].max() == 512


def test_min_llr_equal_to_a_cell_with_dominance(orc, ctx):
    # minLLR is exactly the LLR of some cell (inclusive); cells with k11 up to ~20 make the dominance filter record
    mats = work_rows([300, 700, 1500, 5000], 300, False, seed=77)
    base = rowref.expected(ctx, mats, [(M_ALL, 50, None)] * 2, 1)[1]
    ctx.train_csr(mats, [(M_ALL, 50, None)] * 2, seed=1)
    evaluated_without = ctx.last_stats.llr_evaluated[1]
    for row, rank in ((2, 25), (3, 49)):
        t = float(base.llr[base.row_ptr[row] + rank])
        exp, _, got = run(orc, ctx, mats, [(M_ALL, 50, t), (M_ALL, 50, t)], tag=f"minLLR={t!r}")
        assert (got[1][5] >= t).all() and (got[1][5] == t).any()
        # the filter dropped cells: the cut is the same with and without minLLR, so the evaluations it saved on top of
        # the run without minLLR come from frontiers recorded by cells failing minLLR
        st = ctx.last_stats
        assert st.llr_evaluated[1] < st.distinct_cells[1] and st.llr_evaluated[1] < evaluated_without, \
            (st.llr_evaluated[1], st.distinct_cells[1], evaluated_without)


@pytest.mark.parametrize("k11_max,ok", [(1023, True), (1024, False)])
def test_count_width_limit(orc, ctx, k11_max, ok):
    # 3M columns leave 10 count bits: a co-occurrence count of 2^10 - 1 fills the count field, 2^10 cannot be stored
    n = k11_max + 5
    mats = [csr([[0]] * k11_max, 1, n), csr([[0, 5]] * k11_max + [[5]], 3_000_000, n)]
    params = [(M_ALL, 50, None)] * 2
    if ok:
        exp, _, got = run(orc, ctx, mats, params, tag="count width")
        assert got[1][6].tolist() == [k11_max, k11_max]
    else:
        with pytest.raises(ur.CcoError) as e:
            ctx.train_csr(mats, params, seed=1)
        assert e.value.status == -6


# ---- the fp64 edge (DESIGN.md 3.1): the cut and the dominance filter against the computed values -----------------------
def test_key_cut_tie_under_fp64(orc, ctx):
    # N = 2e7, one item bought by user 0; columns X (id 1, colB 9 271 424) and Y (id 0, colB 9 271 425) each co-occur
    # once with it.  Their computed LLRs are equal, so (llr desc, col asc) keeps Y; a cut by key would keep X.
    n, cx = 20_000_000, 9_271_424
    rp = np.zeros(n + 1, dtype=np.int64)
    rp[1:cx + 1] = np.arange(2, 2 * cx + 1, 2)
    rp[cx + 1:] = 2 * cx + 1
    ci = np.empty(2 * cx + 1, dtype=np.int32)
    ci[0:2 * cx:2], ci[1:2 * cx:2], ci[-1] = 0, 1, 0
    a = (n, 1, np.concatenate([[0], np.ones(n, dtype=np.int64)]), np.zeros(1, dtype=np.int32))
    mats = [a, (n, 2, rp, ci)]
    params = [(M_ALL, 1, None)] * 2
    # the case only tests something if the device evaluates the two LLRs to the same value
    v = ctx.debug_llr([1, 1], [0, 0], [cx - 1, cx], [n - cx, n - cx - 1])
    assert v[0] == v[1], f"no fp64 tie on this device: {v[0]!r} (colB {cx}) vs {v[1]!r} (colB {cx + 1})"
    exp, paths, got = run(orc, ctx, mats, params, tag="fp64 key-cut tie")
    p = paths[1][0]
    assert p.keyed and p.group == 32 and not p.cut        # without the fp64 test the cut would run on this row
    assert got[1][4].tolist() == [0]


def test_dominance_filter_under_fp64(orc, ctx):
    # N = 1e6, rowA = 20, k11 = 3: P (colB 149 995) computes to 3.7e-9 and Q (colB 149 996) to 7.5e-9.  With minLLR
    # 5e-9, P fails and Q passes; P is the 32nd cell in table order, so it is evaluated before Q is filtered.
    n, ra = 1_000_000, 20
    strong = list(range(31))                  # 31 strongly associated columns first in key order (colB 3..33)
    P, Q = 31, 32
    b_rows = [[] for _ in range(n)]
    for u in range(3):
        b_rows[u] = strong + [P, Q]
    f = ra
    for j in strong:
        for k in range(j):
            b_rows[f + k].append(j)
    for j, cb in ((P, 149_995), (Q, 149_996)):
        for k in range(cb - 3):
            b_rows[f + k].append(j)
    b_rows = [sorted(r) for r in b_rows]
    a_rows = [[0] if u < ra else [] for u in range(n)]
    mats = [csr(a_rows, 1, n), csr(b_rows, 33, n)]
    params = [(M_ALL, 50, 5e-9)] * 2
    # the case only tests something if the device evaluates P below minLLR and Q at or above it
    v = ctx.debug_llr([3, 3], [ra - 3, ra - 3], [149_992, 149_993], [n - ra - 149_992, n - ra - 149_993])
    assert v[0] < 5e-9 <= v[1], f"no fp64 crossing on this device: P {v[0]!r}, Q {v[1]!r}"
    exp, paths, got = run(orc, ctx, mats, params, tag="fp64 dominance")
    p = paths[1][0]
    assert not p.keyed and p.dense and p.group == 32
    assert Q in got[1][4].tolist() and P not in got[1][4].tolist()


def test_zz_path_coverage(request):
    """Every owner in dense and hashed form, keyed and colB rows, the three key-cut depths, no-cut and multi-pass rows.
    Checked when every other test of this module has run before it in this session (a full module run, in order)."""
    others = {it.nodeid for it in request.node.parent.collect() if it.nodeid != request.node.nodeid}
    if not others <= RAN:
        pytest.skip(f"coverage is checked on a full run of the module: {len(others - RAN)} of its tests have not run")
    cells = sorted(COVERED, key=str)
    capman = request.config.pluginmanager.get_plugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print("\nrow-kernel paths covered (owner threads, table, score path, cut, passes):")
        for c in cells:
            print("  %s" % (c,))
    for g in (1024, 512, 256, 128, 32):
        for t in ("dense", "hash"):
            assert any(c[0] == g and c[1] == t for c in cells), (g, t)
    assert any(c[2] == "keyed" for c in cells) and any(c[2] == "colB" for c in cells)
    for cut in ("key1", "key2", "key3", "colB", "nocut"):
        assert any(c[3] == cut for c in cells), cut
    assert any(c[4] == "multi" for c in cells)
