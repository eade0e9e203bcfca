"""CPU tests of the row-path model (tests/row_paths.py) and of the fp64 edge of the level-1 cut and the dominance filter.

The cut and the filter rely on the LLR being monotone in colB and k11.  The real-valued LLR is; its fp64 evaluation is
not, once adjacent colB values are closer than the evaluation error.  These tests pin instances of that (with the
oracle's own evaluation order and glibc log), show with 50-digit arithmetic that the real values are monotone there,
and check that the host's exactness test (cco_api.cu cut_exact) rejects those shapes and accepts C3 and C4."""
from decimal import Decimal

import numpy as np
import pytest

import row_paths as rp
from llr_exact import cut_c_max, llr_exact


# ---- the path model ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top_k", [1, 50, 64, 65, 128, 129, 224, 225, 1000])
@pytest.mark.parametrize("n_cols_b", [1, 300, 512, 4096, 70_000, 3_000_000])
def test_bins_partition_the_work_axis(top_k, n_cols_b):
    cfgs, h_thr = rp.bins(top_k, n_cols_b)
    assert h_thr[-1] == 0 and all(x >= y for x, y in zip(h_thr, h_thr[1:]))
    groups = [c.group for c in cfgs]
    assert all(x >= y for x, y in zip(groups, groups[1:]))       # larger rows never get fewer threads
    for c in cfgs:
        assert c.cbuf >= top_k + c.group and c.cbuf & (c.cbuf - 1) == 0
        assert c.final_max >= top_k and c.keep_max >= c.final_max
        assert c.dense == (n_cols_b <= c.slots) and c.slots > 0
    # every w > 0 lands in one bin, a hashed bin never takes a row above its capacity unless it is the multi-pass bin
    for w in sorted({1, 2, 255, 256, 257, 4097, 8193, 22_528, 22_529, 45_057, 65_535, 65_536, 2 ** 32 - 1} | set(h_thr)):
        if w <= 0:
            continue
        b = rp.bin_of(w, h_thr)
        assert b is not None and (b == 0 or w <= h_thr[b - 1])
        if b > 0 and not cfgs[b].dense:
            assert w <= cfgs[b].cap
    assert rp.bin_of(0, h_thr) is None


def test_h100_bin_boundaries_at_top_k_50():
    # the boundaries the directed GPU cases sit on (H100: 232 448 B of opt-in shared memory per block)
    cfgs, h_thr = rp.bins(50, 70_000)
    cap = cfgs[1].cap
    assert cap == 22_528 and [c.group for c in cfgs] == [1024, 1024, 512, 256, 128, 32, 32, 32]
    assert h_thr == [cap, 8192, 4096, 2048, 1024, 512, 256, 0]
    assert not any(c.dense for c in cfgs)
    cfgs, h_thr = rp.bins(50, 300)
    assert all(c.dense for c in cfgs) and h_thr == [2 ** 32 - 1, 8192, 4096, 2048, 1024, 512, 256, 0]
    assert rp.row_path(50_000, 5, 70_000, 5, 5, 10 ** 6, 50).n_pass == 3
    assert rp.row_path(cap + 1, 5, 70_000, 5, 5, 10 ** 6, 50).n_pass == 2
    assert rp.row_path(cap, 5, 70_000, 5, 5, 10 ** 6, 50).bin == 1


def test_warp_owned_rows_end_at_top_k_224():
    assert rp.warp_ok(224) and not rp.warp_ok(225)
    assert rp.row_path(100, 1, 300, 1, 1, 1000, 224).group == 32
    assert rp.row_path(100, 1, 300, 1, 1, 1000, 225).group == 128


def test_key_cut_depth():
    assert [rp.key_levels(n) for n in (1, 512, 513, 2 ** 18, 2 ** 18 + 1, 2 ** 27)] == [1, 1, 2, 2, 3, 3]
    assert rp.key_levels(100_000) == 2 and rp.key_levels(1_000_000) == 3


def test_count_bits_limit():
    assert rp.count_bits(3_000_000) == 10 and rp.count_bits(70_000) == 15
    assert rp.counts_fit(3_000_000, 1023, 5000) and not rp.counts_fit(3_000_000, 1024, 5000)


@pytest.mark.parametrize("n_users,n_cols,top_k", [(1_000_000, 100_000, 50), (10_000_000, 1_000_000, 50)])
def test_c3_c4_shaped_rows_are_keyed_and_cut(n_users, n_cols, top_k):
    # C3 / C4 with m = 500: every marginal after downsampling is ~560 at most
    for ra in (1, 50, 300, 600):
        for w in (1, 300, 5000, 60_000, 70_000):
            p = rp.row_path(w, ra, n_cols, 600, 600, n_users, top_k)
            assert p.keyed and p.levels == rp.key_levels(n_cols) and not p.dense
            assert p.cut == (w < 65_536)


# ---- the fp64 edge ------------------------------------------------------------------------------------------------------
def llr_k1(orc, n, ra, cb, k=1):
    return orc.llr(k, ra - k, cb - k, n - ra - cb + k)


def test_key_cut_tie_instance(orc):
    # N = 2e7, rowA = 1, k11 = 1: two adjacent colB values give the same fp64 LLR; the real values differ by ~2.2e-7
    n = 20_000_000
    a, b = llr_k1(orc, n, 1, 9_271_424), llr_k1(orc, n, 1, 9_271_425)
    assert a == b == 1.5375904440879822
    assert llr_exact(n, 1, 9_271_424) - llr_exact(n, 1, 9_271_425) > Decimal("2e-7")
    assert not rp.cut_exact(n, 1, 9_271_425)           # the kernel runs such rows without the cut


def test_dominance_filter_instance(orc):
    # N = 1e6, rowA = 20, k11 = 3, near independence: the fp64 LLR INCREASES from colB 149 995 to 149 996
    n = 1_000_000
    a, b = llr_k1(orc, n, 20, 149_995, 3), llr_k1(orc, n, 20, 149_996, 3)
    assert 0 < a < 5e-9 <= b and (a, b) == (3.725290298461914e-09, 7.450580596923828e-09)
    assert 20 * 149_996 < 3 * n                          # both on the positive side, where the filter applies
    ea, eb = llr_exact(n, 20, 149_995, 3), llr_exact(n, 20, 149_996, 3)
    assert ea > eb > 0                                   # the real LLR decreases: the defect is rounding alone
    # the filter's margin: a cell records a frontier only if v + 2 eps < minLLR
    assert a + 2 * rp.llr_error_bound(n) > 5e-9


def first_non_decreasing(orc, n, ra, lo, hi):
    """First colB in [lo, hi) whose computed k11 = 1 LLR is not strictly above the next one's (None if there is none)."""
    prev = llr_k1(orc, n, ra, lo)
    for c in range(lo + 1, hi + 1):
        cur = llr_k1(orc, n, ra, c)
        if not cur < prev:
            return c - 1
        prev = cur
    return None


def test_scan_where_adjacent_colb_stops_decreasing(orc):
    # rowA = 1: strictly decreasing for small colB, ties by colB ~ 4e6 at N = 5e7, increases further up
    n = 50_000_000
    assert first_non_decreasing(orc, n, 1, 1, 20_000) is None
    c = first_non_decreasing(orc, n, 1, 3_990_000, 4_010_000)
    assert c is not None and 3.9e6 < c < 4.1e6
    assert llr_exact(n, 1, c) > llr_exact(n, 1, c + 1)
    seen_increase = False
    for lo in (15_000_000, 20_000_000):
        vals = [llr_k1(orc, n, 1, x) for x in range(lo, lo + 4000)]
        seen_increase |= any(y > x for x, y in zip(vals, vals[1:]))
    assert seen_increase
    # rowA = 50, N = 1e8: increases too, inside the strongly positive side (2 rowA colB < N)
    n, ra = 100_000_000, 50
    vals = [llr_k1(orc, n, ra, x) for x in range(990_000, 994_000)]
    assert 2 * ra * 994_000 < n and any(y > x for x, y in zip(vals, vals[1:]))


@pytest.mark.parametrize("n", [10 ** 5, 10 ** 6, 10 ** 7, 5 * 10 ** 7, 2 * 10 ** 8])
@pytest.mark.parametrize("ra", [1, 7, 60, 600])
def test_cut_exact_bound_holds_where_it_admits_the_cut(orc, n, ra):
    # the largest max colB that cut_exact admits for this rowA (on the strongly positive side): computed values
    # strictly decrease right up to it
    eps = rp.llr_error_bound(n)
    c_max = cut_c_max(n, ra)
    assert first_non_decreasing(orc, n, ra, max(1, c_max - 3000), c_max) is None
    # and the real gap there is above the bound's 2 eps
    assert float(llr_exact(n, ra, c_max - 1) - llr_exact(n, ra, c_max)) > 2 * eps


def test_cut_exact_at_benchmark_shapes():
    assert rp.cut_exact(1_000_000, 600, 600) and rp.cut_exact(10_000_000, 600, 600)
    assert not rp.cut_exact(20_000_000, 1, 9_271_425) and not rp.cut_exact(50_000_000, 1, 4_000_000)


@pytest.mark.parametrize("n", [5 * 10 ** 7, 10 ** 8, 2 ** 31 - 1])
def test_default_downsampling_keeps_the_cut_at_large_n(orc, n):
    # m = 500 keeps every marginal near 560: the cut stays on for every supported N, and the computed k11 = 1 LLRs of
    # every rowA up to 600 do decrease strictly over colB 1..600 there
    assert rp.cut_exact(n, 600, 600)
    for ra in (1, 2, 50, 600):
        assert first_non_decreasing(orc, n, ra, 1, 600) is None
    # the bound turns the cut off only when max colB nears 1 / eps
    assert not rp.cut_exact(n, 600, int(1.05 / rp.llr_error_bound(n)))
