"""The key-range plan (tests/key_ranges_ref.py, restating the host plan of enqueue_indicator) without a GPU: the ranges
tile the key space, each fits the packed word, greedy is minimal against brute force, and the two-range arithmetic of
DESIGN.md 3.1 "key ranges" holds on its worked shapes."""
import functools

import numpy as np
import pytest

import key_ranges_ref as kr


def check_tiling(p, n, mk, max_a, cap=0):
    assert p[0][0] == 0 and p[-1][1] == n
    for (a0, a1), (b0, _) in zip(p, p[1:]):
        assert a1 == b0
    for k0, k1 in p:
        assert k1 > k0
        assert kr.fits(k1 - k0, min(max_a, int(mk[k1 - 1])))
        if cap:
            assert k1 - k0 <= cap


def brute_min_ranges(mk, max_a, cap=0):
    n = len(mk)

    @functools.lru_cache(maxsize=None)
    def best(k0):
        if k0 == n:
            return 0
        r = None
        for k1 in range(k0 + 1, n + 1):
            if cap and k1 - k0 > cap:
                break
            if kr.fits(k1 - k0, min(max_a, int(mk[k1 - 1]))):
                b = best(k1)
                if b is not None and (r is None or b + 1 < r):
                    r = b + 1
        return r
    return best(0)


def test_packed_word_rule_matches_the_documented_bounds():
    # past 4 194 302 columns: 23 key bits, 9 count bits (counts < 512); 4 194 302 columns keep 22 key bits
    assert kr.fits(4_194_303, 511) and not kr.fits(4_194_303, 512)
    assert kr.fits(4_194_302, 1023) and not kr.fits(4_194_302, 1024)
    # 1M columns: 20 key bits, counts < 4096
    assert kr.fits(1_000_000, 4095) and not kr.fits(1_000_000, 4096)
    assert kr.fits(2 ** 31 - 2, 1) and not kr.fits(2 ** 31 - 2, 2)      # the largest item space: one count bit


@pytest.mark.parametrize("seed", range(40))
def test_greedy_plan_tiles_fits_and_is_minimal(seed):
    # word widths scaled down: a small item space only splits when counts are large, so draw counts near 2^(32 - kb)
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 40))
    top = int(rng.integers(1, 31))
    mk = np.sort(rng.integers(0, 2 ** top, n))
    if seed % 3 == 0:
        mk[-1] = int(rng.integers(2 ** 26, 2 ** 30))     # a column whose counts fit only a very short range, or none
    max_a = int(rng.integers(1, 2 ** 30))
    cap = int(rng.integers(0, 6))
    try:
        p = kr.plan(mk, max_a, cap)
    except ValueError:
        assert brute_min_ranges(mk, max_a, cap) is None
        return
    check_tiling(p, n, mk, max_a, cap)
    assert len(p) == brute_min_ranges(mk, max_a, cap)


@pytest.mark.parametrize("cap", [1, 2, 31, 32, 33])
def test_cap_alone_cuts_ceil_n_over_cap_where_the_word_fits(cap):
    mk = np.sort(np.random.default_rng(cap).integers(0, 560, 1000))
    p = kr.plan(mk, 560, cap)
    check_tiling(p, 1000, mk, 560, cap)
    assert len(p) == -(-1000 // cap)
    assert kr.n_ranges(mk, 560, 0) == 1


@pytest.mark.parametrize("n_cols", [4_194_303, 8_500_000, 12_000_000, 16_777_214])
def test_two_ranges_below_2_24_columns_at_m_500(n_cols):
    # m = 500: marginals scatter up to ~560.  Any item space below 2^24 - 1 columns needs at most two ranges while
    # nnz(B') < 2^30: keys with colB < 256 (24 key bits, 8 count bits), then at most nnz / 256 keys with colB >= 256
    nnz = 2 ** 30 - 1
    n_hot = nnz // 560                      # the most columns that can reach colB 560
    mk = np.zeros(n_cols, dtype=np.int64)
    mk[-n_hot:] = 560
    mk[-n_hot - 1000:-n_hot] = 255
    p = kr.plan(mk, 560)
    check_tiling(p, n_cols, mk, 560)
    assert len(p) == 2
    assert kr.n_ranges(mk, 560) == 2


def test_limit_test_shape_needs_two_ranges():
    # the packed-word limit test's matrices: 3M columns, three columns co-occurring 3000 times, m = 10^6
    mk = np.sort(np.concatenate([np.full(3_000_000 - 3, 12), [3000, 3001, 3002]]))
    assert not kr.fits(3_000_000, 3000)
    assert kr.n_ranges(mk, 3050) == 2
    assert kr.plan(mk, 3050) == [(0, 2_999_997), (2_999_997, 3_000_000)]


def test_a_single_key_that_does_not_fit_is_refused():
    with pytest.raises(ValueError):
        kr.plan(np.array([1, 2 ** 30]), 2 ** 30)
