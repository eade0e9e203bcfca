"""Exact references for one LLR (Mahout LogLikelihood.logLikelihoodRatio) and the cells its error bound is tested on.

The row kernel's cut and dominance filter rest on eps(N) (cco_api.cu llr_error_bound) bounding |computed - real| of one
fp64 LLR.  These helpers give the real value two ways:
  llr_decimal     50 significant digits in `decimal`, one cell at a time (the yardstick);
  llr_longdouble  the same formula over int64 arrays in x86-64 extended precision (64-bit mantissa): the bulk reference
                  for millions of cells, held within eps / 1000 of llr_decimal up to N = 2^31 - 1
                  (tests/test_llr_exact.py).
"""
from __future__ import annotations

from decimal import Decimal, localcontext

import numpy as np

import row_paths
from row_paths import llr_error_bound as eps   # the one Python copy of the bound

GRID_N = [2, 3, 10, 10 ** 3, 10 ** 6, 10 ** 7, 2 * 10 ** 7, 10 ** 8, 2 ** 31 - 1]
GRID_CELLS = 120_000        # edge_cells per N of the full grid
ORC_FLAG_ENTROPY_VARARGS = 2      # oracle/cco_oracle.h


def llr_decimal(k11: int, k12: int, k21: int, k22: int, prec: int = 50) -> Decimal:
    """The real LLR, 2 (rowEntropy + columnEntropy - matrixEntropy), with xLogX in `prec`-digit decimal."""
    with localcontext() as c:
        c.prec = prec
        xl = lambda x: Decimal(0) if x == 0 else Decimal(x) * Decimal(x).ln()
        n = k11 + k12 + k21 + k22
        row = xl(n) - xl(k11 + k12) - xl(k21 + k22)
        col = xl(n) - xl(k11 + k21) - xl(k12 + k22)
        mat = xl(n) - xl(k11) - xl(k12) - xl(k21) - xl(k22)
        return 2 * (row + col - mat)


def llr_exact(n: int, ra: int, cb: int, k: int = 1) -> Decimal:
    """The real LLR of a cell given by (N, rowA, colB, k11), 50 significant digits."""
    return llr_decimal(k, ra - k, cb - k, n - ra - cb + k)


def cut_c_max(n: int, ra: int) -> int:
    """The largest max colB that row_paths.cut_exact admits for max rowA = ra, capped at the strongly positive side
    (2 ra colB < N), the only side where the kernel cuts"""
    lo, hi = 1, (n - 1) // (2 * ra) - 1
    assert row_paths.cut_exact(n, ra, lo)
    if row_paths.cut_exact(n, ra, hi):
        lo = hi
    while hi - lo > 1:                                   # cut_exact is monotone in max colB
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if row_paths.cut_exact(n, ra, mid) else (lo, mid)
    return lo


def _check_longdouble():
    if np.finfo(np.longdouble).nmant < 63:
        raise RuntimeError(f"llr_longdouble needs a 64-bit long double mantissa (x86-64 extended precision); this "
                           f"platform's np.longdouble has {np.finfo(np.longdouble).nmant + 1} bits")


def _xlogx(x: np.ndarray) -> np.ndarray:
    x = x.astype(np.longdouble)
    return np.where(x > 0, x * np.log(np.where(x > 0, x, 1)), np.longdouble(0))


def llr_longdouble(k11, k12, k21, k22) -> np.ndarray:
    """The real LLR of every cell of int64 arrays, as np.longdouble (unclamped: rounding can leave tiny negatives)."""
    _check_longdouble()
    k11, k12, k21, k22 = (np.asarray(x, dtype=np.int64) for x in (k11, k12, k21, k22))
    n = k11 + k12 + k21 + k22
    xn = _xlogx(n)
    row = xn - _xlogx(k11 + k12) - _xlogx(k21 + k22)
    col = xn - _xlogx(k11 + k21) - _xlogx(k12 + k22)
    mat = xn - _xlogx(k11) - _xlogx(k12) - _xlogx(k21) - _xlogx(k22)
    return 2 * (row + col - mat)


def edge_cells(n: int, rng: np.random.Generator, count: int):
    """`count` cells (k11, k12, k21, k22) of int64 with k11 + k12 + k21 + k22 = n, all >= 0.

    rowA and colB each from {1, 2, 30..34, 600, random <= 600, ~N/2, N - 1, random} (clipped to 1..N - 1); k11 at its
    lower limit max(0, rowA + colB - N), its upper limit min(rowA, colB), at independence round(rowA colB / N) + d for
    d in -3..3 (the cancellation-limited cells, on both sides of the association), or random in between."""
    top = max(n - 1, 1)

    def marginal():
        pick = rng.integers(0, 10, count)
        choices = [np.ones(count, np.int64), np.full(count, 2, np.int64), rng.integers(30, 35, count),
                   np.full(count, 600, np.int64), rng.integers(1, 601, count), n // 2 + rng.integers(-2, 3, count),
                   np.full(count, n - 1, np.int64), rng.integers(1, top + 1, count),
                   rng.integers(1, 601, count), rng.integers(1, top + 1, count)]
        m = np.choose(pick, choices).astype(np.int64)
        return np.clip(m, 1, top)

    ra, cb = marginal(), marginal()
    lo = np.maximum(0, ra + cb - n)
    hi = np.minimum(ra, cb)
    indep = (2 * ra * cb + n) // (2 * n) + rng.integers(-3, 4, count)     # round(ra cb / N) + d
    rand = lo + (rng.random(count) * (hi - lo + 1)).astype(np.int64)
    pick = rng.integers(0, 6, count)
    k11 = np.choose(pick, [lo, hi, indep, indep, indep, rand])
    k11 = np.clip(k11, lo, hi)
    k12, k21 = ra - k11, cb - k11
    k22 = n - ra - cb + k11
    assert (k22 >= 0).all() and (k12 >= 0).all() and (k21 >= 0).all() and (k11 >= 0).all()
    return k11, k12, k21, k22


def oracle_llr(orc, cells, flags):
    """The oracle's LLR (glibc log) of every cell; flags: 0 or ORC_FLAG_ENTROPY_VARARGS"""
    f = orc.lib().orc_llr
    return np.fromiter((f(a, b, c, d, flags) for a, b, c, d in zip(*(x.tolist() for x in cells))), np.float64,
                       len(cells[0]))


def check_against_real(v, real, n, tag):
    """Computed LLRs v against the real values: |v - real| <= eps(N), v finite and >= 0, v == 0 only where the real value
    is <= eps(N).  -> the largest |v - real| / eps"""
    e = eps(n)
    assert np.isfinite(v).all(), f"{tag}: non-finite LLR"
    neg = np.nonzero(v < 0)[0]
    assert not len(neg), f"{tag}: negative LLR {v[neg[0]]!r} (real {float(real[neg[0]])!r}) at cell {neg[0]}"
    err = np.abs(v.astype(np.longdouble) - real)
    ratio = err / np.longdouble(e)
    bad = np.nonzero(ratio > 1)[0]
    assert not len(bad), f"{tag}: |v - real| = {float(ratio[bad[0]]):.3f} eps at cell {bad[0]}: {v[bad[0]]!r} vs " \
                         f"{float(real[bad[0]])!r}"
    zero = np.nonzero((v == 0) & (real > e))[0]
    assert not len(zero), f"{tag}: LLR 0 where the real value {float(real[zero[0]])!r} exceeds eps {e!r}"
    return float(ratio.max())


def grid(n: int, count: int = GRID_CELLS):
    """The full grid of one N: edge_cells with a seed of its own (the CPU and the device tests check the same cells)."""
    return edge_cells(n, np.random.default_rng(n), count)


def report(request, title: str, lines):
    """Print past pytest's capture (the worst ratios are part of what these tests measure)."""
    capman = request.config.pluginmanager.get_plugin("capturemanager")
    with capman.global_and_fixture_disabled():
        print("\n" + title)
        for line in lines:
            print("  " + line)
