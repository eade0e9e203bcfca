"""CPU checks of the fp64 LLR error bound eps(N) = 2^-47 N ln N (cco_api.cu llr_error_bound, DESIGN.md 3.1).

The extended-precision reference of tests/llr_exact.py against 50-digit decimal, then the oracle's LLR (glibc log, both
entropy orders) against that reference on the edge grid: within eps, never negative, and 0 only where the real value is
below eps.  The same grid runs on the device in tests/test_gpu_llr_exact.py."""
from fractions import Fraction

import numpy as np
import pytest

import llr_exact as lx

@pytest.mark.parametrize("n", lx.GRID_N)
def test_longdouble_reference_against_decimal(n):
    rng = np.random.default_rng(1000 + n)
    cells = lx.edge_cells(n, rng, 220)
    ld = lx.llr_longdouble(*cells)
    bound = Fraction(lx.eps(n)) / 1000
    worst = Fraction(0)
    for i, t in enumerate(zip(*cells)):
        real = Fraction(lx.llr_decimal(*map(int, t)))
        err = abs(Fraction(*ld[i].as_integer_ratio()) - real)
        assert err < bound, f"N={n} cell {t}: long double {ld[i]!r} vs {float(real)!r}"
        worst = max(worst, err)
    assert float(worst) < float(bound)


def test_longdouble_refuses_a_short_mantissa(monkeypatch):
    class Short:
        nmant = 52
    monkeypatch.setattr(lx.np, "finfo", lambda t: Short)
    with pytest.raises(RuntimeError, match="64-bit long double mantissa"):
        lx.llr_longdouble([1], [0], [0], [1])


def test_edge_cells_cover_the_limits():
    n = 10 ** 6
    k11, k12, k21, k22 = lx.edge_cells(n, np.random.default_rng(0), 50_000)
    ra, cb = k11 + k12, k11 + k21
    assert ((k11 + k12 + k21 + k22) == n).all() and min(k11.min(), k12.min(), k21.min(), k22.min()) >= 0
    for v in (1, 2, 30, 34, 600, n // 2, n - 1):
        assert (ra == v).any() and (cb == v).any(), v
    assert (k11 == np.maximum(0, ra + cb - n)).any() and (k11 == np.minimum(ra, cb)).any()
    assert (ra * cb > k11 * n).any() and (ra * cb < k11 * n).any()     # both sides of the association
    assert (np.abs(k11 * n - ra * cb) < n).sum() > 10_000               # cells at independence


def test_oracle_llr_within_eps_on_the_grid(orc, request):
    lines = []
    for n in lx.GRID_N:
        cells = lx.grid(n)
        real = lx.llr_longdouble(*cells)
        worst = []
        for flags in (0, lx.ORC_FLAG_ENTROPY_VARARGS):
            worst.append(lx.check_against_real(lx.oracle_llr(orc, cells, flags), real, n, f"oracle N={n} flags={flags}"))
        lines.append(f"N = {n:>10}: left-to-right {worst[0]:.4f} eps, varargs {worst[1]:.4f} eps")
    lx.report(request, "oracle (glibc log): largest |computed - real| / eps per N", lines)
