"""Brute-force expected indicators that share the kernel's LLR arithmetic.

For the matrices, params, seed and flags of a train, `expected()` returns what the device must write, bit for bit:
  cells      every non-zero cell of A'^T B' from the oracle's sampler (`orc.downsample`, bit-exact with the device) and
             its integer product (`orc.cooccurrence`);
  LLR        of every cell from the device's own `llr_cells` (`ctx.debug_llr`), with rowA, colB and N of the sampled
             matrices;
  selection  v > 0, v >= minLLR (inclusive), the diagonal skipped for A'^T A', sorted by (llr desc, col asc), the first
             top_k of each row.
So the comparison does not depend on whether the device `log` and glibc's agree in the last ulp: it checks the row
kernel's count, compaction, cut, dominance filter and select exactly, ties included, and that the kernel's hoisted LLR
(x12tab, ColTerm, row_e) equals `llr_cells` bit for bit at every kept cell.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import row_paths
import universal_recommender_b200 as ur
from oracle import oracle as orc


@dataclass
class Expected:
    row_ptr: np.ndarray
    col: np.ndarray
    llr: np.ndarray
    count: np.ndarray
    # the shape the row kernel schedules by (row_paths.row_path)
    work: np.ndarray        # w_a = sum over the users of a of deg_B'(u)
    ra: np.ndarray          # colA of A'
    n_cols_b: int
    max_marg_a: int
    max_marg_b: int
    n_users: int
    top_k: int
    distinct: int           # non-zero cells of A'^T B' (diagonal included)

    def paths(self):
        """RowPath (or None: no work) of every output row."""
        return [row_paths.row_path(int(w), int(r), self.n_cols_b, self.max_marg_a, self.max_marg_b, self.n_users,
                                   self.top_k) for w, r in zip(self.work, self.ra)]


def oracle_sampler(c, m: int, seed: int, flags: int = 0):
    """The default preparation: orc_train's canonicalisation and sampler -> (sampled orc.Csr, raw counts, marginals)"""
    return orc.downsample(orc.canonicalize(c), m, seed, flags)


def sampled(mats, params, seed: int, flags: int = 0, sampler=None):
    """[(A' or B'_i as orc.Csr, its column marginals)] exactly as the train samples them (orc_train).  sampler: another
    preparation of the same shape as `oracle_sampler` (e.g. sampler_ref.csr_sampler(orc.Csr))."""
    sampler = sampler or oracle_sampler
    out = []
    for (nr, nc, rp, ci), p in zip(mats, params):
        d, _, marg = sampler(orc.Csr(nr, nc, rp, ci), int(p[0]), seed, flags & 3)
        out.append((d, marg.astype(np.int64)))
    return out


def expected(ctx, mats, params, seed: int, flags: int = 0, sampler=None) -> list[Expected]:
    sm = sampled(mats, params, seed, flags, sampler)
    a, marg_a = sm[0]
    n = int(a.n_rows)
    n_items = int(a.n_cols)
    a_rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(a.row_ptr))
    out = []
    for i, (p, (b, marg_b)) in enumerate(zip(params, sm)):
        top_k, min_llr = int(p[1]), p[2]
        rp, ci, cn = orc.cooccurrence(a, b)
        row = np.repeat(np.arange(n_items, dtype=np.int64), np.diff(rp))
        k11 = cn.astype(np.int64)
        ra, cb = marg_a[row], marg_b[ci]
        if len(k11):
            v = ctx.debug_llr(k11, ra - k11, cb - k11, n - ra - cb + k11, flags & ur.FLAG_ENTROPY_VARARGS)
        else:
            v = np.zeros(0, dtype=np.float64)
        keep = v > 0.0
        if min_llr is not None:
            keep &= v >= min_llr
        if i == 0:
            keep &= ci != row
        row, col, v, k11 = row[keep], ci[keep].astype(np.int64), v[keep], k11[keep]
        order = np.lexsort((col, -v, row))
        row, col, v, k11 = row[order], col[order], v[order], k11[order]
        rank = np.arange(len(row)) - np.searchsorted(row, row, side="left")
        sel = rank < top_k
        row, col, v, k11 = row[sel], col[sel], v[sel], k11[sel]
        row_ptr = np.zeros(n_items + 1, dtype=np.int64)
        np.cumsum(np.bincount(row, minlength=n_items), out=row_ptr[1:])
        deg_b = np.diff(b.row_ptr)
        work = np.bincount(a.col_idx, weights=deg_b[a_rows], minlength=n_items).astype(np.int64) if n_items else \
            np.zeros(0, np.int64)
        out.append(Expected(row_ptr, col.astype(np.int32), v, k11.astype(np.int32), work, marg_a[:n_items],
                            int(b.n_cols), int(marg_a.max(initial=0)), int(marg_b.max(initial=0)), n, top_k, len(ci)))
    return out


def assert_matches(exp: list[Expected], got, tag: str = ""):
    """The device result (ctx.train_csr) against the reference, bit for bit, LLR bit patterns included."""
    assert len(exp) == len(got), tag
    for i, (e, g) in enumerate(zip(exp, got)):
        _, _, _, rp, ci, ll, cn = g
        lens_e, lens_g = np.diff(e.row_ptr), np.diff(rp)
        bad = np.nonzero(lens_e != lens_g)[0]
        assert not len(bad), f"{tag} indicator {i}: row lengths differ at rows {bad[:8]} ({lens_e[bad[:8]]} vs {lens_g[bad[:8]]})"
        for name, x, y in (("columns", e.col, ci), ("counts", e.count, cn),
                           ("LLR bits", e.llr.view(np.uint64), np.asarray(ll, dtype=np.float64).view(np.uint64))):
            diff = np.nonzero(x != y)[0]
            if len(diff):
                r = int(np.searchsorted(e.row_ptr, diff[0], side="right") - 1)
                s, t = int(e.row_ptr[r]), int(e.row_ptr[r + 1])
                raise AssertionError(f"{tag} indicator {i}: {name} differ first in row {r}: expected cols {e.col[s:t][:8]} "
                                     f"llr {e.llr[s:t][:8]}, got cols {ci[s:t][:8]} llr {ll[s:t][:8]}")
