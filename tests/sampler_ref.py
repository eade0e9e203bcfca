"""The train's preparation stage restated in plain numpy, from the text of include/cco_b200.h "Sampler".

This is an independent reading of the contract, next to the C oracle (`orc.canonicalize`, `orc.downsample`): the CPU
tests pin the oracle against it, the GPU tests pin the device against both.
  canonical   every row's columns ascending and distinct (`np.unique` per row)
  raw counts  d_u = row length, c_j = `np.bincount` of the canonical columns
  rates       min(m, d_u) / d_u and min(m, c_j) / c_j, IEEE fp64 division; the row rate with `//` under ROWRATE_INTDIV
  hash        h = mix64(mix64((uint32 seed) << 32 | (uint32) u) + (uint32) j * 0x9e3779b97f4a7c15), uint64 arithmetic
  keep        (h >> 11) * 2^-53 <= min(row rate, column rate), in fp64 -- the literal predicate (the device compares the
              53-bit integer with floor(rate * 2^53) instead, so agreeing with this also checks that the two are one)
  A'^T        the sampled matrix transposed (item -> users in ascending order)
  P           sum over users of deg_A'(u) * deg_B'(u): the products of A'^T B'
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

FLAG_ROWRATE_INTDIV = 1
_M1 = np.uint64(0xbf58476d1ce4e5b9)
_M2 = np.uint64(0x94d049bb133111eb)
_GOLDEN = np.uint64(0x9e3779b97f4a7c15)


@dataclass
class Sampled:
    row_ptr: np.ndarray     # int64 [n_rows + 1]
    col_idx: np.ndarray     # int32, the kept entries in row order
    raw: np.ndarray         # int32 [n_cols], raw column counts c_j
    new: np.ndarray         # int32 [n_cols], post-sample column counts
    keep: np.ndarray        # bool per entry of the canonical input
    kept: np.ndarray        # int64 [n_rows], kept entries per user


def mix64(z) -> np.ndarray:
    z = np.asarray(z, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        z ^= z >> np.uint64(30)
        z *= _M1
        z ^= z >> np.uint64(27)
        z *= _M2
        z ^= z >> np.uint64(31)
    return z


def hash64(seed: int, u, j) -> np.ndarray:
    """h of user(s) u and item(s) j (numpy broadcasting)."""
    s = np.uint64(int(seed) & 0xffffffff)
    u = np.asarray(u, dtype=np.int64).astype(np.uint64) & np.uint64(0xffffffff)
    j = np.asarray(j, dtype=np.int64).astype(np.uint64) & np.uint64(0xffffffff)
    with np.errstate(over="ignore"):
        return mix64(mix64((s << np.uint64(32)) | u) + j * _GOLDEN)


def u01(h) -> np.ndarray:
    return (np.asarray(h, dtype=np.uint64) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def canonicalize(n_rows: int, row_ptr, col_idx):
    """-> (row_ptr, col_idx) with every row's columns ascending and distinct."""
    rp = np.asarray(row_ptr, dtype=np.int64)
    ci = np.asarray(col_idx, dtype=np.int64)
    rows = [np.unique(ci[rp[r]:rp[r + 1]]) for r in range(n_rows)]
    out = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum([len(x) for x in rows], out=out[1:])
    col = np.concatenate(rows).astype(np.int32) if rows else np.zeros(0, np.int32)
    return out, col


def row_rates(d, m: int, flags: int = 0) -> np.ndarray:
    d = np.asarray(d, dtype=np.int64)
    md = np.minimum(d, m)
    safe = np.maximum(d, 1)
    if flags & FLAG_ROWRATE_INTDIV:
        return (md // safe).astype(np.float64)
    return md.astype(np.float64) / safe.astype(np.float64)


def col_rates(c, m: int) -> np.ndarray:
    c = np.asarray(c, dtype=np.int64)
    return np.minimum(c, m).astype(np.float64) / np.maximum(c, 1).astype(np.float64)


def downsample(n_rows: int, n_cols: int, row_ptr, col_idx, m: int, seed: int, flags: int = 0,
               raw_counts=None, user_base: int = 0) -> Sampled:
    """sampleDownAndBinarize of a canonical matrix.  raw_counts: the column counts to sample by (default: this matrix's
    own; a block of users is sampled with the whole matrix's); user_base: the global id of row 0 (of such a block)."""
    rp = np.asarray(row_ptr, dtype=np.int64)
    ci = np.asarray(col_idx, dtype=np.int32)
    d = np.diff(rp)
    user = np.repeat(np.arange(n_rows, dtype=np.int64), d)
    raw = np.bincount(ci, minlength=n_cols).astype(np.int32) if raw_counts is None else np.asarray(raw_counts, np.int32)
    rate = np.minimum(row_rates(d, m, flags)[user], col_rates(raw, m)[ci])
    keep = u01(hash64(seed, user_base + user, ci)) <= rate
    kept = np.bincount(user[keep], minlength=n_rows).astype(np.int64)
    out_rp = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(kept, out=out_rp[1:])
    col = ci[keep]
    new = np.bincount(col, minlength=n_cols).astype(np.int32)
    return Sampled(out_rp, col, raw, new, keep, kept)


def downsample_block(n_rows: int, n_cols: int, row_ptr, col_idx, lo: int, hi: int, raw_counts, m: int, seed: int,
                     flags: int = 0) -> Sampled:
    """the users [lo, hi) of a canonical matrix sampled as the rank owning them samples them: global user ids, the
    whole matrix's raw counts.  row_ptr / keep / kept cover the block only."""
    rp = np.asarray(row_ptr, dtype=np.int64)
    q0, q1 = int(rp[lo]), int(rp[hi])
    return downsample(hi - lo, n_cols, rp[lo:hi + 1] - q0, np.asarray(col_idx, np.int32)[q0:q1], m, seed, flags,
                      raw_counts=raw_counts, user_base=lo)


def prepare(n_rows: int, n_cols: int, row_ptr, col_idx, m: int, seed: int, flags: int = 0) -> Sampled:
    """canonicalise, then sample: the train's preparation of one matrix"""
    rp, ci = canonicalize(n_rows, row_ptr, col_idx)
    return downsample(n_rows, n_cols, rp, ci, m, seed, flags)


def transpose(n_rows: int, n_cols: int, row_ptr, col_idx):
    """A^T of a canonical matrix -> (item_ptr int64 [n_cols + 1], users int64, ascending inside each item)"""
    rp = np.asarray(row_ptr, dtype=np.int64)
    ci = np.asarray(col_idx, dtype=np.int64)
    user = np.repeat(np.arange(n_rows, dtype=np.int64), np.diff(rp))
    order = np.lexsort((user, ci))
    ptr = np.zeros(n_cols + 1, dtype=np.int64)
    np.cumsum(np.bincount(ci, minlength=n_cols), out=ptr[1:])
    return ptr, user[order]


def products(a_row_ptr, b_row_ptr) -> int:
    """P = sum over users of deg_A'(u) * deg_B'(u)"""
    return int(np.dot(np.diff(np.asarray(a_row_ptr, np.int64)), np.diff(np.asarray(b_row_ptr, np.int64))))


def products_by_transpose(n_rows: int, n_cols_a: int, a_row_ptr, a_col_idx, b_row_ptr) -> int:
    """P the way the row kernel accumulates it: over the users of every column of A'^T"""
    _, users = transpose(n_rows, n_cols_a, a_row_ptr, a_col_idx)
    return int(np.diff(np.asarray(b_row_ptr, np.int64))[users].sum())


def csr_sampler(csr_type):
    """The preparation as rowref.sampled(sampler=...) takes it: (raw matrix of csr_type, m, seed, flags) ->
    (canonical sampled matrix of csr_type, raw column counts, post-sample column counts)"""
    def sample(c, m: int, seed: int, flags: int = 0):
        s = prepare(int(c.n_rows), int(c.n_cols), c.row_ptr, c.col_idx, m, seed, flags)
        return csr_type(c.n_rows, c.n_cols, s.row_ptr, s.col_idx), s.raw, s.new
    return sample
