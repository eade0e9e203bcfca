"""Directed matrices for the train's preparation stage (canonicalisation, raw column counts, sampler, A'^T).

k_sample_count (cco_sampler.cuh) walks chunks of 256 stored entries per warp, in batches of 32 entries, with a window of
32 consecutive rows in registers; k_col_histogram_flat aggregates equal column ids of a warp and spreads its atomics over
16 replicated copies by CTA.  The shapes below put row starts, runs of empty rows, window slides, matrix ends, rate
thresholds and column groups on exactly those edges.  Every shape is canonical (columns ascending and distinct per row);
`messy` turns one into the unsorted, duplicated input that canonicalize_device has to repair.

Each shape is (name, (n_rows, n_cols, row_ptr int64, col_idx int32), m): m makes the sampler active on it.
"""
from __future__ import annotations

import numpy as np

CHUNK, BATCH = 256, 32


def csr(rows, n_cols):
    rp = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=rp[1:])
    ci = np.array([c for r in rows for c in r], dtype=np.int32)
    return (len(rows), n_cols, rp, ci)


class _Rows:
    """rows with distinct ascending columns drawn from a skewed (Zipf-like) column law, so that some columns are hot"""

    def __init__(self, n_cols: int, seed: int, skew: float = 0.8):
        self.n_cols = n_cols
        self.rng = np.random.default_rng(seed)
        w = 1.0 / np.power(np.arange(1, n_cols + 1, dtype=np.float64), skew)
        self.p = w / w.sum()
        self.rows: list[list[int]] = []
        self.nnz = 0

    def add(self, length: int):
        assert length <= self.n_cols
        r = sorted(self.rng.choice(self.n_cols, length, replace=False, p=self.p).tolist()) if length else []
        self.rows.append(r)
        self.nnz += length

    def empty(self, n: int):
        for _ in range(n):
            self.add(0)

    def pad_to(self, modulus: int, residue: int):
        """one filler row, so that the next row starts at an entry offset = residue (mod modulus)"""
        need = (residue - self.nnz) % modulus
        if need:
            self.add(need)

    def done(self):
        return csr(self.rows, self.n_cols)


def row_lengths():
    """rows of 0, 1, 31, 32, 33, 255, 256, 257 and 5000 entries starting on, one before and one after a chunk boundary
    and a batch boundary"""
    b = _Rows(6000, 1)
    for length in (0, 1, 31, 32, 33, 255, 256, 257, 5000):
        for modulus in (CHUNK, BATCH):
            for delta in (0, -1, 1):
                b.pad_to(modulus, delta % modulus)
                b.add(length)
                b.add(3)
    return b.done()


def empty_runs():
    """runs of 31, 32, 33, 64 and 1000 empty rows: at the start, inside a chunk, at a chunk boundary, straddling the
    entries of a chunk boundary, and at the end"""
    b = _Rows(300, 2)
    b.empty(33)                                     # at the start: the first chunk's 32-ary search skips them
    for run in (31, 32, 33, 64, 1000):
        b.add(5)
        b.empty(run)                                # inside a chunk
        b.add(7)
        b.pad_to(CHUNK, 0)
        b.empty(run)                                # exactly at a chunk boundary (the rows before end on it)
        b.add(40)
        b.pad_to(CHUNK, CHUNK - 3)
        b.add(6)                                    # this row straddles the boundary ...
        b.empty(run)                                # ... and the run follows inside the next chunk
        b.add(1)
        b.pad_to(BATCH, BATCH - 1)
        b.add(1)
        b.empty(run)                                # between two one-entry rows of one batch
        b.add(1)
    b.add(9)
    b.empty(1000)                                   # at the end
    return b.done()


def short_rows():
    """one-entry rows after a long row: the window (loaded at the long row) slides in the middle of a batch; then
    one-entry rows with an empty row between each, so that a batch spans 64 rows"""
    b = _Rows(500, 3)
    for lead in (40, 300, 1):
        b.add(lead)
        for _ in range(100):
            b.add(1)
        for _ in range(100):
            b.add(1)
            b.empty(1)
    b.pad_to(CHUNK, 7)
    for _ in range(70):
        b.add(1)
    return b.done()


def sized(n_rows: int, nnz: int, n_cols: int = 700, seed: int = 4):
    """n_rows rows holding exactly nnz entries (lengths as even as possible, the remainder on the first rows)"""
    b = _Rows(n_cols, seed)
    q, r = divmod(nnz, n_rows)
    for i in range(n_rows):
        b.add(q + (1 if i < r else 0))
    return b.done()


def thresholds(m: int, n_cols: int = 64):
    """rows of exactly m and m + 1 entries, a column in exactly m rows (col 0) and one in exactly m + 1 rows (col 1);
    the other columns fill the rows round robin"""
    n_rows = 3 * (m + 1)
    rows = []
    for r in range(n_rows):
        d = m if r % 2 == 0 else m + 1
        cols = []
        if r < m:
            cols.append(0)
        if r < m + 1:
            cols.append(1)
        t = 0
        while len(cols) < d:
            c = 2 + (r * 5 + t) % (n_cols - 2)
            t += 1
            if c not in cols:
                cols.append(c)
        rows.append(sorted(cols))
    return csr(rows, n_cols)


def one_column(n_rows: int = 20_000):
    """n_cols = 1: every entry in one column (full warps in one __match_any_sync group), nnz not a multiple of 32,
    enough CTAs to wrap the 16 histogram copies"""
    rows = [[0] if (r % 7 != 3) else [] for r in range(n_rows)]
    return csr(rows, 1)


def last_column(n_rows: int = 9_001, n_cols: int = 50_000):
    """ids at n_cols - 1 in most rows (one hot column, the largest id), a few other columns beside it"""
    rows = []
    for r in range(n_rows):
        row = [n_cols - 1] if r % 5 else []
        if r % 3 == 0:
            row = [r % 97, (r * 31) % 1000 + 100] + row
        rows.append(sorted(set(row)))
    return csr(rows, n_cols)


def shapes():
    """[(name, matrix, m)] -- m puts the sampler to work on rows and columns"""
    return [
        ("row_lengths", row_lengths(), 40),
        ("empty_runs", empty_runs(), 20),
        ("short_rows", short_rows(), 25),
        ("rows1_nnz256", sized(1, 256), 100),
        ("rows1_nnz257", sized(1, 257), 100),
        ("rows31_nnz512", sized(31, 512), 10),
        ("rows32_nnz513", sized(32, 513), 10),
        ("rows33_nnz768", sized(33, 768), 12),
        ("rows33_nnz769", sized(33, 769), 12),
        ("rows32_nnz1", sized(32, 1), 1),
        ("thresholds_m8", thresholds(8), 8),
        ("thresholds_m1", thresholds(1), 1),
        ("one_column", one_column(), 1000),
        ("last_column", last_column(), 300),
    ]


def settings(m: int):
    """(m, seed, flags) to sample a shape with: its own m, m + 1, 1 and 2^31 - 1, seeds 0, -1 and 2^31 - 1 (the
    uint32 cast of the hash), and the Int/Int row rate (flags = 1, CCO_FLAG_ROWRATE_INTDIV)"""
    return [(m, 77, 0), (m, 0, 0), (m, -1, 1), (m + 1, 2 ** 31 - 1, 0), (1, 3, 0), (2 ** 31 - 1, 5, 0)]


def user_blocks(n_rows: int, world: int):
    """the users each rank of a `world`-rank job samples (user_block in cco_api.cu): S = ceil(U / W); the last blocks
    may be empty"""
    s = -(-n_rows // world)
    return [(min(r * s, n_rows), min(min(r * s, n_rows) + s, n_rows)) for r in range(world)]


def messy(mat, seed: int, n_rows: int | None = None):
    """the same matrix as unsorted, duplicated input (canonicalised, it is the matrix again), optionally padded to
    n_rows rows (the pad rows hold entries, so the largest row ids are used): shuffled rows, rows with every entry
    twice or three times, all-duplicate rows (one column repeated), heavy (> 256 entries) rows reversed, and sorted rows
    with an equal neighbour"""
    nr, nc, rp, ci = mat
    rng = np.random.default_rng(seed)
    rows = [list(ci[rp[r]:rp[r + 1]]) for r in range(nr)]
    n_rows = nr if n_rows is None else n_rows
    for r in range(nr, n_rows):
        rows.append(sorted(set(rng.integers(0, nc, 1 + r % 4).tolist())))
    out = []
    for r, row in enumerate(rows):
        kind = r % 5
        if not row:
            out.append(row)
        elif len(row) == 1 and kind != 4:
            out.append(row * (2 + r % 6))                                # all duplicates of one column
        elif len(row) > CHUNK:
            out.append(row[::-1] + row[: len(row) // 3])                 # heavy, unsorted, with duplicates
        elif kind == 0:
            out.append(list(rng.permutation(row)))                       # shuffled
        elif kind == 1:
            out.append(list(rng.permutation(row + row)))                 # every entry twice
        elif kind == 2:
            out.append((row + row + row)[::-1])                          # every entry three times, descending
        elif kind == 3:
            out.append(sorted(row + row[: 1 + len(row) // 2]))           # sorted, equal neighbours
        else:
            out.append(row)                                              # already canonical
    return csr(out, nc)
