"""Test-side model of the path every output row takes through `k_rows`.

A numpy/Python restatement of the decisions of `make_cfg` and `enqueue_indicator` (universal_recommender_b200/csrc/
cco_api.cu) and of the per-row branches of `k_rows` (csrc/cco_kernels.cuh).  Each assignment names the source statement
it restates.  The GPU tests use it to check that a hand-made input reaches the path it targets; if the kernel's
scheduling changes, this file has to change with it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

SMEM_OPTIN_H100 = 232_448   # cudaDeviceProp::sharedMemPerBlockOptin of an H100 (227 KB)
CUT_BINS = 512              # cco_kernels.cuh: kCutBins
CUT_MAX_WORK = 65536        # k_rows: `a.row_work[item] < 65536u` (u16 cut bins cannot overflow)


def next_pow2(x: int) -> int:
    p = 1                   # cco_api.cu next_pow2
    while p < x:
        p <<= 1
    return p


@dataclass(frozen=True)
class BinCfg:
    group: int
    slots: int
    cap: int
    cbuf: int
    keep_max: int
    final_max: int
    dense: bool


def make_cfg(group: int, want_slots: int, top_k: int, n_cols_b: int, smem_optin: int = SMEM_OPTIN_H100) -> BinCfg:
    groups = 2 if group == 32 else 1                                            # `groups = group == 32 ? 2 : 1`
    final_max = next_pow2(top_k)                                                # `f.final_max = next_pow2(top_k)`
    cbuf = next_pow2(top_k + max(group, 128) + (64 if group == 32 else 0))     # `f.cbuf = next_pow2(top_k + ...)`
    if group == 32 and top_k + 32 <= 96:
        cbuf = 128                                                              # `if (group == 32 && top_k + 32 <= 96)`
    keep_max = max(final_max, (cbuf - group) // 2)                              # `f.keep_max = ...`
    caux = 0 if group == 32 else keep_max                                       # `f.caux = ...`
    fixed = (cbuf + caux) * 16 + 2 * 256 + 512 + 1024 + (group // 32) * 256     # `size_t fixed = ...`
    avail = (smem_optin - 1024) // groups                                       # `size_t avail = ...`
    max_slots = ((avail - fixed) // 4) & ~1023                                  # `int max_slots = ...`
    slots = min(want_slots, max_slots)                                          # `f.slots = ...`
    return BinCfg(group, slots, slots // 2, cbuf, keep_max, final_max,         # `f.cap = f.slots / 2`
                  n_cols_b <= slots)                                            # `f.dense = n_cols_b <= f.slots`


def warp_ok(top_k: int) -> bool:
    return top_k + 32 <= 256                                                    # enqueue_indicator: `warp_ok = k_eff + 32 <= 256`


def bin_specs(top_k: int) -> list[tuple[int, int, int]]:
    """(group, table words, largest w) per bin, largest rows first (enqueue_indicator: `spec`)."""
    spec = [(1024, 1 << 20, 0xFFFFFFFF), (1024, 1 << 20, 0xFFFFFFFF), (512, 16384, 8192), (256, 8192, 4096)]
    spec.append((128, 4096, 2048))                                              # both branches of `if (warp_ok)`
    if warp_ok(top_k):
        spec += [(32, 2048, 1024), (32, 1024, 512), (32, 512, 256)]
    return spec


def bins(top_k: int, n_cols_b: int, smem_optin: int = SMEM_OPTIN_H100):
    """-> (configs, h_thr): bin b takes rows with h_thr[b-1] >= w > h_thr[b] (k_bin_bounds; h_thr[-1] = inf, and the
    last bin ends at the first row without work)."""
    spec = bin_specs(top_k)
    cfgs = [make_cfg(g, s, top_k, n_cols_b, smem_optin) for g, s, _ in spec]   # `cfgs[b] = make_cfg(...)`
    h_thr = []
    for b in range(len(spec)):
        f = cfgs[min(b + 1, len(spec) - 1)]                                     # `cfgs[std::min(b + 1, kBins - 1)]`
        lim = spec[b + 1][2] if b + 1 < len(spec) else 0                        # `lim = b + 1 < kBins ? ... : 0u`
        if b + 1 < len(spec) and not f.dense:
            lim = min(lim, f.cap)                                               # `lim = std::min(lim, f.cap)`
        if b > 0:
            lim = min(lim, h_thr[b - 1])                                        # `h_thr[b] = std::min(h_thr[b], h_thr[b - 1])`
        h_thr.append(lim)
    return cfgs, h_thr


def bin_of(w: int, h_thr: list[int]) -> int | None:
    if w <= 0:
        return None                                                             # k_bin_bounds: rows without work run no kernel
    for b, t in enumerate(h_thr):
        if w > t:                                                               # `sorted_work[mid] > t`
            return b
    return None


def count_bits(n_cols_b: int) -> int:
    kb = 1
    while (1 << kb) - 1 <= n_cols_b:                                            # `while (((1LL << key_bits) - 1) <= n_cols_b)`
        kb += 1
    return 32 - kb                                                              # `count_bits = 32 - key_bits`


def counts_fit(n_cols_b: int, max_marg_a: int, max_marg_b: int) -> bool:
    cb = count_bits(n_cols_b)                                                   # `k11_max >= (1LL << count_bits)` -> UNSUPPORTED
    return cb >= 1 and min(max_marg_a, max_marg_b) < (1 << cb)


def key_shift(n_cols_b: int) -> int:
    s = 0
    while (max(n_cols_b - 1, 0) >> s) >= CUT_BINS:                              # `a.key_shift` loop
        s += 1
    return s


def key_levels(n_cols_b: int) -> int:
    """Radix levels of the key cut: the first covers key bits [shift, 32), each next one 9 bits lower (k_rows
    `sh = sh > 9 ? sh - 9 : 0`) until bit 0."""
    s, levels = key_shift(n_cols_b), 1
    while s > 0:
        s = s - 9 if s > 9 else 0
        levels += 1
    return levels


def llr_error_bound(n_users: int) -> float:
    return math.ldexp(n_users * math.log(n_users), -47) if n_users > 1 else 0.0  # cco_api.cu llr_error_bound


def cut_exact(n_users: int, max_marg_a: int, max_marg_b: int) -> bool:
    n, r, c = float(n_users), float(max_marg_a), float(max_marg_b)             # cco_api.cu cut_exact
    if r <= 0.0 or c <= 0.0:
        return True
    g = 2.0 / min(r * c, 0.5 * n)                                               # `g = 2.0 / std::min(r * c, 0.5 * n)`
    d = n - c - r + 1.0
    if d > 0.0:
        g = max(g, 2.0 * (1.0 / c - (r - 1.0) / d))                             # `g = std::max(g, 2 (1/c - (r-1)/d))`
    return g > 2.0 * llr_error_bound(n_users)


@dataclass(frozen=True)
class RowPath:
    bin: int
    group: int          # threads owning the row (32 = a warp)
    dense: bool
    n_pass: int
    keyed: bool
    cut: bool           # the level-1 cut runs
    levels: int         # key-cut radix levels (keyed rows; 1 for colB rows)

    def cell(self):
        """The coverage cell of the row: (owner, table, score path, cut depth or 'no cut', passes)."""
        cut = ("key%d" % self.levels if self.keyed else "colB") if self.cut else "nocut"
        return (self.group, "dense" if self.dense else "hash", "keyed" if self.keyed else "colB", cut,
                "multi" if self.n_pass > 1 else "single")


def row_path(w: int, ra: int, n_cols_b: int, max_marg_a: int, max_marg_b: int, n_users: int, top_k: int,
             smem_optin: int = SMEM_OPTIN_H100) -> RowPath | None:
    cfgs, h_thr = bins(top_k, n_cols_b, smem_optin)
    w32 = min(w, 0xFFFFFFFF)                                                    # k_row_work: `saturated at 2^32-1`
    b = bin_of(w32, h_thr)
    if b is None:
        return None
    f = cfgs[b]
    n_pass = 1
    if not f.dense:
        dbound = min(w32, n_cols_b)                                             # `dbound = w < n_cols_b ? w : n_cols_b`
        n_pass = max((dbound + f.cap - 1) // f.cap, 1)                          # `n_pass = (dbound + cap - 1) / cap`
    keyed = 2 * ra * max_marg_b < n_users                                       # `keyed = 2ull * ra * a.max_marg_b < N`
    cut = cut_exact(n_users, max_marg_a, max_marg_b) and w32 < CUT_MAX_WORK     # `a.cut_ok && a.row_work[item] < 65536u`
    return RowPath(b, f.group, f.dense, n_pass, keyed, cut, key_levels(n_cols_b) if keyed else 1)
