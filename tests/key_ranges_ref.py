"""Host restatement of the key-range plan (DESIGN.md 3.1 "key ranges", include/cco_b200.h CCO_FLAG_KEY_RANGES).

B' columns are numbered by key = rank under (colB ascending, column id ascending), so `marg_key` (colB per key) is
non-decreasing and a key range [k0, k1) has its largest colB at k1 - 1.  The range's counts fit the packed 32-bit word
(key << count_bits | count) when bitlen(k1 - k0 + 1) + bitlen(min(max colA, marg_key[k1 - 1])) <= 32, with at least one
count bit.  The plan cuts greedily from key 0 upward, each range as long as it fits (and at most `cap` keys when cap > 0).
"""
from __future__ import annotations

import numpy as np


def fits(n_keys: int, k11_max: int) -> bool:
    """Keys 0 .. n_keys - 1 and counts up to k11_max in one 32-bit word: keys need (1 << kb) - 1 > n_keys."""
    kb = int(n_keys + 1).bit_length()
    cb = 32 - kb
    return cb >= 1 and int(k11_max) < (1 << cb)


def marg_key(marg_b) -> np.ndarray:
    """colB of every key: the column marginals in key order."""
    return np.sort(np.asarray(marg_b, dtype=np.int64), kind="stable")


def plan(marg_keys, max_marg_a: int, cap: int = 0) -> list[tuple[int, int]]:
    """Greedy key ranges [(k0, k1), ...] tiling [0, len(marg_keys)); raises ValueError if one key alone does not fit."""
    mk = np.asarray(marg_keys, dtype=np.int64)
    n = len(mk)

    def ok(k0, k1):
        return fits(k1 - k0, min(int(max_marg_a), int(mk[k1 - 1])))

    out, k0 = [], 0
    while k0 < n:
        top = min(n, k0 + cap) if cap > 0 else n
        if not ok(k0, k0 + 1):
            raise ValueError(f"key {k0}: its counts do not fit the packed word")
        lo, hi = k0 + 1, top
        while lo < hi:
            mid = lo + (hi - lo + 1) // 2
            if ok(k0, mid):
                lo = mid
            else:
                hi = mid - 1
        out.append((k0, lo))
        k0 = lo
    return out


def n_ranges(marg_b, max_marg_a: int, cap: int = 0) -> int:
    """What the device reports in last_key_ranges for one indicator: 1 when no plan is cut (the word fits and no cap,
    or an empty item space), else the plan's length."""
    mk = marg_key(marg_b)
    whole = fits(len(mk), min(int(max_marg_a), int(mk.max(initial=0))))
    if len(mk) == 0 or (whole and cap <= 0):
        return 1
    return len(plan(mk, max_marg_a, cap))
