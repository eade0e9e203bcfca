"""Host restatement of the key-path ingest of an interned event log (CCO_LOG_INTERN_IDS): Preparator.prepare's rules over
integer keys, the way the device computes them -- the first entry of every key (a minimum over entry indices), a count
gate that counts duplicates, secondary users by a direct rank lookup, and the item gate over the surviving entries."""
from __future__ import annotations

from typing import Sequence

import numpy as np


def _group(keys: np.ndarray, n_keys: int, gate: np.ndarray | None, need: int) -> np.ndarray:
    """rank of every key (-1: not in the dictionary): the keys with >= need entries among those the gate passes (gate[e] >=
    0), numbered by their first such entry"""
    e = np.arange(len(keys), dtype=np.int64)
    ok = np.ones(len(keys), bool) if gate is None else gate >= 0
    first = np.full(n_keys, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(first, keys[ok], e[ok])
    count = np.bincount(keys[ok], minlength=n_keys)
    passing = np.flatnonzero((count >= need) & (count > 0))
    order = passing[np.argsort(first[passing], kind="stable")]
    rank = np.full(n_keys, -1, np.int64)
    rank[order] = np.arange(len(order))
    return rank


def ingest_keys(types: Sequence[tuple[np.ndarray, np.ndarray]], n_user_keys: int, n_item_keys: int, min_events_per_user: int):
    """types[t] = (user keys, item keys) of the training entries of name t, in the log's order.
    -> (user keys in dictionary order, [item keys in dictionary order per type], [(row_ptr, col_idx) per type])"""
    need = max(min_events_per_user, 1)
    urank = np.full(n_user_keys, -1, np.int64)
    user_order = np.zeros(0, np.int64)
    items, mats = [], []
    for t, (uk, ik) in enumerate(types):
        uk, ik = np.asarray(uk, np.int64), np.asarray(ik, np.int64)
        if t == 0:
            urank = _group(uk, n_user_keys, None, need)
            user_order = np.argsort(np.where(urank >= 0, urank, len(urank)), kind="stable")[: int((urank >= 0).sum())]
        uid = urank[uk] if len(uk) else np.zeros(0, np.int64)
        irank = _group(ik, n_item_keys, uid, 1)
        iid = np.where(uid >= 0, irank[ik] if len(ik) else ik, -1)
        items.append(np.argsort(np.where(irank >= 0, irank, len(irank)), kind="stable")[: int((irank >= 0).sum())])
        keep = uid >= 0
        n_cols = max(int((irank >= 0).sum()), 1)
        cells = np.unique(uid[keep] * n_cols + iid[keep])
        rows, cols = cells // n_cols, cells % n_cols
        row_ptr = np.zeros(len(user_order) + 1, np.int64)
        np.cumsum(np.bincount(rows, minlength=len(user_order)), out=row_ptr[1:])
        mats.append((row_ptr, cols.astype(np.int32)))
    return user_order, items, mats
