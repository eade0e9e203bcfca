"""Host-side mirror of Preparator.prepare + the two IndexedDatasetSpark.apply builders
(src/main/scala/Preparator.scala:44-87, 100-216): event (user, item) string pairs
per event name -> IndexedDatasets that share one user dictionary.

This is the INPUT side of the hot-path boundary (SURVEY.md 8a-H1).  `prepare` is host logic and the definition the
device path is held to; `prepare_on_device` returns the same value, built by cco_ingest_strings (SURVEY.md 8f-1)."""
from __future__ import annotations

from typing import Sequence

import numpy as np

from .indexed_dataset import BiDictionary, IndexedDataset


def _build(pairs: Sequence[tuple[str, str]], row_ids: BiDictionary, freeze_rows: bool) -> IndexedDataset:
    """IndexedDatasetSpark.apply(elements, existingRowIDs) (Preparator.scala:160-214): events of
    unknown users are dropped when a dictionary is passed in; item ids always come from the events
    that survive; duplicates collapse (`setQuick(col, 1.0)`)."""
    col_ids = BiDictionary()
    rows: list[int] = []
    cols: list[int] = []
    for user, item in pairs:
        if freeze_rows:
            r = row_ids.get(user)
            if r < 0:
                continue
        else:
            r = row_ids.add(user)
        rows.append(r)
        cols.append(col_ids.add(item))
    n_rows = row_ids.size
    r = np.asarray(rows, dtype=np.int64)
    c = np.asarray(cols, dtype=np.int64)
    if len(r):
        keys = np.unique(r * max(col_ids.size, 1) + c)   # dedup + sort by (row, col)
        r, c = keys // max(col_ids.size, 1), keys % max(col_ids.size, 1)
    row_ptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=n_rows), out=row_ptr[1:])
    return IndexedDataset(row_ptr, c.astype(np.int32), row_ids, col_ids, n_rows=n_rows, n_cols=col_ids.size)


def indexed_dataset_min_events(pairs: Sequence[tuple[str, str]], min_events_per_user: int) -> BiDictionary:
    """IndexedDatasetSpark.apply(elements, minEventsPerUser) (Preparator.scala:102-158): the dictionary
    of users with >= minEventsPerUser events, counting duplicates (`items.size` over groupByKey, :129-132)."""
    counts: dict[str, int] = {}
    for user, _ in pairs:
        counts[user] = counts.get(user, 0) + 1
    return BiDictionary(u for u, n in counts.items() if n >= min_events_per_user)


def prepare(actions: Sequence[tuple[str, Sequence[tuple[str, str]]]],
            min_events_per_user: int | None = None) -> list[tuple[str, IndexedDataset]]:
    """Preparator.prepare (Preparator.scala:44-87).  `actions` = TrainingData.actions, first = primary.
    Every later event type is restricted to the users known so far and all share one row space."""
    user_dict: BiDictionary | None = None
    out: list[tuple[str, IndexedDataset]] = []
    for idx, (name, pairs) in enumerate(actions):
        if idx == 0 and min_events_per_user is not None:
            passing = indexed_dataset_min_events(pairs, min_events_per_user)
            ids = _build(pairs, passing, freeze_rows=True)            # :62 rebuilt on passing users only
        elif user_dict is None:
            ids = _build(pairs, BiDictionary(), freeze_rows=False)
        else:
            ids = _build(pairs, user_dict, freeze_rows=True)          # :69 IndexedDatasetSpark(eventRDD, userDictionary)
        user_dict = ids.row_ids
        out.append((name, ids))
    return out


def prepare_on_device(actions: Sequence[tuple[str, Sequence[tuple[str, str]]]], min_events_per_user: int | None = None,
                      ctx=None) -> list[tuple[str, IndexedDataset]]:
    """`prepare` on the GPU: the same input and the same return value (host CSR + BiDictionaries, the secondary datasets
    sharing the primary's row_ids object).  Dictionaries and matrices are built by cco_ingest_strings; the host only
    encodes the ids (encode_ids) and decodes the dictionaries.  Callers that already hold id columns in the offsets +
    bytes layout skip the encoding with CcoContext.ingest_strings."""
    from .similarity_analysis import default_context, encode_ids
    if not actions:
        return []
    ctx = ctx or default_context()
    columns = []
    for _, pairs in actions:
        users, items = (list(x) for x in zip(*pairs)) if len(pairs) else ([], [])
        columns.append((*encode_ids(users), *encode_ids(items)))
    ds, user_ids, item_ids = ctx.ingest_strings(columns, min_events_per_user or 0)
    try:
        row_ids = BiDictionary(user_ids)
        out = []
        for t, (name, _) in enumerate(actions):
            n_rows, n_cols, row_ptr, col_idx = ctx.dataset_matrix(ds, t)
            out.append((name, IndexedDataset(row_ptr, col_idx, row_ids, BiDictionary(item_ids[t]), n_rows=n_rows, n_cols=n_cols)))
    finally:
        ctx.free_dataset(ds)
    return out
