"""Directed event sets for PopModel's rank histograms (k_pop_count, k_pop_score in csrc/cco_format.cuh; the bucket edges
of pop_args in csrc/cco_api.cu).

A random millisecond stream over days never lands on an inner bucket edge; these shapes put events one millisecond before,
on and after every edge of every mode, for windows whose durations cover every residue mod 2 and mod 3 (and durations too
short to have an older bucket at all), at starts of 0, the 2020s, before 1970 and straddling 0.  Further shapes hold every
subset of the buckets an item can be present in, the two empty-bucket rules, zero and negative scores, keys outside
[0, n_items), one hot key and a stream longer than one pass of the counting grid.

Each shape is (name, mode, start_ms, end_ms, n_items, items, times): items are integer keys, -1 and n_items included
where the shape says so (cco_pop_model skips them; a string route has no such key and drops those events first).
"""
from __future__ import annotations

import popmodel_ref as ref

MODES = ("popular", "trending", "hot")
DAY = 86_400_000
DURATIONS = tuple(range(14)) + tuple(7 * DAY + r for r in range(6))
STARTS = {"zero": 0, "2020s": 1_700_000_000_123, "before1970": -3 * 365 * DAY - 7}


def buckets(mode, start, end):
    e = ref.edges(mode, start, end)
    return list(zip(e[:-1], e[1:]))


def _present_everywhere(mode, start, end, item, k):
    """events that put `item` into every bucket that can hold an event, a different number in each so that scores differ"""
    items, times = [], []
    for b, (lo, hi) in enumerate(buckets(mode, start, end)):
        if hi > lo:
            n = 1 + (k + 2 * b) % 4
            items += [item] * n
            times += [lo] * (n - 1) + [hi - 1]
    return items, times


def edge_shape(mode, start, dur):
    """item k sits one millisecond before, on and after edge k, and in every bucket; the last item is in every bucket only"""
    end = start + dur
    edges = ref.edges(mode, start, end)
    items, times = [], []
    for k, e in enumerate(edges):
        items += [k, k, k]
        times += [e - 1, e, e + 1]
    for k in range(len(edges) + 1):
        i, t = _present_everywhere(mode, start, end, k, k)
        items += i
        times += t
    return len(edges) + 1, items, times


def edge_shapes():
    out = []
    for mode in MODES:
        for dur in DURATIONS:
            starts = dict(STARTS, straddle0=-(dur // 2) - (dur % 2))
            for sname, start in starts.items():
                n, items, times = edge_shape(mode, start, dur)
                out.append((f"edges-{mode}-dur{dur}-{sname}", mode, start, start + dur, n, items, times))
    return out


def _in_bucket(bk, b, n, item, frac=0):
    lo, hi = bk[b]
    return [item] * n, [lo + (frac * (hi - lo - 1)) // 4] * n


def subset_shape(mode, start, dur):
    """item s - 1 is present in exactly the buckets of bit set s, for every non-empty s; only the full set scores"""
    bk = buckets(mode, start, start + dur)
    items, times = [], []
    for s in range(1, 1 << len(bk)):
        for b in range(len(bk)):
            if (s >> b) & 1:
                i, t = _in_bucket(bk, b, 1 + (s + b) % 3, s - 1, s % 5)
                items += i
                times += t
    return (1 << len(bk)) - 1, items, times


def rule_shapes():
    out = []
    start, dur = STARTS["2020s"], 7 * DAY + 5
    end = start + dur
    for mode in ("trending", "hot"):
        bk = buckets(mode, start, end)
        nb = len(bk)
        n, items, times = subset_shape(mode, start, dur)
        out.append((f"subsets-{mode}", mode, start, end, n, items, times))
        # one bucket without any event, the others busy: older (empty result), middle (empty result, hot), newer (the join
        # then has no item, but for another reason than the older / middle rule)
        for empty in range(nb):
            items, times = [], []
            for b in range(nb):
                if b != empty:
                    for item in range(3):
                        i, t = _in_bucket(bk, b, item + 1, item, item)
                        items += i
                        times += t
            out.append((f"bucket{empty}-empty-{mode}", mode, start, end, 3, items, times))
        # nothing in the window: every event is before the start, on the end or after it
        out.append((f"all-empty-{mode}", mode, start, end, 2, [0, 1, 0, 1], [start - 1, end, end + 1, start - DAY]))
        out.append((f"no-events-{mode}", mode, start, end, 2, [], []))
        # scores: zero on purpose (present with 0, not absent), negative, positive
        counts = {"trending": [(2, 2), (1, 1), (5, 1), (1, 5), (3, 4)],
                  "hot": [(1, 2, 3), (2, 2, 2), (3, 2, 1), (1, 3, 1), (3, 1, 3), (1, 1, 4), (4, 1, 1)]}[mode]
        items, times = [], []
        for item, cs in enumerate(counts):
            for b, c in enumerate(cs):
                i, t = _in_bucket(bk, b, c, item, item % 5)
                items += i
                times += t
        out.append((f"scores-{mode}", mode, start, end, len(counts), items, times))
    out.append(("all-empty-popular", "popular", start, end, 2, [0, 1, 0], [start - 1, end, end + 1]))
    out.append(("no-events-popular", "popular", start, end, 2, [], []))
    return out


def key_shapes():
    """keys outside [0, n_items) among valid ones, one key hit by whole warps, and more events than one pass of a grid of
    8 CTAs of 256 threads per SM on a 132-SM device (270 336 threads)"""
    out = []
    start, dur = STARTS["2020s"], 7 * DAY + 4
    end = start + dur
    for mode in MODES:
        bk = buckets(mode, start, end)
        n_items = 5
        # the out-of-range keys carry the ONLY events of the older bucket of item-less rankings below, and many everywhere:
        # counted, they would change totals and scores
        items, times = [], []
        for b in range(len(bk)):
            for key, n in ((-1, 7), (n_items, 9), (0, 2), (4, 3 + b)):
                i, t = _in_bucket(bk, b, n, key, b)
                items += i
                times += t
        out.append((f"keys-outside-{mode}", mode, start, end, n_items, items, times))
        if mode != "popular":
            # only out-of-range keys in the older bucket: totals[0] must stay 0, so the result is empty
            items, times = _in_bucket(bk, 0, 40, -1)
            i2, t2 = _in_bucket(bk, 0, 40, n_items)
            items, times = items + i2, times + t2
            for b in range(1, len(bk)):
                i, t = _in_bucket(bk, b, 3, 1)
                items += i
                times += t
            out.append((f"keys-outside-only-older-{mode}", mode, start, end, n_items, items, times))
        # one hot key: 4096 consecutive events of key 2 in each bucket, a few of other keys between
        items, times = [], []
        for b in range(len(bk)):
            i, t = _in_bucket(bk, b, 4096 + 32 * b + b, 2, 1)
            items += i + [0, 1]
            times += t + [bk[b][0], bk[b][1] - 1]
        out.append((f"hot-key-{mode}", mode, start, end, 3, items, times))
        # more than one grid-stride pass: 300 007 events round-robin over 1000 keys and over the buckets' edges
        n = 300_007
        e = ref.edges(mode, start, end)
        probe = [start - 1] + [x + d for x in e for d in (-1, 0, 1)] + [start + dur // 5, end - dur // 7]
        items = [(q * 7) % 1000 for q in range(n)]
        times = [probe[(q * 13 + q // 1000) % len(probe)] for q in range(n)]
        out.append((f"grid-stride-{mode}", mode, start, end, 1000, items, times))
    return out


def shapes():
    return edge_shapes() + rule_shapes() + key_shapes()


def in_range(shape):
    """the shape without its out-of-range keys: what a route keyed by id strings can be given"""
    name, mode, start, end, n, items, times = shape
    keep = [q for q, j in enumerate(items) if 0 <= j < n]
    return name, mode, start, end, n, [items[q] for q in keep], [times[q] for q in keep]
