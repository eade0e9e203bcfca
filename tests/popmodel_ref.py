"""TEST INFRASTRUCTURE: PopModel's rank histograms read from PopModel.scala:113-182 alone, statement by statement.

Not derived from oracle/pop_oracle.py: that restatement computes bucket edges as start + k * (dur // n); this one builds
the Joda Interval objects the Scala builds (older, then middle from older's end and older's duration, then newer from
middle's end to the interval's end) and runs PEventStore.find, groupByKey and join over them.  tests/test_popmodel_ref.py
holds the two against each other on the directed shapes of tests/popmodel_shapes.py.  Scores are exact Python ints."""
from __future__ import annotations


class Interval:
    """org.joda.time.Interval: [start, end) in integer milliseconds, end >= start"""

    def __init__(self, start: int, end: int):
        if end < start:
            raise ValueError("The end instant must be greater than the start instant")
        self.start, self.end = int(start), int(end)

    @property
    def duration_millis(self) -> int:
        return self.end - self.start


def _java_div(a: int, b: int) -> int:
    """Java's long division truncates toward zero (durations are never negative, so this equals a // b here)"""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def find(events, interval: Interval):
    """PEventStore.find(startTime = interval.getStart, untilTime = interval.getEnd): startTime <= t < untilTime"""
    return [e for e in events if interval.start <= e[1] and e[1] < interval.end]


def calc_popular(events, interval: Interval) -> dict:
    """:113-122 -- events per targetEntityId in the interval; an item without an event there is not in the RDD"""
    out: dict = {}
    for item, _, n in find(events, interval):
        out[item] = out.get(item, 0) + n
    return out


def join(a: dict, b: dict) -> dict:
    """RDD.join: the keys of both sides, (a's value, b's value)"""
    return {k: (a[k], b[k]) for k in a if k in b}


def calc_trending(events, interval: Interval) -> dict:
    """:128-148"""
    half = _java_div(interval.duration_millis, 2)
    older = Interval(interval.start, interval.start + half)
    newer = Interval(interval.start + half, interval.end)
    older_pop = calc_popular(events, older)
    if not older_pop:                       # olderPopRDD.isEmpty() -> sc.emptyRDD
        return {}
    newer_pop = calc_popular(events, newer)
    return {item: n - o for item, (n, o) in join(newer_pop, older_pop).items()}


def calc_hot(events, interval: Interval) -> dict:
    """:153-182"""
    older = Interval(interval.start, interval.start + _java_div(interval.duration_millis, 3))
    middle = Interval(older.end, older.end + older.duration_millis)
    newer = Interval(middle.end, interval.end)
    older_pop = calc_popular(events, older)
    if not older_pop:
        return {}
    middle_pop = calc_popular(events, middle)
    if not middle_pop:
        return {}
    newer_pop = calc_popular(events, newer)
    new_velocity = {item: n - m for item, (n, m) in join(newer_pop, middle_pop).items()}
    old_velocity = {item: m - o for item, (m, o) in join(middle_pop, older_pop).items()}
    return {item: nv - ov for item, (nv, ov) in join(new_velocity, old_velocity).items()}


def pop_model(mode: str, items, times_ms, start_ms: int, end_ms: int, multiplicity=None) -> dict:
    """{item: integer score} of one ranking; items may be any hashable keys.  multiplicity[q] > 0: entry q stands for that
    many events of the same item at the same time (a ten-million-event stream written as a few entries)"""
    events = [(i, int(t), int(n)) for i, t, n in zip(items, times_ms, multiplicity or [1] * len(items))]
    interval = Interval(start_ms, end_ms)
    return {"popular": calc_popular, "trending": calc_trending, "hot": calc_hot}[mode](events, interval)


def edges(mode: str, start_ms: int, end_ms: int) -> list:
    """the bucket edges of a mode, oldest first: [start, inner..., end]"""
    iv = Interval(start_ms, end_ms)
    if mode == "popular":
        return [iv.start, iv.end]
    if mode == "trending":
        return [iv.start, iv.start + _java_div(iv.duration_millis, 2), iv.end]
    older_end = iv.start + _java_div(iv.duration_millis, 3)
    return [iv.start, older_end, older_end + (older_end - iv.start), iv.end]
