"""The DataSource's eventWindow on the H100 (cco_event_log_begin_window): every calc_all_from_events / calc_pop_from_events
body under a window equals calc_all_on_device / calc_pop_on_device fed the host mirror's cleaned events, byte for byte,
and the drop counts equal the mirror's, at any chunking."""
import json

import pytest

import universal_recommender_b200 as ur
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from test_gpu_event_log_edges import docs_of, info_matches
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu

CUT = NOW - 5 * DAY
W = E.EventWindow("5 days", True)
AP = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy", "view"], "seed": 1, "rankings": [
    {"name": "popRank", "type": "popular", "eventNames": ["buy", "view"], "duration": "3650 days"},
    {"name": "trendRank", "type": "trending", "eventNames": ["buy"], "duration": "30 days"},
    {"name": "hotRank", "type": "hot", "eventNames": ["view"], "duration": "30 days"},
    {"name": "uniqueRank", "type": "random", "duration": "3650 days"}]})


def row(name, u, i=None, t=NOW - DAY, etype="user", **kw) -> dict:
    r = {"event": name, "entityType": etype, "entityId": u}
    if i is not None:
        r.update(targetEntityType="item", targetEntityId=i)
    r.update(kw)
    r["eventTime"] = iso_ms(t)
    return r


def dump(rows) -> bytes:
    return b"".join((r if isinstance(r, bytes) else json.dumps(r).encode()) + b"\n" for r in rows)


def check(ctx, data, window=W, now=NOW, min_events=0, chunks=(None,)):
    """device == mirror for the whole read and each chunk size; returns the mirror"""
    m = E.read_export(data, window, now)
    kw = dict(now_ms=now, ctx=ctx)
    want = ur.calc_all_on_device(m.events, m.set_events, AP, min_events, ranking_events=m.ranking_events, **kw)
    want_pop = ur.calc_pop_on_device(want, m.events, m.set_events, AP, ranking_events=m.ranking_events, **kw)
    assert ur.calc_all_from_events(data, AP, min_events, event_window=window, **kw) == want
    assert ur.calc_pop_from_events(want, data, AP, event_window=window, **kw) == want_pop
    for chunk in chunks:
        with ctx.read_events(data, chunk_bytes=chunk, window=window, now_ms=now) as log:
            assert log.window_stats() == (m.n_expired, m.n_duplicates)
            info_matches(log.info(), m, len(E.export_lines(data)))
            if chunk is not None:
                assert ur.calc_all_from_events(log, AP, min_events, **kw) == want
                assert ur.calc_pop_from_events(want, log, AP, **kw) == want_pop
    return m


def test_expiry_at_the_cutoff(ctx):
    rows = [row("buy", "u1", "i%d" % k, t) for k, t in enumerate([CUT - 1, CUT, CUT + 1, NOW])] + [row("view", "u1", "i0", CUT + 1)]
    for window in (W, E.EventWindow("5 days")):
        m = check(ctx, dump(rows), window)
        assert (m.n_expired, m.n_duplicates) == (2, 0)
        assert [i for _, _, i, _ in m.events] == ["i2", "i3", "i0"]


def test_old_set_and_unset_stay_an_old_delete_goes(ctx):
    rows = [row("buy", "u1", "a", NOW), row("buy", "u2", "b", NOW), row("view", "u1", "b", NOW),
            row("$set", "a", t=CUT - 9, etype="item", properties={"f": 1, "g": "x"}),
            row("$delete", "a", t=CUT - 5, etype="item"),                      # expired: the $set above counts again
            row("$unset", "a", t=CUT - 1, etype="item", properties={"g": None}),
            row("$set", "b", t=CUT - 3, etype="item", properties={"f": 2}),
            row("$delete", "b", t=CUT + 3, etype="item"),                      # kept: b has no properties
            row("$set", "u1", t=CUT - 7, properties={"age": 3}),                # a user's $set: kept, ignored
            row("$delete", "u1", t=CUT - 7)]                                   # expired
    data = dump(rows)
    assert E.read_export(data).set_events == []
    m = check(ctx, data)
    assert [(i, {k: v.text for k, v in d.items()}) for i, d in m.set_events] == [("a", {"f": "1"})]
    assert (m.n_expired, m.n_ignored) == (2, 1)


def test_duplicates_collapse_and_differences_stay(ctx):
    base = row("buy", "u1", "i1", NOW - 3 * DAY, prId="p", tags=["t"], properties={"a": 1, "b": [1, 2]})
    same = [dict(base, eventId="x"), dict(base, eventTime=iso_ms(NOW - DAY)), dict(base, creationTime=iso_ms(NOW)),
            dict(reversed(list(base.items())))]
    rep = json.dumps(base).replace('"properties": {', '"properties": {"a": 0, "b": 7, ', 1).encode()   # repeated names
    perm = dict(base, properties={"b": [1, 2], "a": 1})
    view = row("view", "u1")
    nulls = [dict(view, targetEntityType=None, targetEntityId=None), dict(view, prId=None), view]
    differ = [dict(base, tags=["t", "u"]), dict(base, tags=[]), dict(base, prId="q"), {k: v for k, v in base.items() if k != "prId"},
              dict(base, properties={"a": 2, "b": [1, 2]}), dict(base, properties={"a": 1}), dict(base, targetEntityType="thing"),
              dict(base, entityId="u2"), dict(base, event="view")]
    m = check(ctx, dump([base] + same + [rep, perm] + nulls + differ), chunks=(None, 64, 300))
    assert m.n_duplicates == len(same) + 2 + 2 and m.n_expired == 0


def test_no_tags_null_tags_and_empty_tags_are_one(ctx):
    b = row("buy", "u1", "i1")
    m = check(ctx, dump([b, dict(b, tags=None), dict(b, tags=[]), dict(b, tags=["x"])]))
    assert m.n_duplicates == 2


def test_the_kept_copy_is_the_latest_ties_to_the_later_line(ctx):
    # u1 buys i1 at t1 and t2 > t1: the kept time is t2, read back with one-millisecond popular windows
    t1, t2 = NOW - 3 * DAY, NOW - 2 * DAY + 17
    rows = [row("buy", "u1", "i1", t1), row("buy", "u2", "i2", t1), row("buy", "u1", "i1", t2), row("buy", "u1", "i1", t1 + 5)]
    data = dump(rows)
    check(ctx, data)
    with ctx.read_events(data, window=W, now_ms=NOW) as log:
        body = ctx.rerank_model(b"", rankings=[(f"r{k}", "popular", t, t + 1, ["buy"]) for k, t in enumerate([t1, t2, t1 + 5])], log=log)
    assert {d["id"]: sorted(k for k in d if k != "id") for d in docs_of(body)} == {"i1": ["r1"], "i2": ["r0"]}
    # equal times: the later line stays, so the first appearance of i1 moves after i2
    tie = dump([row("buy", "u1", "i1", t1), row("buy", "u2", "i2", t1), row("buy", "u1", "i1", t1)])
    m = check(ctx, tie)
    assert [i for _, _, i, _ in m.events] == ["i2", "i1"]


def test_min_events_per_user_counts_after_the_window(ctx):
    rows = [row("buy", "u1", "i1", NOW - DAY), row("buy", "u1", "i1", NOW - 2 * DAY), row("buy", "u2", "i1"), row("buy", "u2", "i2"),
            row("buy", "u3", "i2"), row("buy", "u3", "i3"), row("view", "u3", "i1")]
    for min_events in (1, 2):
        check(ctx, dump(rows), min_events=min_events)
    plain = ur.calc_all_from_events(dump(rows), AP, 2, now_ms=NOW, ctx=ctx)
    assert plain != ur.calc_all_from_events(dump(rows), AP, 2, now_ms=NOW, ctx=ctx, event_window=W)


def test_duplicates_across_every_chunking(ctx):
    rows = [row("buy", f"u{k % 3}", f"i{k % 3}", NOW - k * DAY // 2) for k in range(6)]       # u0 i0 / u1 i1 / u2 i2, twice
    rows += [row("view", "u1", "i0", NOW - 6 * DAY - k) for k in range(2)]                     # expired
    rows += [row("$set", "i0", t=NOW - k, etype="item", properties={"p": 1}) for k in range(2)]
    data = dump(rows)
    m = E.read_export(data, W, NOW)
    assert (m.n_duplicates, m.n_expired) == (4, 2)
    want = None
    rk = [("p", "popular", 0, NOW + 1, ["buy", "view"]), ("r", "random", 0, NOW + 1, [])]
    for chunk in list(range(64, len(data) + 1)):
        with ctx.read_events(data, chunk_bytes=chunk, window=W, now_ms=NOW) as log:
            assert log.window_stats() == (m.n_expired, m.n_duplicates), chunk
            info_matches(log.info(), m, len(rows))
            body = ctx.rerank_model(b"", rankings=rk, log=log)
        want = want or body
        assert body == want, chunk
    check(ctx, data, chunks=(64, 100, 1000))


def test_random_exports(ctx):
    for seed in range(3):
        data = random_export(seed, 3000)
        for window in (W, E.EventWindow("5 days"), E.EventWindow(None, True)):
            check(ctx, data, window, chunks=(4096,))


def test_a_3mb_duplicate(ctx):
    big = {"v": "x" * (3 << 20)}
    rows = [row("buy", "u1", "i1"), row("$set", "i1", etype="item", properties=big), row("buy", "u2", "i1"),
            row("$set", "i1", t=NOW - 2 * DAY, etype="item", properties=big), row("$set", "i1", etype="item", properties={"v": "y"})]
    m = check(ctx, dump(rows), chunks=(1 << 20,))
    assert m.n_duplicates == 1


def test_no_window_and_an_empty_window_are_the_plain_read(ctx):
    data = random_export(5, 2000)
    plain = ur.calc_all_from_events(data, AP, 0, now_ms=NOW, ctx=ctx)
    for window in (None, E.EventWindow()):
        assert ur.calc_all_from_events(data, AP, 0, now_ms=NOW, ctx=ctx, event_window=window) == plain
        with ctx.read_events(data, chunk_bytes=4096, window=window, now_ms=NOW) as log:
            assert log.window_stats() == (0, 0)
            assert ur.calc_all_from_events(log, AP, 0, now_ms=NOW, ctx=ctx) == plain
    with pytest.raises(ValueError):
        with ctx.read_events(data) as log:
            ur.calc_all_from_events(log, AP, 0, now_ms=NOW, ctx=ctx, event_window=W)


def test_bad_lines_fail_as_without_the_window(ctx):
    old = NOW - 9 * DAY
    bad_props = b'{"event":"$set","entityType":"item","entityId":"i","properties":{"a" 1},"eventTime":"%s"}' % iso_ms(NOW).encode()
    cases = [[row("buy", "u", "i"), row("buy", "", "i", old)],                      # an expired empty id
             [row("buy", "u", "i"), bad_props, row("buy", "u", "i"), bad_props],   # a duplicate with a malformed properties object
             [row("buy", "u", "i"), row("buy", "u", "i", old), b'{"event":"buy"}']]
    for rows in cases:
        data = dump(rows)
        with pytest.raises(ur.CcoError) as plain:
            ctx.read_events(data)
        for chunk in (None, 64):
            with pytest.raises(ur.CcoError) as windowed:
                ctx.read_events(data, chunk_bytes=chunk, window=W, now_ms=NOW)
            assert str(windowed.value) == str(plain.value)
