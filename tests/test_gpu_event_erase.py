"""Erasure on the H100 (cco_event_log_erase, EventLog.erase): erasing users and items from a resident extendable log gives
every consumer's output a fresh read of the export without their lines gives -- ingest, calc_all, calc_pop, user and mixed
queries, refresh_properties and intern_stats -- for every flag combination, window and chunking, with the counters,
erased() and resident bytes held to the host mirror (events.erase_kept); erase composes with extend, save / load and the
clean write-back; and its edges and refusals."""
import ctypes as C
import json
import random

import numpy as np
import pytest

import universal_recommender_b200 as ur
from test_event_erase import id_sets, without
from test_event_extend import SEAM_CASES, W, dump, parsed
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from test_gpu_event_snapshot import image, state
from test_gpu_event_window import AP
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu

FLAGS = {"plain": {}, "history": dict(keep_history=True), "intern": dict(intern_ids=True),
         "all": dict(keep_history=True, intern_ids=True)}
WINDOWS = {"none": None, "both": W, "dedup": E.EventWindow(None, True)}
CHUNKS = {"one": None, "900": 900}


def consumers(ctx, log, now, flags, names) -> dict:
    """state() of test_gpu_event_snapshot without the counters, the ingest over `names` and the mixed queries of items
    taken from that ingest (an erase can leave a name without lines, which a fresh read does not list)"""
    out = state(ctx, log, now, flags)
    for k in ("info", "stats", "resident"):
        out.pop(k)
    ds, users, items = ctx.ingest_event_log(log, names)
    try:
        out["ingest"] = (users, items, [[np.asarray(a).tolist() for a in ctx.dataset_to_host(ds, t)] for t in range(len(names))])
    finally:
        ctx.free_dataset(ds)
    if "mixed_queries" in out:
        some = list(out["user_queries"][1])[:4] + ["nobody"]
        items_ = (items[0] if items else [])[:len(some)]
        items_ = items_ + [None] * (len(some) - len(items_))
        mq = ur.mixed_queries_from_events(log, out["calc_all"], AP, None, some, items_, [None] * len(some), now_ms=now, ctx=ctx)
        out["mixed_queries"] = (mq[0], np.asarray(mq[1]).tolist())
    return out


def info_counts(info) -> tuple:
    """what info says of the retained lines, names without events left out"""
    tr = {n: c for n, c in zip(info.names, info.n_training) if c}
    rk = {n: c for n, c in zip(info.names, info.n_ranking) if c}
    return tr, rk, info.n_property_events, info.n_property_items, info.n_property_fields, info.n_ignored


def assert_erased(ctx, log, data: bytes, users, items, window, now, flags, chunk=None, kept=None):
    """log (read from data in one read, or extended: kept, the mirror's state before the erase) after erase(users, items):
    its consumers against a fresh read of data - E, its counters against the mirror, and, for a log read in one chunk, its
    resident bytes against the fresh read's (an extend's buffers grow geometrically, a read's are exact)"""
    exact = kept is None and chunk is None
    kept = kept if kept is not None else E.clean_kept(parsed(data), window, now)
    want_kept, n = E.erase_kept(kept, users, items)
    st = log.erase(users=users, items=items)
    assert st.n_lines == n
    info = log.info()
    rest = without(data, users, items)
    with ctx.read_events(rest, chunk_bytes=chunk, window=window, now_ms=now, extendable=True, **flags) as fresh:
        fi = fresh.info()
        names = info.names or ["none"]
        assert consumers(ctx, log, now, flags, names) == consumers(ctx, fresh, now, flags, names)
        assert info_counts(info) == info_counts(fi)
        fresh_kept = E.clean_kept(parsed(rest), window, now)
        if exact:
            extra = len(want_kept.dup_times) - len(fresh_kept.dup_times)
            assert log.resident_bytes() == fresh.resident_bytes() + 8 * extra
    assert info.n_lines == len(E.export_lines(data))
    assert log.window_stats() == (want_kept.n_expired, want_kept.n_duplicates)
    assert log.erased() == n
    assert info.n_lines == len(want_kept.events) + want_kept.n_expired + want_kept.n_duplicates + log.erased()
    return want_kept, st


@pytest.mark.parametrize("chunk", sorted(CHUNKS))
@pytest.mark.parametrize("window", sorted(WINDOWS))
@pytest.mark.parametrize("flags", sorted(FLAGS))
def test_flags_windows_and_chunks(ctx, flags, window, chunk):
    data = random_export(21, 300)
    w, fl, cb = WINDOWS[window], FLAGS[flags], CHUNKS[chunk]
    for users, items in id_sets(data, 5)[:3]:
        with ctx.read_events(data, chunk_bytes=cb, window=w, now_ms=NOW, extendable=True, **fl) as log:
            assert_erased(ctx, log, data, users, items, w, NOW, fl, cb)


@pytest.mark.parametrize("case", sorted(SEAM_CASES))
def test_seam_cases_erase_then_extend_and_extend_then_erase(ctx, case):
    a, b, now1, now2 = SEAM_CASES[case]
    da, db = dump(a), dump(b)
    for flags in (FLAGS["plain"], FLAGS["all"]):
        for users, items in [(["u1"], []), ([], ["i1"]), ([], ["i2"]), (["u2"], ["i1"])]:
            with ctx.read_events(da, window=W, now_ms=now1, extendable=True, **flags) as log:
                log.erase(users=users, items=items)
                log.extend(db, window=W, now_ms=now2)
                with ctx.read_events(without(da, users, items) + db, window=W, now_ms=now2, extendable=True, **flags) as fresh:
                    names = log.info().names or ["none"]
                    assert consumers(ctx, log, now2, flags, names) == consumers(ctx, fresh, now2, flags, names)
                    kept, n = E.erase_kept(E.clean_kept(parsed(da), W, now1), users, items)
                    kept = E.extend_clean(kept, parsed(da + db)[len(a):], W, now2)
                    assert log.window_stats() == (kept.n_expired, kept.n_duplicates) and log.erased() == n
                    assert log.info().n_lines == len(kept.events) + kept.n_expired + kept.n_duplicates + n
            with ctx.read_events(da, window=W, now_ms=now1, extendable=True, **flags) as log:
                log.extend(db, window=W, now_ms=now2)
                kept = E.extend_clean(E.clean_kept(parsed(da), W, now1), parsed(da + db)[len(a):], W, now2)
                assert_erased(ctx, log, da + db, users, items, W, now2, flags, kept=kept)


def test_two_erases_are_one_erase_of_the_union(ctx):
    data = random_export(8, 400)
    (u1, i1), (u2, i2) = id_sets(data, 1)[2], id_sets(data, 2)[2]
    for flags in (FLAGS["plain"], FLAGS["all"]):
        with ctx.read_events(data, window=W, now_ms=NOW, extendable=True, **flags) as one, \
                ctx.read_events(data, window=W, now_ms=NOW, extendable=True, **flags) as two:
            one.erase(users=u1 + u2, items=i1 + i2)
            two.erase(users=u1, items=i1)
            two.erase(users=u2, items=i2)
            assert one.erased() == two.erased() > 0
            assert image(one) == image(two)


def test_erase_save_load_extend(ctx):
    lines = random_export(9, 400).splitlines()
    a, b = b"".join(x + b"\n" for x in lines[:250]), b"".join(x + b"\n" for x in lines[250:])
    users, items = id_sets(a, 3)[2]
    flags = FLAGS["all"]
    with ctx.read_events(a, window=W, now_ms=NOW, extendable=True, **flags) as log:
        before = image(log)
        n = log.erase(users=users, items=items).n_lines
        assert n > 0
        img = image(log)
        assert img != before
        with ctx.load_events(img) as back:
            assert back.erased() == n and image(back) == img
            back.extend(b, window=W, now_ms=NOW + DAY)
            with ctx.read_events(without(a, users, items) + b, window=W, now_ms=NOW + DAY, extendable=True, **flags) as fresh:
                names = back.info().names
                assert consumers(ctx, back, NOW + DAY, flags, names) == consumers(ctx, fresh, NOW + DAY, flags, names)
            assert back.erased() == n
            assert back.info().n_lines == len(lines)


@pytest.mark.parametrize("compress", [False, True], ids=["plain", "compress"])
def test_write_clean_after_an_erase(ctx, compress):
    from test_gpu_event_clean import clean, with_folds
    data = with_folds(random_export(12, 500), 12)
    for window in (E.EventWindow("5 days", True), None):
        for users, items in id_sets(data, 4)[:3] + [([], [f"fold{k}" for k in range(0, 40, 3)])]:
            with ctx.read_events(data, chunk_bytes=4096, window=window, now_ms=NOW, extendable=True) as log:
                log.erase(users=users, items=items)
                assert clean(log, data, compress_properties=compress) == E.clean_export(without(data, users, items), window, NOW, compress)


def test_erase_everything(ctx):
    data = random_export(3, 300)
    evs = parsed(data)
    users = sorted({e.entity_id for e in evs})
    items = sorted({e.target_id for e in evs if e.target_id is not None} | {e.entity_id for e in evs})
    for flags in (FLAGS["plain"], FLAGS["all"]):
        with ctx.read_events(data, window=W, now_ms=NOW, extendable=True, **flags) as log:
            log.erase(users=users, items=items)
            info = log.info()
            assert sum(info.n_training) == sum(info.n_ranking) == info.n_property_events == 0
            with pytest.raises(ValueError) as e1:
                ur.calc_all_from_events(log, AP, 0, now_ms=NOW, ctx=ctx)
            with ctx.read_events(without(data, users, items), window=W, now_ms=NOW, extendable=True, **flags) as fresh:
                with pytest.raises(ValueError) as e2:
                    ur.calc_all_from_events(fresh, AP, 0, now_ms=NOW, ctx=ctx)
            assert str(e1.value) == str(e2.value)
            if flags:
                assert log.intern_stats() == (0, 0)
            assert info.n_lines == info.n_ignored + sum(log.window_stats()) + log.erased()


def test_an_erase_that_matches_nothing_leaves_the_log_as_it_was(ctx):
    data = random_export(6, 300)
    for flags in (FLAGS["plain"], FLAGS["all"]):
        with ctx.read_events(data, chunk_bytes=1000, window=W, now_ms=NOW, extendable=True, **flags) as log:
            img, rb = image(log), log.resident_bytes()
            for users, items in [([], []), (["nobody", "nobody"], ["nothing", ""])]:
                st = log.erase(users=users, items=items)
                assert (st.n_lines, st.n_training, st.n_ranking, st.n_property_events) == (0, 0, 0, 0)
                assert log.resident_bytes() == rb and image(log) == img and log.erased() == 0


# (the id as its export spells it, the decoded id): escapes, escape-class characters, 4-byte and 2-byte UTF-8, 1 500 bytes
ODD = [(b'"b\\u006ft"', "bot"), (b'"q\\"x\\\\y\\n"', 'q"x\\y\n'), ('"\U0001F600\u00e9"'.encode(), "\U0001F600\u00e9"),
       (b'"' + b"L" * 1500 + b'"', "L" * 1500), (b'"i\\u0031"', "i1")]


def test_escapes_utf8_long_ids_and_lanes(ctx):
    """ids spelled with \\u escapes are erased by their decoded form; escape-class, 4-byte UTF-8 and 1 500-byte ids; the
    matches on the entries of lanes 0, 31 and 32 (and 63, 64), each odd id as a user and as an item"""
    lanes = (0, 31, 32, 63, 64)
    lines = []
    for k in range(70):
        j = lanes.index(k) if k in lanes else -1
        u = ODD[j][0] if j >= 0 else b'"u%d"' % (k % 9)
        i = ODD[(j + 1) % len(ODD)][0] if j >= 0 else b'"i%d"' % (k % 11)
        lines.append(b'{"event":"view","entityType":"user","entityId":%s,"targetEntityType":"item","targetEntityId":%s,"eventTime":"%s"}'
                     % (u, i, iso_ms(NOW - 1000 * k).encode()))
    data = b"\n".join(lines) + b"\n"
    decoded = [d for _, d in ODD]
    evs = parsed(data)
    assert {e.entity_id for e in evs} >= set(decoded) and {e.target_id for e in evs} >= set(decoded)
    for flags in (FLAGS["plain"], FLAGS["intern"]):
        for users, items in [(decoded[:2], []), ([], decoded[2:]), (decoded, decoded)]:
            with ctx.read_events(data, window=None, now_ms=NOW, extendable=True, **flags) as log:
                _, st = assert_erased(ctx, log, data, users, items, None, NOW, flags)
                assert st.n_lines > 0


def test_targeted_set_and_delete_of_erased_items(ctx):
    rows = [
        {"event": "$set", "entityType": "item", "entityId": "a", "properties": {"f": 1}},
        {"event": "$set", "entityType": "item", "entityId": "a", "targetEntityType": "item", "targetEntityId": "gone", "properties": {"g": 2}},
        {"event": "$set", "entityType": "item", "entityId": "gone", "properties": {"f": 3}},
        {"event": "$delete", "entityType": "item", "entityId": "gone"},
        {"event": "$set", "entityType": "item", "entityId": "gone", "properties": {"h": 4}},
        {"event": "$set", "entityType": "item", "entityId": "b", "properties": {"h": 5}},
        {"event": "buy", "entityType": "user", "entityId": "u1", "targetEntityType": "item", "targetEntityId": "gone"},
        {"event": "buy", "entityType": "user", "entityId": "u1", "targetEntityType": "item", "targetEntityId": "a"},
        {"event": "buy", "entityType": "user", "entityId": "u2", "targetEntityType": "item", "targetEntityId": "b"},
    ]
    for k, r in enumerate(rows):
        r["eventTime"] = iso_ms(NOW - 1000 * (len(rows) - k))
    data = b"".join(json.dumps(r).encode() + b"\n" for r in rows)
    for flags in (FLAGS["plain"], FLAGS["all"]):
        for window in (None, W):
            with ctx.read_events(data, window=window, now_ms=NOW, extendable=True, **flags) as log:
                _, st = assert_erased(ctx, log, data, [], ["gone"], window, NOW, flags)
                assert (st.n_lines, st.n_property_events, st.n_ranking, st.n_training) == (5, 4, 2, 1)


def test_more_entries_than_one_launch_has_threads(ctx):
    """300 000 training lines: the probe kernels' grid-stride loops run past one launch's 270 336 threads"""
    n = 300_000
    rows = [b'{"event":"view","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"i%d","eventTime":"%s"}'
            % (k % 5003, k % 2999, iso_ms(NOW - 1000 * (k % 86400)).encode()) for k in range(n)]
    data = b"\n".join(rows) + b"\n"
    rng = random.Random(3)
    users = [f"u{k}" for k in rng.sample(range(5003), 50)]
    items = [f"i{k}" for k in rng.sample(range(2999), 30)]
    for flags in (FLAGS["plain"], FLAGS["intern"]):
        with ctx.read_events(data, window=W, now_ms=NOW, extendable=True, **flags) as log:
            assert_erased(ctx, log, data, users, items, W, NOW, flags)


def test_refusals(ctx):
    data = dump(SEAM_CASES["a_expires"][0])
    L = N.lib()
    off = (C.c_int64 * 3)(0, 1, 2)

    def refused(h, message, n_users=1, offsets=off, status=N.E_INVALID_ARG):
        assert L.cco_event_log_erase(h, n_users, offsets, b"u1", 0, None, None, None) == status
        assert L.cco_last_error().decode() == message

    with ctx.read_events(data, window=W, now_ms=NOW, keep_history=True) as log:
        refused(log._h, "the log was read without CCO_LOG_EXTENDABLE (cco_event_log_begin_ex)")
        with pytest.raises(N.CcoError, match="CCO_LOG_EXTENDABLE"):
            log.erase(users=["u1"])
    with ctx.read_events(data, window=W, now_ms=NOW, extendable=True) as log:
        refused(log._h, "users: a negative count", n_users=-1)
        refused(log._h, "users: offsets[2] = 0 decreases", n_users=2, offsets=(C.c_int64 * 3)(0, 1, 0))
        refused(log._h, "users: offsets[0] = -1 is negative", offsets=(C.c_int64 * 2)(-1, 0))
        assert L.cco_event_log_erase(log._h, 0, None, None, 1, (C.c_int64 * 2)(0, 1), None, None) == N.E_INVALID_ARG
        assert L.cco_last_error().decode() == "null argument"
        assert L.cco_event_log_erase(log._h, 1, None, None, 0, None, None, None) == N.E_INVALID_ARG
        assert L.cco_last_error().decode() == "null argument"
        x = C.c_void_p()
        assert L.cco_event_log_clean_begin(log._h, 0, C.byref(x)) == N.OK
        refused(log._h, "a cleaner of the log is open (cco_event_log_clean_free)")
        L.cco_event_log_clean_free(x)
        assert L.cco_event_log_extend(log._h, None) == N.OK   # unfinished
        refused(log._h, "the log is not finished (cco_event_log_finish)")
        n = C.c_int64()
        assert L.cco_event_log_erased(log._h, C.byref(n)) == N.E_INVALID_ARG
        assert L.cco_event_log_finish(log._h) == N.OK
        assert log.erase(users=["u1"]).n_lines == 1 and log.erased() == 1   # still usable after the refusals
    with ctx.read_events(dump(SEAM_CASES["a_expires"][0]), window=W, now_ms=NOW, extendable=True) as log:
        with pytest.raises(N.CcoError):
            log.extend(b'{"event":"buy"}\n', window=W, now_ms=NOW)
        assert L.cco_event_log_erase(log._h, 1, off, b"u1", 0, None, None, None) == N.E_INVALID_ARG
        assert L.cco_last_error().decode().startswith("the read of this log failed: line 2:")
