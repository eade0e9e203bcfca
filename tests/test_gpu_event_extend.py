"""Extendable event logs on the H100 (cco_event_log_extend): a log read over A and extended with B under a later window is
the log one read of A followed by B under that window gives -- info, window_stats, the ingest's dictionaries and dataset,
and the bodies of calc_all_from_events, calc_pop_from_events, user_queries_from_events and mixed_queries_from_events."""
import json
import os
import random
import subprocess

import numpy as np
import pytest

import universal_recommender_b200 as ur
from test_event_extend import SEAM_CASES, W, build_c_program, dump
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from test_gpu_event_window import AP
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu

WINDOWS = {"none": None, "duration": E.EventWindow("5 days"), "dedup": E.EventWindow(None, True), "both": W}


def outputs(ctx, log, now) -> dict:
    """everything a consumer reads from a log"""
    out = {"info": log.info(), "stats": log.window_stats()}
    names = out["info"].names or ["none"]
    ds, users, items = ctx.ingest_event_log(log, names)
    try:
        out["ingest"] = (users, items, [[np.asarray(a).tolist() for a in ctx.dataset_to_host(ds, t)] for t in range(len(names))])
    finally:
        ctx.free_dataset(ds)
    kw = dict(now_ms=now, ctx=ctx)
    try:
        body = ur.calc_all_from_events(log, AP, 0, **kw)
    except ValueError as e:   # no event of the model's names: both logs say so
        out["calc_all"] = str(e)
        return out
    out["calc_all"] = body
    out["calc_pop"] = ur.calc_pop_from_events(body, log, AP, **kw)
    uq = ur.user_queries_from_events(log, AP, None, None, **kw)
    out["user_queries"] = (uq[0], list(uq[2]))
    some = list(uq[2])[:4] + ["nobody"]
    items_ = (items[0] if items else [])[:len(some)]
    items_ = items_ + [None] * (len(some) - len(items_))
    mq = ur.mixed_queries_from_events(log, body, AP, None, some, items_, [None] * len(some), **kw)
    out["mixed_queries"] = (mq[0], np.asarray(mq[1]).tolist())
    return out


def assert_extends_like_one_read(ctx, a: bytes, b: bytes, w1, now1, w2, now2, chunk_bytes=None):
    """read A extendable, extend with B, finish; the same outputs as one read of A + B (A's last line closed) under w2"""
    joined = a + (b"\n" if a and not a.endswith(b"\n") else b"") + b
    with ctx.read_events(a, chunk_bytes=chunk_bytes, window=w1, now_ms=now1, keep_history=True, extendable=True) as log:
        log.extend(b, window=w2, now_ms=now2)
        got = outputs(ctx, log, now2)
        with ctx.read_events(joined, window=w2, now_ms=now2, keep_history=True) as fresh:
            want = outputs(ctx, fresh, now2)
        assert got == want
        return got, log.resident_bytes()


def timed_export(seed: int, n: int, days: int) -> bytes:
    """random_export with its eventTimes spread over `days` days before NOW (its identities and repeats kept)"""
    rng = random.Random(seed)
    out = []
    for line in random_export(seed, n).splitlines():
        r = json.loads(line)
        r["eventTime"] = iso_ms(NOW - rng.randint(0, days * DAY))
        out.append(json.dumps(r).encode())
    return b"\n".join(out) + b"\n"


@pytest.mark.parametrize("newline", [True, False])
def test_split_points(ctx, newline):
    lines = random_export(3, 240).splitlines()
    n = len(lines)
    for k in (0, 1, n // 2, n - 1, n):
        a = b"\n".join(lines[:k]) + (b"\n" if newline and k else b"")
        b = b"".join(x + b"\n" for x in lines[k:])
        assert_extends_like_one_read(ctx, a, b, W, NOW, W, NOW + DAY // 2)


@pytest.mark.parametrize("window", sorted(WINDOWS))
def test_windows(ctx, window):
    lines = random_export(5, 300).splitlines()
    a, b = b"".join(x + b"\n" for x in lines[:170]), b"".join(x + b"\n" for x in lines[170:])
    w = WINDOWS[window]
    for now2 in (NOW, NOW + 1, NOW + 2 * DAY):
        assert_extends_like_one_read(ctx, a, b, w, NOW, w, now2)


@pytest.mark.parametrize("case", sorted(SEAM_CASES))
def test_seam_cases(ctx, case):
    a, b, now1, now2 = SEAM_CASES[case]
    for w in (W, E.EventWindow("5 days"), E.EventWindow(None, True)):
        assert_extends_like_one_read(ctx, dump(a), dump(b), w, now1, w, now2 if w.duration else now1)


def test_names_new_in_b_and_names_that_expire(ctx):
    old = [{"event": "gone", "entityType": "user", "entityId": "u1", "targetEntityType": "item", "targetEntityId": "i1",
            "eventTime": iso_ms(NOW - 4 * DAY)},
           {"event": "buy", "entityType": "user", "entityId": "u2", "targetEntityType": "item", "targetEntityId": "i2",
            "eventTime": iso_ms(NOW - DAY)}]
    new = [{"event": "fresh", "entityType": "user", "entityId": "u3", "targetEntityType": "item", "targetEntityId": "i1",
            "eventTime": iso_ms(NOW)},
           {"event": "buy", "entityType": "user", "entityId": "u3", "targetEntityType": "item", "targetEntityId": "i2",
            "eventTime": iso_ms(NOW)}]
    got, _ = assert_extends_like_one_read(ctx, dump(old), dump(new), W, NOW, W, NOW + 2 * DAY)
    info = got["info"]
    assert info.names == ["gone", "buy", "fresh"] and info.n_training == [0, 2, 1]
    assert got["stats"][0] == 1


def test_an_expired_delete_brings_the_sets_back(ctx):
    a, b, now1, now2 = SEAM_CASES["properties_around_the_cutoff"]
    got, _ = assert_extends_like_one_read(ctx, dump(a), dump(b), W, now1, W, now2)
    with ctx.read_events(dump(a), window=W, now_ms=now1) as log:
        before = log.info()
    assert (before.n_property_items, got["info"].n_property_items) == (1, 1)
    assert b'"f":1' in got["calc_all"].replace(b" ", b"")


def test_lines_of_b_straddle_small_chunks(ctx):
    lines = random_export(7, 200).splitlines()
    a, b = b"".join(x + b"\n" for x in lines[:90]), b"".join(x + b"\n" for x in lines[90:])
    assert_extends_like_one_read(ctx, a, b, W, NOW, W, NOW + DAY, chunk_bytes=300)


def test_ten_one_day_extends(ctx):
    """each step equals a fresh read of everything so far under its window; the resident bytes then stay within a small
    factor of a fresh extendable read's"""
    lines = timed_export(11, 1200, 15).splitlines()
    w = E.EventWindow("5 days", True)
    parts = np.array_split(np.arange(len(lines)), 11)
    part = lambda k: b"".join(lines[i] + b"\n" for i in parts[k])
    now = NOW - 10 * DAY
    with ctx.read_events(part(0), window=w, now_ms=now, keep_history=True, extendable=True) as log:
        for k in range(1, 11):
            now += DAY
            log.extend(part(k), window=w, now_ms=now)
            upto = b"".join(part(j) for j in range(k + 1))
            with ctx.read_events(upto, window=w, now_ms=now, keep_history=True) as fresh:
                assert outputs(ctx, log, now) == outputs(ctx, fresh, now)
        with ctx.read_events(upto, window=w, now_ms=now, keep_history=True, extendable=True) as fresh:
            rb, fb = log.resident_bytes(), fresh.resident_bytes()
        assert log.window_stats()[0] > 0
        # the same retained lines; buffers are exact fits after a compaction, geometric before one
        assert rb <= 2 * fb + (64 << 10), (rb, fb)


def test_errors(ctx):
    data = dump(SEAM_CASES["a_expires"][0])
    with ctx.read_events(data, window=W, now_ms=NOW, keep_history=True) as log:
        with pytest.raises(N.CcoError, match="CCO_LOG_EXTENDABLE"):
            log.extend(b"", window=W, now_ms=NOW)
    with ctx.read_events(data, window=W, now_ms=NOW, extendable=True) as log:
        with pytest.raises(N.CcoError, match="cannot|before"):
            log.extend(b"", window=W, now_ms=NOW - 1)
        with pytest.raises(N.CcoError, match="remove_duplicates"):
            log.extend(b"", window=E.EventWindow("5 days"), now_ms=NOW)
        bad = N.EventWindowT(NOW, 1, 7)
        assert N.lib().cco_event_log_extend(log._h, bad) == N.E_INVALID_ARG
        # still usable: a slide-only extend
        log.extend(b"", window=W, now_ms=NOW + DAY)
        assert log.info().n_lines == 2
        # an unfinished log: extend twice without finishing in between
        assert N.lib().cco_event_log_extend(log._h, None) == N.OK
        assert N.lib().cco_event_log_extend(log._h, None) == N.E_INVALID_ARG
        assert N.lib().cco_event_log_finish(log._h) == N.OK
    g = ur.CcoContext(devices=[0])
    try:
        with pytest.raises(N.CcoError) as e:
            g.read_events(data, window=W, now_ms=NOW, extendable=True)
        assert e.value.status == N.E_UNSUPPORTED
    finally:
        g.close()


def test_a_bad_line_in_b_names_the_global_line(ctx):
    a = dump(SEAM_CASES["a_expires"][0])
    b = dump(SEAM_CASES["b_later"][1]) + b'{"event":"buy","entityType":"user"}\n'
    with pytest.raises(N.CcoError) as whole:
        ctx.read_events(a + b, window=W, now_ms=NOW).free()
    with ctx.read_events(a, window=W, now_ms=NOW, extendable=True) as log:
        with pytest.raises(N.CcoError) as ext:
            log.extend(b, window=W, now_ms=NOW)
        assert "line 3" in str(whole.value) and str(ext.value) == str(whole.value)
        with pytest.raises(N.CcoError, match="failed"):
            log.info()


def test_c_program_reads_extends_and_reports(ctx, tmp_path):
    lines = random_export(13, 200).splitlines()
    a, b = b"".join(x + b"\n" for x in lines[:120]), b"".join(x + b"\n" for x in lines[120:])
    (tmp_path / "a.json").write_bytes(a)
    (tmp_path / "b.json").write_bytes(b)
    c1, c2 = NOW - 5 * DAY, NOW - 4 * DAY
    exe = build_c_program(tmp_path)
    p = subprocess.run([exe, str(tmp_path / "a.json"), str(tmp_path / "b.json"), str(c1), str(c2), "1"], capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout, p.stderr)
    x, d, n, resident = (int(v) for v in p.stdout.split())
    with ctx.read_events(a, chunk_bytes=1 << 16, window=W, now_ms=NOW, extendable=True) as log:
        log.extend(b, window=W, now_ms=NOW + DAY)
        assert (x, d, n, resident) == (*log.window_stats(), log.info().n_lines, log.resident_bytes())
    with ctx.read_events(a + b, window=W, now_ms=NOW + DAY) as fresh:
        assert (x, d) == fresh.window_stats()
