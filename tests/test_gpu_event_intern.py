"""Interned event logs on the H100 (CCO_LOG_INTERN_IDS): a log whose user and item ids took 32-bit keys as its lines were
read gives every consumer what the same lines read without interning give -- the ingest (now built from the keys) for any
names and min_events_per_user, and info, window_stats, calc_all, calc_pop, user and mixed queries -- across windows,
chunkings, extends and forced hash collisions; its intern tables hold exactly the ids of the retained training events."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import universal_recommender_b200 as ur
from test_event_extend import ROOT, W, dump
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from test_gpu_event_extend import WINDOWS, outputs, timed_export
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu


def ingest(ctx, log, names, min_events=0):
    ds, users, items = ctx.ingest_event_log(log, names, min_events)
    try:
        return users, items, [[np.asarray(a).tolist() for a in ctx.dataset_to_host(ds, t)] for t in range(len(names))]
    finally:
        ctx.free_dataset(ds)


def consumers(ctx, log, now, history):
    """outputs() of test_gpu_event_extend; without history only what needs none"""
    if history:
        return outputs(ctx, log, now)
    names = log.info().names or ["none"]
    return {"info": log.info(), "stats": log.window_stats(), "ingest": ingest(ctx, log, names)}


def ingest_variants(ctx, log):
    names = log.info().names
    lists = [names, names[::-1], names[:1], names[1:2] + ["absent"], ["absent"] + names[:2]]
    return [ingest(ctx, log, nm, m) for nm in lists if nm for m in (0, 1, 3)]


def live_ids(kept: E.KeptEvents) -> tuple[int, int]:
    """the distinct users and items of the training events the host mirror keeps"""
    train = [e for e in kept.events if e.entity_type == "user" and e.target_type == "item"]
    return len({e.entity_id for e in train}), len({e.target_id for e in train})


def retained_ids(data: bytes, window, now) -> tuple[int, int]:
    return live_ids(E.clean_kept([E.parse_line(i, raw) for i, raw in enumerate(E.export_lines(data))], window, now))


@pytest.mark.parametrize("history", [False, True])
@pytest.mark.parametrize("window", sorted(WINDOWS))
def test_interned_read_equals_plain_read(ctx, window, history):
    data = random_export(5, 400)
    w = WINDOWS[window]
    with ctx.read_events(data, window=w, now_ms=NOW, keep_history=history, intern_ids=True) as a, \
            ctx.read_events(data, window=w, now_ms=NOW, keep_history=history) as b:
        assert consumers(ctx, a, NOW, history) == consumers(ctx, b, NOW, history)
        assert ingest_variants(ctx, a) == ingest_variants(ctx, b)
        assert a.intern_stats() == retained_ids(data, w, NOW)


def test_small_chunks_straddle_ids_and_grow_the_tables(ctx):
    data = timed_export(21, 900, 8)
    for chunk in (120, 700, 4096):
        with ctx.read_events(data, chunk_bytes=chunk, window=W, now_ms=NOW, keep_history=True, intern_ids=True) as a, \
                ctx.read_events(data, window=W, now_ms=NOW, keep_history=True) as b:
            assert outputs(ctx, a, NOW) == outputs(ctx, b, NOW)
            assert ingest_variants(ctx, a) == ingest_variants(ctx, b)
            assert a.intern_stats() == retained_ids(data, W, NOW)


def test_ten_one_day_extends(ctx):
    """an interned and a plain extendable log side by side: after each extend, a fresh plain read's outputs, the mirror's
    live ids, and the resident bytes of a fresh interned extendable read"""
    lines = timed_export(11, 1200, 15).splitlines()
    # a few users and items that act only on the first day: their lines all expire during the run
    first_day = [json.dumps({"event": "buy", "entityType": "user", "entityId": f"gone{k}", "targetEntityType": "item",
                             "targetEntityId": f"gone-item{k}", "eventTime": iso_ms(NOW - 12 * DAY)}).encode() for k in range(5)]
    w = E.EventWindow("5 days", True)
    parts = np.array_split(np.arange(len(lines)), 11)
    part = lambda k: (b"".join(x + b"\n" for x in first_day) if k == 0 else b"") + b"".join(lines[i] + b"\n" for i in parts[k])
    now = NOW - 10 * DAY
    kw = dict(window=w, keep_history=True, extendable=True)
    with ctx.read_events(part(0), now_ms=now, intern_ids=True, **kw) as log, ctx.read_events(part(0), now_ms=now, **kw) as plain:
        first = [E.parse_line(i, raw) for i, raw in enumerate(E.export_lines(part(0)))]
        kept, n_lines, saw_gone = E.clean_kept(first, w, now), len(first), []
        for k in range(1, 11):
            now += DAY
            log.extend(part(k), window=w, now_ms=now)
            plain.extend(part(k), window=w, now_ms=now)
            upto = b"".join(part(j) for j in range(k + 1))
            with ctx.read_events(upto, window=w, now_ms=now, keep_history=True) as fresh:
                want = outputs(ctx, fresh, now)
            assert outputs(ctx, log, now) == want
            assert outputs(ctx, plain, now) == want
            with ctx.read_events(upto, now_ms=now, intern_ids=True, **kw) as fresh:
                assert log.resident_bytes() == fresh.resident_bytes()
                assert log.intern_stats() == fresh.intern_stats()
            new = [E.parse_line(n_lines + i, raw) for i, raw in enumerate(E.export_lines(part(k)))]
            kept, n_lines = E.extend_clean(kept, new, w, now), n_lines + len(new)
            assert log.intern_stats() == live_ids(kept)
            saw_gone.append(any(e.entity_id.startswith("gone") for e in kept.events))
        assert saw_gone[0] and not saw_gone[-1]   # the first day's ids left the tables on the way


def id_edge_export() -> bytes:
    ids = ["a", "abcdefg", "abcdefgh", "abcdefghi", "abcdefghijklmnop", "abcdefghijklmnopq", "x" * 1500,
           "abcdefgh-tail1", "abcdefgh-tail2", "abcdefghijklmnop-1", "abcdefghijklmnop-2", "é", "日本語", "😀id", "a\"b", "a\\b"]
    out = []
    for k, u in enumerate(ids):
        for j, i in enumerate(ids[k:k + 4]):
            out.append(json.dumps({"event": "buy" if j % 2 else "view", "entityType": "user", "entityId": u,
                                   "targetEntityType": "item", "targetEntityId": i, "eventTime": iso_ms(NOW - DAY)},
                                  ensure_ascii=bool(j % 2)))
    # JSON escapes that decode to ids above: one key each
    out.append('{"event":"buy","entityType":"user","entityId":"\\u0061","targetEntityType":"item","targetEntityId":"\\u00e9",'
               f'"eventTime":"{iso_ms(NOW - DAY)}"}}')
    out.append('{"event":"view","entityType":"user","entityId":"a\\u0022b","targetEntityType":"item","targetEntityId":"\\/x",'
               f'"eventTime":"{iso_ms(NOW - DAY)}"}}')
    return ("\n".join(out) + "\n").encode("utf-8")


@pytest.mark.parametrize("bits", [64, 4, 0])
def test_string_edges_and_hash_collisions(ctx, bits):
    data = id_edge_export() + random_export(9, 200)
    ctx.debug_intern_hash_bits(bits)
    try:
        for chunk in (None, 256):
            with ctx.read_events(data, chunk_bytes=chunk, window=W, now_ms=NOW, keep_history=True, intern_ids=True) as a, \
                    ctx.read_events(data, window=W, now_ms=NOW, keep_history=True) as b:
                assert outputs(ctx, a, NOW) == outputs(ctx, b, NOW)
                assert ingest_variants(ctx, a) == ingest_variants(ctx, b)
                assert a.intern_stats() == retained_ids(data, W, NOW)
                users = ingest(ctx, a, ["buy", "view"])[0]
                assert "a" in users and "a\"b" in users and "x" * 1500 in users
    finally:
        ctx.debug_intern_hash_bits(64)


def test_repeat_ingest_is_the_same(ctx):
    data = random_export(3, 300)
    with ctx.read_events(data, window=W, now_ms=NOW, intern_ids=True) as log:
        names = log.info().names
        assert ingest(ctx, log, names, 2) == ingest(ctx, log, names, 2)
        assert ingest_variants(ctx, log) == ingest_variants(ctx, log)


def test_errors(ctx):
    data = random_export(3, 50)
    with ctx.read_events(data, window=W, now_ms=NOW, extendable=True) as log:
        with pytest.raises(N.CcoError, match="CCO_LOG_INTERN_IDS"):
            log.intern_stats()
    assert N.lib().cco_debug_intern_hash_bits(ctx._h, 65) == N.E_INVALID_ARG
    h = C.c_void_p()
    assert N.lib().cco_event_log_begin_ex(ctx._h, 1, None, 8, C.byref(h)) == N.E_INVALID_ARG   # unknown flags are refused
    g = ur.CcoContext(devices=[0])
    try:
        with pytest.raises(N.CcoError) as e:
            g.read_events(data, window=W, now_ms=NOW, intern_ids=True)
        assert e.value.status == N.E_UNSUPPORTED
    finally:
        g.close()
    # a bad line in an extend names its global line, and the log fails
    a = dump([{"event": "buy", "entityType": "user", "entityId": "u", "targetEntityType": "item", "targetEntityId": "i",
               "eventTime": iso_ms(NOW)}] * 2)
    b = b'{"event":"buy","entityType":"user","entityId":"v","targetEntityType":"item","targetEntityId":"j","eventTime":"' + \
        iso_ms(NOW).encode() + b'"}\n{"event":"buy","entityType":"user"}\n'
    with pytest.raises(N.CcoError) as whole:
        ctx.read_events(a + b, window=W, now_ms=NOW).free()
    with ctx.read_events(a, window=W, now_ms=NOW, extendable=True, intern_ids=True) as log:
        with pytest.raises(N.CcoError) as ext:
            log.extend(b, window=W, now_ms=NOW)
        assert "line 3" in str(whole.value) and str(ext.value) == str(whole.value)
        with pytest.raises(N.CcoError, match="failed"):
            log.intern_stats()


def test_c_program_reads_extends_ingests_and_reports(ctx, tmp_path):
    lines = timed_export(13, 300, 8).splitlines()
    a, b = b"".join(x + b"\n" for x in lines[:180]), b"".join(x + b"\n" for x in lines[180:])
    (tmp_path / "a.json").write_bytes(a)
    (tmp_path / "b.json").write_bytes(b)
    libdir = os.path.dirname(N.LIB_PATH)
    exe = str(tmp_path / "event_intern_abi_check")
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_intern_abi_check.c"), "-o", exe, "-L", libdir, "-lcco_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    p = subprocess.run([exe], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout.strip() == "ok", (p.stdout, p.stderr)
    c1, c2 = NOW - 5 * DAY, NOW - 4 * DAY
    p = subprocess.run([exe, str(tmp_path / "a.json"), str(tmp_path / "b.json"), str(c1), str(c2)], capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout, p.stderr)
    got = [int(v) for v in p.stdout.split()]
    w = E.EventWindow("5 days", True)
    with ctx.read_events(a, chunk_bytes=1 << 16, window=w, now_ms=NOW, extendable=True, intern_ids=True) as log:
        log.extend(b, window=w, now_ms=NOW + DAY)
        users, items, _ = ingest(ctx, log, ["buy", "view"])
        assert got == [*log.intern_stats(), len(users), len(items[0]), len(items[1]), log.resident_bytes()]
    with ctx.read_events(a + b, window=w, now_ms=NOW + DAY) as fresh:
        assert (users, items) == ingest(ctx, fresh, ["buy", "view"])[:2]
