"""Clean write-back on the H100 (cco_event_log_clean_*, EventLog.write_clean, ur.clean_export): the compacted export is
events.clean_export's, byte for byte, for every window shape and source split, for logs read with every flag, extended
or loaded; lines at the warp-lane edges of the compaction; sources that are not what the log read fail naming the line and
leave no file; the compacted export trains to the same model; and the log is unchanged by a clean."""
import ctypes
import io
import json
import os
import random

import pytest

import universal_recommender_b200 as ur
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from test_gpu_event_extend import outputs, timed_export
from test_gpu_event_window import AP
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu

WINDOWS = {"none": None, "duration": E.EventWindow("5 days"), "dedup": E.EventWindow(None, True), "both": E.EventWindow("5 days", True)}


def with_folds(data: bytes, seed: int, n: int = 300) -> bytes:
    """data followed by $set / $unset lines of items of their own (ids no other line uses), with repeated and unset names,
    so that compressProperties has groups to fold"""
    rng = random.Random(seed)
    rows = []
    for k in range(n):
        props = {f"p{rng.randint(0, 6)}": rng.choice([1, "x", [1, 2], {"a": k}]) for _ in range(rng.randint(0, 4))}
        rows.append(json.dumps({"event": rng.choice(["$set", "$set", "$unset"]), "entityType": "item", "entityId": f"fold{rng.randint(0, 40)}",
                                "properties": props, "eventTime": iso_ms(NOW - rng.randint(0, 9 * DAY))}).encode())
    return data + b"\n".join(rows) + b"\n"


def clean(log, src, **kw) -> bytes:
    f = io.BytesIO()
    log.write_clean(src, f, **kw)
    return f.getvalue()


@pytest.mark.parametrize("compress", [False, True], ids=["plain", "compress"])
@pytest.mark.parametrize("name", list(WINDOWS))
def test_byte_parity_buffers_parts_and_splits(ctx, tmp_path, name, compress):
    w = WINDOWS[name]
    data = with_folds(random_export(11, 700), 11)
    want = E.clean_export(data, w, NOW, compress)
    with ctx.read_events(data, window=w, now_ms=NOW, extendable=True) as log:
        assert clean(log, data, compress_properties=compress) == want
        lines = data.splitlines()
        parts = []
        for k, (a, b) in enumerate([(0, 200), (200, 201), (201, 500), (500, len(lines))]):   # parts without a trailing '\n'
            p = tmp_path / f"part-{k:05d}"
            p.write_bytes(b"\n".join(lines[a:b]))
            parts.append(str(p))
        out = tmp_path / "clean.json"
        st = log.write_clean(str(tmp_path), str(out), compress_properties=compress)
        assert out.read_bytes() == want
        assert (st.n_lines, st.n_written, st.n_bytes) == (len(lines), len(E.export_lines(want)), len(want))
        kept = len(E.export_lines(E.clean_export(data, w, NOW)))
        assert st.n_written == kept - st.n_folded + st.n_compressed and (st.n_compressed > 30) == compress
        assert (st.n_expired, st.n_duplicates) == log.window_stats()
        assert not [n for n in os.listdir(tmp_path) if n.endswith(".tmp")]
        for step in (1, 7, 63, 64, 65, 4093):   # pieces that split lines at many byte positions
            assert clean(log, (data[k:k + step] for k in range(0, len(data), step)), compress_properties=compress) == want
    with ctx.read_events(data, chunk_bytes=3000, window=w, now_ms=NOW, extendable=True) as log:   # many device chunks
        assert clean(log, data, compress_properties=compress) == want


@pytest.mark.parametrize("history", [False, True])
@pytest.mark.parametrize("intern", [False, True])
def test_logs_read_extended_and_loaded(ctx, tmp_path, history, intern):
    w1, w2 = E.EventWindow("5 days", True), E.EventWindow("5 days", True)
    a, b = with_folds(timed_export(5, 500, 9), 5), with_folds(timed_export(6, 300, 3), 6, 100)
    with ctx.read_events(a, window=w1, now_ms=NOW, extendable=True, keep_history=history, intern_ids=intern) as log:
        assert clean(log, a) == E.clean_export(a, w1, NOW)
        log.extend(b, window=w2, now_ms=NOW + 2 * DAY)
        want = E.clean_export(a + b, w2, NOW + 2 * DAY)
        want_c = E.clean_export(a + b, w2, NOW + 2 * DAY, True)
        assert clean(log, [a, b]) == want
        assert clean(log, [a, b], compress_properties=True) == want_c
        snap = tmp_path / "log.snap"
        log.save(str(snap))
    with ctx.load_events(str(snap)) as loaded:
        assert clean(loaded, [a, b]) == want
        assert clean(loaded, [a, b], compress_properties=True) == want_c


def sized_line(n: int, k: int) -> bytes:
    """a training line of exactly n bytes (its '\\n' excluded)"""
    head = json.dumps({"event": "view", "entityType": "user", "entityId": f"u{k}", "targetEntityType": "item",
                       "targetEntityId": f"i{k % 7}", "eventTime": iso_ms(NOW - 1000 * k), "pad": ""}, separators=(",", ":"))
    assert len(head) <= n, n
    return head[:-2].encode() + b"x" * (n - len(head)) + b'"}'


def test_lane_edges_and_many_lines(ctx):
    # a warp copies a line's 8-byte words, one per lane: lines of 31, 32, 33, 64 and 65 words, a byte short, exact and
    # over, and lines at every alignment
    edges = [8 * n + d for n in (31, 32, 33, 64, 65) for d in (-1, 0, 1, 3)] + [1500]
    lengths = edges * 3 + list(range(180, 260))
    lines = [sized_line(n, k) for k, n in enumerate(lengths)]
    assert set(edges) <= {len(x) for x in lines}
    big = json.dumps({"event": "$set", "entityType": "item", "entityId": "i1", "properties": {"v": "y" * (3 << 20)},
                      "eventTime": iso_ms(NOW)}).encode()
    many = [sized_line(180 + k % 50, k) for k in range(40_000)]   # more kept lines than one launch has warps
    data = b"\n".join(lines + [big] + many)
    for w in (None, E.EventWindow("5 days", True)):
        want = E.clean_export(data, w, NOW)
        with ctx.read_events(data, chunk_bytes=1 << 20, window=w, now_ms=NOW, extendable=True) as log:
            assert clean(log, data) == want
            assert clean(log, (data[k:k + 1000003] for k in range(0, len(data), 1000003))) == want


def test_fold_group_and_field_edges(ctx):
    """folded groups of 0, 1, 31, 32, 33, 64 and 65 lines and of as many fields, with $unsets among them, and groups that
    only unset"""
    sizes = [0, 1, 31, 32, 33, 64, 65]
    rows, k = [], 0
    for n_lines in sizes:
        for n_fields in sizes:
            for kind in ("set", "unset"):
                item = f"g{n_lines}-{n_fields}-{kind}"
                for j in range(n_lines):
                    ev = "$unset" if kind == "unset" or j % 5 == 3 else "$set"
                    props = {f"f{(j + q) % max(n_fields, 1)}": j * 100 + q for q in range(n_fields)}
                    rows.append(json.dumps({"event": ev, "entityType": "item", "entityId": item, "properties": props,
                                            "eventTime": iso_ms(NOW - 1000 * ((k * 7919) % 5000))}).encode())
                    k += 1
    rng = random.Random(3)
    rng.shuffle(rows)
    data = b"\n".join(rows) + b"\n"
    want = E.clean_export(data, None, NOW, True)
    got_sizes = {len(json.loads(x)["properties"]) for x in E.export_lines(want)}
    assert {0, 1, 31, 32, 33, 64, 65} <= got_sizes, sorted(got_sizes)
    with ctx.read_events(data, window=E.EventWindow(None, True), now_ms=NOW, extendable=True) as log:
        assert clean(log, data, compress_properties=True) == E.clean_export(data, E.EventWindow(None, True), NOW, True)
    with ctx.read_events(data, chunk_bytes=1 << 16, now_ms=NOW, extendable=True) as log:
        f = io.BytesIO()
        st = log.write_clean(data, f, compress_properties=True)
        assert f.getvalue() == want
        groups = {(n, m, kd) for n in sizes for m in sizes for kd in ("set", "unset") if n >= 2}
        assert st.n_compressed == len(groups)


def mismatches(data: bytes):
    """(name, source) pairs that are not what a dedup log of `data` read"""
    lines = data.splitlines()
    kept = E.clean_events([E.parse_line(i, r) for i, r in enumerate(lines)], E.EventWindow("5 days", True), NOW)[0]
    e = next(e for e in kept if e.event == "buy")
    moved = lines[:]
    o = json.loads(moved[e.line])
    o["eventTime"] = iso_ms(e.time_ms + 1)
    moved[e.line] = json.dumps(o).encode()
    changed = lines[:]
    o = json.loads(changed[e.line])
    o["entityId"] = o["entityId"] + "z"
    changed[e.line] = json.dumps(o).encode()
    join = lambda x: b"\n".join(x) + b"\n"
    half = len(lines) // 2
    yield "swapped", join(lines[half:] + lines[:half]), None
    yield "time", join(moved), e.line
    yield "id", join(changed), e.line
    yield "added", join(lines + [lines[0]]), len(lines)
    yield "missing", join(lines[:-1]), len(lines) - 1


def test_source_mismatches_fail_and_leave_no_file(ctx, tmp_path):
    data = random_export(21, 600)
    with ctx.read_events(data, window=E.EventWindow("5 days", True), now_ms=NOW, extendable=True, keep_history=True) as log:
        before = outputs(ctx, log, NOW)
        for name, src, line in mismatches(data):
            out = tmp_path / f"{name}.json"
            with pytest.raises(N.CcoError) as ex:
                log.write_clean(src, str(out))
            assert "line" in str(ex.value), name
            if line is not None:
                assert f"line {line}" in str(ex.value), (name, str(ex.value))
            assert not os.listdir(tmp_path), name
        assert outputs(ctx, log, NOW) == before


def test_round_trip_trains_the_same_model(ctx, tmp_path):
    data = with_folds(timed_export(9, 3000, 30), 9)
    w = E.EventWindow("27 days", True)
    out = tmp_path / "clean.json"
    st = ur.clean_export(data, str(out), w, now_ms=NOW, ctx=ctx)
    assert st.n_lines == len(data.splitlines()) and st.n_bytes == out.stat().st_size
    for later in (NOW, NOW + DAY, NOW + 5 * DAY):
        a = ur.calc_all_from_events(out.read_bytes(), AP, now_ms=later, ctx=ctx, event_window=w)
        b = ur.calc_all_from_events(data, AP, now_ms=later, ctx=ctx, event_window=w)
        assert a == b
    wc = E.EventWindow("27 days", True, True)   # compressProperties: the same documents, properties unordered
    st = ur.clean_export(data, str(out), wc, now_ms=NOW, ctx=ctx)
    assert st.n_folded > 0
    docs = lambda body: sorted(json.dumps(json.loads(x), sort_keys=True) for x in body.splitlines())
    for later in (NOW, NOW + 5 * DAY):
        a = ur.calc_all_from_events(out.read_bytes(), AP, now_ms=later, ctx=ctx, event_window=wc)
        b = ur.calc_all_from_events(data, AP, now_ms=later, ctx=ctx, event_window=wc)
        assert docs(a) == docs(b)


def test_log_unchanged_refusals_and_compression(ctx, tmp_path):
    data = random_export(4, 500)
    w = E.EventWindow("5 days", True)
    with ctx.read_events(data, window=w, now_ms=NOW, extendable=True, keep_history=True) as log:
        snap0, res0, out0 = io.BytesIO(), log.resident_bytes(), outputs(ctx, log, NOW)
        log.save(snap0)
        clean(log, data)
        snap1 = io.BytesIO()
        log.save(snap1)
        assert snap0.getvalue() == snap1.getvalue() and log.resident_bytes() == res0 and outputs(ctx, log, NOW) == out0
        assert clean(log, data, compress_properties=True) == E.clean_export(data, w, NOW, True)
        snap2 = io.BytesIO()
        log.save(snap2)
        assert snap2.getvalue() == snap0.getvalue() and outputs(ctx, log, NOW) == out0
        L, x = ctx._L, ctypes.c_void_p()
        assert L.cco_event_log_clean_begin(log._h, 2, ctypes.byref(x)) == N.E_INVALID_ARG
        assert L.cco_event_log_clean_begin(log._h, 0, ctypes.byref(x)) == N.OK
        assert L.cco_event_log_extend(log._h, None) == N.E_INVALID_ARG
        assert L.cco_event_log_free(log._h) == N.E_INVALID_ARG
        assert L.cco_event_log_clean_free(x) == N.OK
    with ctx.read_events(data, window=w, now_ms=NOW) as plain:
        with pytest.raises(N.CcoInvalidArgument):
            plain.write_clean(data, io.BytesIO())
