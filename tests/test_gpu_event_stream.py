"""Streamed event-log reads (cco_event_log_begin / _append / _finish, CcoContext.read_events over paths, directories and
generators) on the H100: every case gives what cco_event_log_read of the concatenated bytes gives -- info, the ingest's
dictionaries and matrices, the calcAll body (format_model with log=) and the calcPop body (rerank_model with log=) -- and
the same error code and message."""
import ctypes
import json
import random

import pytest

import universal_recommender_b200 as ur
from test_gpu_events import GOOD, random_export
from test_events_mirror import iso_ms
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu

NAMES = ["buy", "view", "like"]
AP = ur.URAlgorithmParams.from_engine_json({"eventNames": NAMES, "seed": 1, "rankings": [
    {"name": "popRank", "type": "popular", "eventNames": ["buy", "view"], "duration": 10 ** 9},
    {"name": "uniqueRank", "type": "random", "duration": 10 ** 9}]})
NOW = 2 * 10 ** 12


def state(ctx, log, full=True):
    """what a log gives: info, the calcAll body and, with full, the ingest and the calcPop body"""
    i = log.info()
    out = [(i.n_lines, i.names, i.n_training, i.n_ranking, i.n_property_events, i.n_property_items, i.n_property_fields, i.n_ignored)]
    try:
        body = ur.calc_all_from_events(log, AP, 0, now_ms=NOW, ctx=ctx)
    except ValueError as e:   # no events of the model's names
        return out + [str(e)]
    out.append(body)
    if full:
        out.append(ur.calc_pop_from_events(body, log, AP, now_ms=NOW, ctx=ctx))
        ds, users, items = ctx.ingest_event_log(log, NAMES + ["nothing"], 2)
        try:
            out += [users, items] + [[getattr(x, "tolist", lambda: x)() for x in ctx.dataset_to_host(ds, t)] for t in range(len(NAMES) + 1)]
        finally:
            ctx.free_dataset(ds)
    return out


def whole(ctx, data: bytes, full=True):
    with ctx.read_events(data) as log:
        return state(ctx, log, full)


def streamed(ctx, pieces, chunk_bytes: int, full=True):
    with ctx.read_events(iter(pieces), chunk_bytes=chunk_bytes) as log:
        return state(ctx, log, full)


def row(name, user, item, t, **kw):
    r = {"event": name, "entityType": "user", "entityId": user, "targetEntityType": "item", "targetEntityId": item, "eventTime": iso_ms(t)}
    r.update(kw)
    return json.dumps(r, ensure_ascii=False).encode()


# a small export with what a split can fall inside: '\r\n', \u escapes, backslash runs, multi-byte UTF-8, a property event,
# an ignored line and a final line without '\n'
SMALL = b"\r\n".join([
    row("buy", "u1", "i1", 1000),
    b'{"event":"view","entityType":"user","entityId":"\\u00fc\\\\\\\\x","targetEntityType":"item","targetEntityId":"i\\u00e9","eventTime":"1970-01-01T00:00:02Z"}',
    "{\"event\":\"buy\",\"entityType\":\"user\",\"entityId\":\"ü2\",\"targetEntityType\":\"item\",\"targetEntityId\":\"𝄞\",\"eventTime\":\"1970-01-01T00:00:03Z\"}".encode(),
    b'{"event":"$set","entityType":"item","entityId":"i1","properties":{"a":"\\"q\\\\","b":[1,2]},"eventTime":"1970-01-01T00:00:01Z"}',
    b'{"event":"rate","entityType":"user","entityId":"u1","eventTime":"1970-01-01T00:00:04Z"}',
    row("like", "u1", "i\\2", 5000)])


def test_every_split_offset_of_a_small_export(ctx):
    """two appends at every byte offset, the staging as large as the first: chunks end at every line and carry every tail"""
    want = whole(ctx, SMALL, full=False)
    for o in range(1, len(SMALL)):
        assert streamed(ctx, [SMALL[:o], SMALL[o:]], o, full=False) == want, o


def test_one_byte_appends(ctx):
    want = whole(ctx, SMALL)
    assert streamed(ctx, [SMALL[k:k + 1] for k in range(len(SMALL))], 1 << 20) == want
    assert streamed(ctx, [SMALL[k:k + 1] for k in range(len(SMALL))], 100) == want


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("chunk_bytes", [64, 1024, 1 << 22])
def test_random_splits_of_random_exports(ctx, seed, chunk_bytes):
    data = random_export(seed)
    want = whole(ctx, data)
    rng = random.Random(seed * 7 + chunk_bytes)
    cuts = sorted(rng.sample(range(1, len(data)), 40))
    pieces = [data[a:b] for a, b in zip([0] + cuts, cuts + [len(data)])]
    assert streamed(ctx, pieces, chunk_bytes) == want
    m = E.read_export(data)
    with ctx.read_events(iter(pieces), chunk_bytes=chunk_bytes) as log:
        info = log.info()
        assert info.names == m.names and info.n_ranking == [len(m.ranking_events[n]) for n in m.names]


def test_a_boundary_right_after_a_newline_and_a_final_newline(ctx):
    data = SMALL + b"\n"
    k = data.index(b"\n") + 1
    assert streamed(ctx, [data[:k], data[k:]], k) == whole(ctx, data)


def test_a_line_longer_than_the_staging_grows_it(ctx):
    big = "x" * (3 << 20)
    data = b"\n".join([row("buy", "u1", "i1", 1), row("buy", "u2", big, 2), row("view", "u2", "i1", 3)])
    want = whole(ctx, data)
    assert streamed(ctx, [data[k:k + 100_000] for k in range(0, len(data), 100_000)], 1 << 20) == want


def test_empty_log(ctx):
    for pieces in ([], [b""]):
        with ctx.read_events(iter(pieces), chunk_bytes=64) as log:
            with ctx.read_events(b"") as w:
                assert state(ctx, log) == state(ctx, w)


def prop(kind, item, t, **props):
    r = {"event": kind, "entityType": "item", "entityId": item, "eventTime": iso_ms(t)}
    if kind != "$delete":
        r["properties"] = props
    return json.dumps(r).encode()


def test_properties_across_chunks(ctx):
    """tied eventTimes of $set / $unset / $delete of one item in different chunks (ties go to the later line); an item whose
    first property event comes after its fields' names first appear; an "id"-only item"""
    rows = [row("buy", f"u{k}", f"i{k % 3}", k) for k in range(6)]
    rows += [prop("$set", "late", 50, color="red", size=1), prop("$set", "i0", 10, color="blue"), prop("$delete", "i0", 10),
             prop("$set", "i0", 10, size=3), row("view", "u1", "i0", 7), prop("$unset", "i1", 20, color=None),
             prop("$set", "i1", 20, color="green", size=2), prop("$unset", "i1", 20, size=None), prop("$set", "x", 5, a=1),
             prop("$unset", "x", 5, a=None), prop("$set", "i2", 1, shape="round"), prop("$delete", "i2", 1)]
    data = b"\n".join(rows) + b"\n"
    want = whole(ctx, data)
    for chunk in (64, 300, 1000):
        assert streamed(ctx, [data], chunk) == want, chunk
    m = E.read_export(data)
    with ctx.read_events(iter([data]), chunk_bytes=64) as log:
        i = log.info()
        assert i.n_property_items == len(m.set_events) and i.n_property_fields == len({f for _, d in m.set_events for f in d})
    assert dict(m.set_events)["x"] == {}


def test_names_across_chunks(ctx):
    rng = random.Random(4)
    rows = [row(rng.choice(["buy", "view"]), f"u{rng.randint(0, 30)}", f"i{rng.randint(0, 40)}", k) for k in range(400)]
    rows.insert(350, row("like", "u1", "i1", 999))   # a name first seen in a late chunk
    data = b"\n".join(rows)
    want = whole(ctx, data)
    for chunk in (200, 4096):
        assert streamed(ctx, [data], chunk) == want


BAD = [
    b'{"event":"buy","entityType":"user","entityId":"","targetEntityType":"item","targetEntityId":"i","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","targetEntityType":"item","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","eventTime":"2020-01-01"}',
    b'{"event":"buy","entityType":"user","entityId":5,"eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z","properties":[]}',
    b'{"event":"buy","entityType":"user","eventTime":"2020-01-01T00:00:00Z"}',
    b'[1]', b'', b'{"event":"buy"', b'{"event":"b\\x"}',
    b'{"event":"$set","entityType":"item","entityId":"i","eventTime":"2020-01-01T00:00:00Z","properties":{"a" 1}}',
]


def error_of(fn):
    with pytest.raises(N.CcoError) as e:
        fn()
    return e.value.status, str(e.value)


@pytest.mark.parametrize("bad", range(len(BAD)))
def test_a_bad_line_anywhere_gives_the_error_of_the_whole_read(ctx, bad):
    n, chunk = 30, 4 * (len(GOOD) + 1)
    for at in (0, 1, 13, 14, 15, n - 1):   # chunk 0, middle chunks, straddling chunk ends, the tail parsed by finish
        if at == n - 1 and not BAD[bad]:
            continue   # an empty last line is no line
        rows = [GOOD] * n
        rows[at] = BAD[bad]
        data = b"\n".join(rows)
        want = error_of(lambda: ctx.read_events(data))
        assert f"line {at}:" in want[1]
        assert error_of(lambda: ctx.read_events(iter([data]), chunk_bytes=chunk)) == want
        cut = sum(len(r) + 1 for r in rows[:at]) + len(rows[at]) // 2
        assert error_of(lambda: ctx.read_events(iter([data[:cut], data[cut:]]), chunk_bytes=chunk)) == want


def test_calls_before_finish_and_after_a_failure(ctx):
    L = N.lib()
    h = ctypes.c_void_p()
    info = N.EventLogInfoT()
    ds = ctypes.c_void_p()
    nm = (ctypes.c_char_p * 1)(b"v")
    assert L.cco_event_log_begin(ctx._h, 4096, ctypes.byref(h)) == N.OK
    try:
        assert L.cco_event_log_append(h, GOOD + b"\n", len(GOOD) + 1) == N.OK
        assert L.cco_event_log_info(h, ctypes.byref(info)) == N.E_INVALID_ARG
        assert L.cco_event_log_ingest(ctx._h, h, 1, nm, 0, ctypes.byref(ds)) == N.E_INVALID_ARG
        bad = GOOD + b"\n[1]\n"
        assert L.cco_event_log_append(h, bad, len(bad)) == N.OK   # staged, not judged yet
        filler = (GOOD + b"\n") * 60
        assert L.cco_event_log_append(h, filler, len(filler)) == N.E_INVALID_ARG   # the staging filled: line 2 is judged
        msg = L.cco_last_error()
        assert b"line 2:" in msg
        for rc in (L.cco_event_log_append(h, GOOD, len(GOOD)), L.cco_event_log_finish(h), L.cco_event_log_info(h, ctypes.byref(info)),
                   L.cco_event_log_ingest(ctx._h, h, 1, nm, 0, ctypes.byref(ds))):
            assert rc == N.E_INVALID_ARG and msg in L.cco_last_error()
    finally:
        assert L.cco_event_log_free(h) == N.OK
    assert L.cco_event_log_begin(ctx._h, 64, ctypes.byref(h)) == N.OK
    try:
        assert L.cco_event_log_finish(h) == N.OK
        assert L.cco_event_log_finish(h) == N.E_INVALID_ARG
        assert L.cco_event_log_append(h, GOOD, len(GOOD)) == N.E_INVALID_ARG
    finally:
        L.cco_event_log_free(h)


def test_directory_of_parts_generator_and_paths_give_the_body_of_the_concatenation(ctx, tmp_path):
    data = random_export(3)   # '\r\n' lines, no final newline
    lines = data.split(b"\r\n")
    d = tmp_path / "export"
    d.mkdir()
    bounds = [0, 100, 101, 400, len(lines)]
    for k, (a, b) in enumerate(zip(bounds, bounds[1:])):
        (d / ("part-%05d" % k)).write_bytes(b"\r\n".join(lines[a:b]))   # no part ends in '\n'
    (d / "part-00009").write_bytes(b"")
    (d / "_SUCCESS").write_bytes(b"")
    (d / ".part-00000.crc").write_bytes(b"junk")
    joined = E.join_parts(E.export_parts(d))
    want = ur.calc_all_from_events(joined, AP, 0, now_ms=NOW, ctx=ctx)
    assert want == ur.calc_all_from_events(data, AP, 0, now_ms=NOW, ctx=ctx)
    assert ur.calc_all_from_events(str(d), AP, 0, now_ms=NOW, ctx=ctx) == want
    with ctx.read_events(d, chunk_bytes=2048) as log:
        assert ur.calc_all_from_events(log, AP, 0, now_ms=NOW, ctx=ctx) == want
    assert ur.calc_all_from_events(E.export_parts(d), AP, 0, now_ms=NOW, ctx=ctx) == want
    gen = (joined[k:k + 777] for k in range(0, len(joined), 777))
    assert ur.calc_all_from_events(gen, AP, 0, now_ms=NOW, ctx=ctx) == want
    f = tmp_path / "export.json"
    f.write_bytes(data)
    with ctx.read_events(str(f), chunk_bytes=1000) as log:
        assert state(ctx, log) == whole(ctx, data)


def test_a_parse_error_names_the_part_and_its_line(ctx, tmp_path):
    d = tmp_path / "export"
    d.mkdir()
    (d / "part-00000").write_bytes(b"\n".join([GOOD] * 5))
    (d / "part-00001").write_bytes(b"\n".join([GOOD] * 3 + [b"[1]"] + [GOOD] * 2) + b"\n")
    for chunk in (100, 1 << 20):
        with pytest.raises(N.CcoInvalidArgument, match=r"line 8:.*part-00001, line 3\)"):
            ctx.read_events(str(d), chunk_bytes=chunk)
