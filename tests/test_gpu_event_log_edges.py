"""cco_event_log_read at its edges on the H100: every parsed eventTime observed exactly through the rankings, accept/reject
agreement with the mirror, backslash runs and escaped member names in the tokenizer, line framing, property aggregation
with ties at scale, and the host/device differences the events.py docstring lists."""
import json
import random

import numpy as np
import pytest

import universal_recommender_b200 as ur
from test_event_log_edges import (ACCEPT_LITERALS, REJECT_LITERALS, decode_literal, mirror_time, ref_time, time_mutants,
                                  time_spellings)
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E
from universal_recommender_b200.ur_model import RawJson

pytestmark = pytest.mark.gpu

GOOD = b'{"event":"v","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z"}'
T0 = b'"eventTime":"2020-01-01T00:00:00Z"'


def docs_of(body: bytes) -> list:
    return [json.loads(x) for x in body.decode("utf-8", "surrogateescape").splitlines()[1::2]]


def raw_ids(ids) -> list:
    """dictionary strings (decoded with surrogateescape) back to their bytes"""
    return [x.encode("utf-8", "surrogateescape") for x in ids]


def ingest_matches(ctx, log, m: E.DataSourceEvents, min_events: int = 0):
    """ingest_event_log of every name equals ingest_strings of the mirror's training events"""
    names = m.names or ["none"]
    by = {n: [(u, i) for u, e, i, _ in m.events if e == n] for n in names}
    cols = [(*ur.encode_ids([u for u, _ in by[n]]), *ur.encode_ids([i for _, i in by[n]])) for n in names]
    ds_a, users_a, items_a = ctx.ingest_strings(cols, min_events)
    ds_b, users_b, items_b = ctx.ingest_event_log(log, names, min_events)
    try:
        assert users_a == users_b and items_a == items_b
        for t in range(len(names)):
            a, b = ctx.dataset_to_host(ds_a, t), ctx.dataset_to_host(ds_b, t)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        ctx.free_dataset(ds_a)
        ctx.free_dataset(ds_b)


def info_matches(info, m: E.DataSourceEvents, n_lines: int):
    assert info.n_lines == n_lines and info.names == m.names and info.n_ignored == m.n_ignored
    assert info.n_training == [sum(1 for _, e, _, _ in m.events if e == n) for n in m.names]
    assert info.n_ranking == [len(m.ranking_events[n]) for n in m.names]
    assert info.n_property_events == len(m.property_events)
    assert info.n_property_items == len(m.set_events)
    assert info.n_property_fields == len({f for _, d in m.set_events for f in d})


def assert_matches_mirror(ctx, data: bytes):
    m = E.read_export(data)
    with ctx.read_events(data) as log:
        info_matches(log.info(), m, len(E.export_lines(data)))
        ingest_matches(ctx, log, m)
    return m


def props_match(ctx, data: bytes) -> bytes:
    """the properties aggregated on the device, written by calcPop into an empty index, equal the mirror's"""
    m = E.read_export(data)
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": m.names or ["x"], "seed": 1, "rankings": [
        {"name": "uniqueRank", "type": "random", "duration": 10 ** 9}]})
    now = 1_600_000_000_000
    want = ur.calc_pop_on_device(b"", m.events, m.set_events, ap, now_ms=now, ctx=ctx, ranking_events=m.ranking_events)
    got = ur.calc_pop_from_events(b"", data, ap, now_ms=now, ctx=ctx)
    assert got == want
    return got


def time_line(k: int, lit: str) -> bytes:
    return ('{"event":"t","entityType":"u","entityId":"u","targetEntityType":"i","targetEntityId":"x%d","eventTime":"%s"}'
            % (k, lit)).encode("utf-8")


# ---- 1 + 2: exact times, accept / reject ---------------------------------------------------------------------------------
def test_device_times_are_exact(ctx):
    ins, sp = time_spellings()
    mut = [t for t in time_mutants() if ref_time(t) is not None]
    acc = [decode_literal(x) for x in ACCEPT_LITERALS]
    cases = [(lit, t) for _, _, lit, _, t in sp] + [(json.dumps(t)[1:-1], ref_time(t)) for t in mut] + \
            [(lit, ref_time(text)) for lit, text in zip(ACCEPT_LITERALS, acc)]
    for lit, t in cases:
        assert E.parse_event_time(decode_literal(lit)) == t   # the mirror stays honest
    items = ["x%d" % k for k in range(len(cases))]
    times = np.array([t for _, t in cases], dtype=np.int64)
    data = b"\n".join(time_line(k, lit) for k, (lit, _) in enumerate(cases)) + b"\n"
    # the windows: every instant, every accepted mutant's and extra spelling's value
    windows = list(dict.fromkeys(ins + [t for _, t in cases[len(sp):]]))
    io, ib = ur.encode_ids(items)
    stream = [(io, ib, times)]
    at = {}
    for k, t in enumerate(times.tolist()):
        at.setdefault(t, []).append(items[k])
    n_hits = 0
    with ctx.read_events(data) as log:
        assert log.info().n_ranking == [len(cases)]
        for c in range(0, len(windows), N.MAX_RANKINGS):
            w = windows[c:c + N.MAX_RANKINGS]
            got = ctx.rerank_model(b"", rankings=[(f"r{q}", "popular", m, m + 1, ["t"]) for q, m in enumerate(w)], log=log)
            want = ctx.rerank_model(b"", rankings=[(f"r{q}", "popular", m, m + 1, stream) for q, m in enumerate(w)])
            assert got == want, w
            have = {d["id"]: {k for k in d if k != "id"} for d in docs_of(got)}
            expect = {}
            for q, m in enumerate(w):
                for it in at.get(m, []):
                    expect.setdefault(it, set()).add(f"r{q}")
            assert have == expect, w
            n_hits += len(have)
    assert len(windows) >= 500 and n_hits >= 3000


def bad_time_log(lit: str) -> bytes:
    return GOOD + b"\n" + GOOD.replace(b"2020-01-01T00:00:00Z", lit.encode("utf-8")) + b"\n" + GOOD + b"\n"


@pytest.mark.parametrize("lit", REJECT_LITERALS)
def test_device_rejects_bad_times(ctx, lit):
    with pytest.raises(N.CcoInvalidArgument, match="line 1"):
        ctx.read_events(bad_time_log(lit))
    with pytest.raises(ValueError, match="line 1"):
        E.read_export(bad_time_log(lit))


def test_device_rejects_the_rejected_mutants(ctx):
    bad = [t for t in time_mutants() if mirror_time(t) is None]
    assert len(bad) > 100
    for t in bad:
        with pytest.raises(N.CcoInvalidArgument, match="line 1"):
            ctx.read_events(bad_time_log(json.dumps(t)[1:-1]))


# ---- 3: tokenizer edges ------------------------------------------------------------------------------------------------------
TAIL = b',"event":"buy","entityType":"user","targetEntityType":"item","targetEntityId":"i%d","eventTime":"2020-01-01T00:00:00Z"}'


def run_lines():
    """(shift, run, closer) for backslash runs of 0-66 escaped backslashes at every offset 0-31 from the line start"""
    return [(k, n, c) for n in range(67) for k in range(32) for c in ("", '\\"')]


def test_backslash_runs_in_ids_ignored_members_and_property_values(ctx):
    lines = []
    for j, (k, n, c) in enumerate(run_lines()):
        run = ("a" + "\\\\" * n + c + "z%d" % j).encode()
        pad = b" " * k
        # in the id
        lines.append(b"{" + pad + b'"entityId":"' + run + b'"' + TAIL % j)
        # in an ignored member ahead of the real ones: a parity slip shifts every later span
        lines.append(b"{" + pad + b'"note":"' + run + b'","entityId":"u%d"' % j + TAIL % j)
        # in a property value, spliced as written
        lines.append(b"{" + pad + b'"properties":{"p":"' + run + b'"},"event":"$set","entityType":"item","entityId":"p%d",' % j + T0 + b"}")
    data = b"\n".join(lines) + b"\n"
    m = assert_matches_mirror(ctx, data)
    assert max(u.count("\\") for u, _, _, _ in m.events) == 66
    body = props_match(ctx, data)
    for j in (0, 65, 2 * 67 * 32 - 1):
        assert b'"p":"a' + b"\\\\" * run_lines()[j][1] in body


def test_an_odd_run_before_the_closing_quote_is_rejected_on_the_same_line(ctx):
    rng = random.Random(4)
    for n in range(67):
        for k in rng.sample(range(32), 3):
            run = b"a" + b"\\" * (2 * n + 1)   # escapes the quote meant to close the string
            where = rng.randrange(3)
            bad = [b"{" + b" " * k + b'"entityId":"' + run + b'"' + TAIL % 0,
                   b"{" + b" " * k + b'"note":"' + run + b'","entityId":"u"' + TAIL % 0,
                   b"{" + b" " * k + b'"properties":{"p":"' + run + b'"},"event":"$set","entityType":"item","entityId":"p",' + T0 + b"}"][where]
            data = GOOD + b"\n" + bad + b"\n" + GOOD
            with pytest.raises(ValueError, match="line 1"):
                E.read_export(data)
            with pytest.raises(N.CcoInvalidArgument, match="line 1"):
                ctx.read_events(data)


def test_escaped_member_names(ctx):
    rows = [
        b'{"\\u0065ventTime":"2020-01-01T00:00:01Z","event":"buy","entity\\u0049d":"u1","entityType":"user","targetEntityType":"item","targetEntityId":"i1"}',
        b'{"event\\u0000":5,"eventTime ":[],"event":"buy","entityId":"u2","entityType":"user","targetEntityType":"item","targetEntityId":"i2",' + T0 + b"}",
        b'{"entityId":"first","entity\\u0049d":"second","event":"buy","entityType":"user","targetEntityType":"item","targetEntityId":"i3",' + T0 + b"}",
        b'{"entity\\u0049d":"first","entityId":"third","event":"buy","entityType":"user","targetEntityType":"item","targetEntityId":"i4",' + T0 + b"}",
        b'{"\\u0065\\u0076\\u0065\\u006e\\u0074":"buy","entityType":"\\u0075ser","entityId":"u5","targetEntityType":"item","target\\u0045ntityId":"i5",' + T0 + b"}",
        b'{"event":"$set","entityType":"item","entityId":"i1","properties":{"color":1,"size":2},' + T0 + b"}",
        b'{"event":"$set","entityType":"item","entityId":"i1","properties":{"c\\u006flor":2},"eventTime":"2020-01-01T00:00:01Z"}',
        b'{"event":"$set","entityType":"item","entityId":"i2","properties":{"c\\u006flor":3,"color":4,"\\u0063olor":5},' + T0 + b"}",
    ]
    data = b"\n".join(rows)
    m = assert_matches_mirror(ctx, data)
    assert [u for u, _, _, _ in m.events] == ["u1", "u2", "second", "third", "u5"]
    assert m.set_events == [("i1", {"color": RawJson("2"), "size": RawJson("2")}),
                            ("i2", {"color": RawJson("5")})]
    with ctx.read_events(data) as log:
        assert log.info().n_property_fields == 2
    body = props_match(ctx, data)
    assert b'"color":2,"size":2' in body and b'"color":5' in body


# ---- 4: framing ----------------------------------------------------------------------------------------------------------------
def test_empty_export(ctx):
    with ctx.read_events(b"") as log:
        info = log.info()
        assert (info.n_lines, info.names, info.n_training, info.n_ranking) == (0, [], [], [])
        assert (info.n_property_events, info.n_property_items, info.n_property_fields, info.n_ignored) == (0, 0, 0, 0)
        ds, users, items = ctx.ingest_event_log(log, ["buy", "view"])
        ctx.free_dataset(ds)
        assert users == [] and items == [[], []]
        assert ctx.rerank_model(b"", rankings=[("r", "popular", 0, 10, ["buy"])], log=log) == b""
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy"], "seed": 1})
    with pytest.raises(ValueError) as a:
        ur.calc_all_on_device([], [], ap, 0, now_ms=0, ctx=ctx, ranking_events={})
    with pytest.raises(ValueError) as b:
        ur.calc_all_from_events(b"", ap, 0, now_ms=0, ctx=ctx)
    assert str(a.value) == str(b.value)


@pytest.mark.parametrize("data,line", [(b"\n", 0), (b"\r\n", 0), (b" \n" + GOOD, 0), (GOOD + b"\n\n" + GOOD, 1), (GOOD + b"\n\r", 1),
                                       (GOOD + b"\n" + GOOD + b"\n\n", 2)])
def test_blank_lines_are_not_events(ctx, data, line):
    with pytest.raises(N.CcoInvalidArgument, match=f"line {line}"):
        ctx.read_events(data)
    with pytest.raises(ValueError, match=f"line {line}"):
        E.read_export(data)


@pytest.mark.parametrize("data", [GOOD + b"\r", GOOD + b"\r\n", b"\t" + GOOD + b"\r\n" + GOOD + b" \r"])
def test_trailing_whitespace_is_accepted(ctx, data):
    assert_matches_mirror(ctx, data)


def export_of_length(n: int, final_newline: bool, seed: int) -> bytes:
    """training lines, spaces after the last line's '{' make the export exactly n bytes"""
    rng = random.Random(seed)
    lines, size = [], 0
    while True:
        ln = (b'{"event":"%s","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"i%d",'
              b'"eventTime":"2020-01-01T00:00:%02dZ"}' % (rng.choice([b"buy", b"view"]), rng.randrange(90), rng.randrange(120), rng.randrange(60)))
        if size + len(ln) + 1 + 160 > n:
            break
        lines.append(ln)
        size += len(ln) + 1
    data = b"\n".join(lines) + (b"\n" if lines else b"")
    last = (b'{"event":"buy","entityType":"user","entityId":"z","targetEntityType":"item","targetEntityId":"z",' + T0 + b"}")
    pad = n - len(data) - len(last) - (1 if final_newline else 0)
    assert pad >= 0
    data += last[:1] + b" " * pad + last[1:] + (b"\n" if final_newline else b"")
    assert len(data) == n
    return data


LENGTHS = [8 * q + d for q in (20, 37, 101) for d in (-1, 0, 1)] + [2048 * q + d for q in (1, 2, 3, 8) for d in (-1, 0, 1)]


@pytest.mark.parametrize("final_newline", [True, False])
def test_lengths_at_word_and_chunk_edges(ctx, final_newline):
    for n in LENGTHS:
        assert_matches_mirror(ctx, export_of_length(n, final_newline, n))


def test_a_3mb_line_among_short_lines(ctx):
    rng = random.Random(8)
    big_id = "".join(rng.choice(["a", "b", "é", '\\"', "\\\\", "\\u00e9", "\\n"]) for _ in range(400_000)).encode()
    big_val = b'{"v":"' + "".join(rng.choice(["x", '\\"', "\\\\", "}", "]", "{"]) for _ in range(1_300_000)).encode() + b'"}'
    short = [b'{"event":"buy","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"i%d",' % (k, k % 7) + T0 + b"}"
             for k in range(300)]
    big = (b'{"event":"$set","entityType":"item","entityId":"' + big_id + b'","properties":{"p":' + big_val + b'},' + T0 + b"}")
    big_user = b'{"event":"buy","entityType":"user","entityId":"' + big_id + b'","targetEntityType":"item","targetEntityId":"i0",' + T0 + b"}"
    assert len(big) + len(big_user) > 3_000_000
    data = b"\n".join(short[:100] + [big] + short[100:200] + [big_user] + short[200:]) + b"\n"
    assert_matches_mirror(ctx, data)
    body = props_match(ctx, data)
    assert b'"p":' + big_val in body


def test_two_million_lines(ctx):
    n = 2_000_000
    u = (np.arange(n, dtype=np.int64) * 7919) % 65_537
    i = (np.arange(n, dtype=np.int64) * 104_729) % 50_021
    line = '{"event":"b","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"i%d","eventTime":"2020-01-01T00:00:00Z"}\n'
    data = "".join([line % (a, b) for a, b in zip(u.tolist(), i.tolist())]).encode()
    users = ["u%d" % a for a in u.tolist()]
    items = ["i%d" % b for b in i.tolist()]
    ds_a, users_a, items_a = ctx.ingest_strings([(*ur.encode_ids(users), *ur.encode_ids(items))], 0)
    with ctx.read_events(data) as log:
        info = log.info()
        assert (info.n_lines, info.names, info.n_training) == (n, ["b"], [n])
        ds_b, users_b, items_b = ctx.ingest_event_log(log, ["b"], 0)
    try:
        assert users_a == users_b and items_a == items_b
        a, b = ctx.dataset_to_host(ds_a, 0), ctx.dataset_to_host(ds_b, 0)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        ctx.free_dataset(ds_a)
        ctx.free_dataset(ds_b)


# ---- 5: property aggregation at scale ------------------------------------------------------------------------------------------
def property_export(seed: int, n: int = 20_000) -> bytes:
    rng = random.Random(seed)
    times = ["2020-01-01T00:00:0%dZ" % k for k in range(5)]
    names = ['"a"', '"b"', '"id"', '"color"', '"c\\u006flor"', '"size"', '"popRank"']
    values = ["1", '"x"', "[1, 2]", '{"k":"}"}', "null", "2.50", "-0.0", "true", '"\\u00e9\\\\"']
    lines = []
    for k in range(n):
        r = rng.random()
        item = "p%d" % rng.randrange(500)
        t = rng.choice(times)
        if r < 0.1:    # training events, so that calcAll has a model
            lines.append('{"event":"buy","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"%s","eventTime":"%s"}'
                         % (rng.randrange(80), item, t))
            continue
        kind = "$set" if r < 0.55 else "$unset" if r < 0.8 else "$delete" if r < 0.92 else "$set"
        etype = "user" if r >= 0.92 else "item"    # $set of a user: not a property event
        members = [f"{rng.choice(names)}:{rng.choice(values)}" for _ in range(rng.choice([0, 1, 1, 2, 3, 4]))]   # names repeat
        props = ',"properties":{%s}' % ",".join(members) if kind != "$delete" or rng.random() < 0.3 else ""
        lines.append('{"event":"%s","entityType":"%s","entityId":"%s","eventTime":"%s"%s}' % (kind, etype, item, t, props))
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("seed", [1, 2])
def test_property_aggregation_with_ties_at_scale(ctx, seed):
    data = property_export(seed)
    m = E.read_export(data)
    assert len(m.property_events) > 15_000 and any(not d for _, d in m.set_events) and any("id" in d for _, d in m.set_events)
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy"], "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": ["buy"], "duration": 10 ** 6},
        {"name": "uniqueRank", "type": "random", "duration": 10 ** 6}]})
    now = 1_577_836_900_000
    want = ur.calc_all_on_device(m.events, m.set_events, ap, 0, now_ms=now, ctx=ctx, ranking_events=m.ranking_events)
    assert ur.calc_all_from_events(data, ap, 0, now_ms=now, ctx=ctx) == want
    pop_want = ur.calc_pop_on_device(want, m.events, m.set_events, ap, now_ms=now, ctx=ctx, ranking_events=m.ranking_events)
    assert ur.calc_pop_from_events(want, data, ap, now_ms=now, ctx=ctx) == pop_want
    with ctx.read_events(data) as log:
        info_matches(log.info(), m, len(E.export_lines(data)))


@pytest.mark.parametrize("id_kept", [True, False])
def test_a_real_id_field_next_to_fieldless_items(ctx, id_kept):
    rows = [b'{"event":"$set","entityType":"item","entityId":"a","properties":{"id":"A","x":1},' + T0 + b"}",
            b'{"event":"$set","entityType":"item","entityId":"b","properties":{"y":1},' + T0 + b"}",
            b'{"event":"$unset","entityType":"item","entityId":"b","properties":{"y":null},"eventTime":"2020-01-01T00:00:01Z"}',
            b'{"event":"$set","entityType":"item","entityId":"c","properties":{},' + T0 + b"}"]
    if not id_kept:
        rows.append(b'{"event":"$unset","entityType":"item","entityId":"a","properties":{"id":0},"eventTime":"2020-01-01T00:00:01Z"}')
    data = b"\n".join(rows)
    m = E.read_export(data)
    with ctx.read_events(data) as log:
        info_matches(log.info(), m, len(rows))
    body = props_match(ctx, data)
    assert {d["id"] for d in docs_of(body)} == {"a", "b", "c"}


# ---- 6: host / device differences -------------------------------------------------------------------------------------------------
def test_a_byte_order_mark_is_refused_on_the_same_line(ctx):
    data = GOOD + b"\n" + b"\xef\xbb\xbf" + GOOD + b"\n" + GOOD
    with pytest.raises(N.CcoInvalidArgument, match="line 1"):
        ctx.read_events(data)
    with pytest.raises(ValueError, match="line 1"):
        E.read_export(data)


def training(uid: bytes, iid: bytes = b"i") -> bytes:
    return b'{"event":"buy","entityType":"user","entityId":"' + uid + b'","targetEntityType":"item","targetEntityId":"' + iid + b'",' + T0 + b"}"


def test_invalid_utf8_is_read_verbatim(ctx):
    bad = [b"u\xff", b"u\xc3", b"u\xed\xa0\x80", b"\xc0\xaf", b"u\xf4\x90\x80\x80"]
    data = b"\n".join(training(x) for x in bad)
    with ctx.read_events(data) as log:
        ds, users, _ = ctx.ingest_event_log(log, ["buy"])
        ctx.free_dataset(ds)
    assert sorted(raw_ids(users)) == sorted(bad)
    with pytest.raises(ValueError, match="line 0"):
        E.read_export(data)


def test_lone_surrogate_escapes_are_written_in_their_3_byte_form(ctx):
    cases = [(b"\\ud800", b"\xed\xa0\x80"), (b"\\uDC00", b"\xed\xb0\x80"), (b"\\ud800\\u0041", b"\xed\xa0\x80A"),
             (b"\\ud800\\ud800", b"\xed\xa0\x80\xed\xa0\x80"), (b"\\udc00\\ud800", b"\xed\xb0\x80\xed\xa0\x80"),
             (b"\\ud800x\\udc00", b"\xed\xa0\x80x\xed\xb0\x80"), (b"\\ud83d\\ude00", "\U0001F600".encode())]
    data = b"\n".join(training(b"u" + esc, b"i" + esc) for esc, _ in cases)
    with ctx.read_events(data) as log:
        ds, users, items = ctx.ingest_event_log(log, ["buy"])
        ctx.free_dataset(ds)
    assert sorted(raw_ids(users)) == sorted(b"u" + raw for _, raw in cases)
    assert sorted(raw_ids(items[0])) == sorted(b"i" + raw for _, raw in cases)
    m = E.read_export(data)   # the mirror reads the line, but its ids are not UTF-8 encodable
    with pytest.raises(UnicodeEncodeError):
        ur.encode_ids([u for u, _, _, _ in m.events])


def test_mismatched_bracket_kinds_in_a_nested_value_are_spliced(ctx):
    line = b'{"event":"$set","entityType":"item","entityId":"i","properties":{"p":{"a":{]},"q":[}{]},' + T0 + b"}"
    with ctx.read_events(line) as log:
        assert log.info().n_property_fields == 2
        body = ctx.rerank_model(b"", log=log)
    assert body == b'{"index":{"_id":"i"}}\n{"id":"i","p":{"a":{]},"q":[}{]}\n'
    with pytest.raises(ValueError, match="line 0"):
        E.read_export(line)
