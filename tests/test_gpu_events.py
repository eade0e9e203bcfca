"""cco_event_log_* on the H100: an event export parsed on the device gives what the host mirror (events.py) gives, through
ingest, calcAll and calcPop, byte for byte."""
import json
import random

import numpy as np
import pytest

import universal_recommender_b200 as ur
from conftest import load_golden
from test_events_mirror import export_of, iso_ms
from test_model_docs import CONFIGS, MODEL_FIXTURES
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E

pytestmark = pytest.mark.gpu


def ap_of(fx, config, recs_model="all"):
    return ur.URAlgorithmParams.from_engine_json({"eventNames": fx["event_names"], "indicators": fx["indicators"], "seed": 1,
                                                  "rankings": fx["rankings"][config], "recsModel": recs_model})


@pytest.mark.parametrize("recs_model", ["all", "collabFiltering"])
@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_calc_all_and_calc_pop_from_the_export_of_a_fixture(ctx, name, config, recs_model):
    fx = load_golden(name)
    data = export_of(fx)
    m = E.read_export(data)
    ap = ap_of(fx, config, recs_model)
    kw = dict(now_ms=fx["now_ms"], ctx=ctx)
    want = ur.calc_all_on_device(m.events, m.set_events, ap, fx["min_events_per_user"], ranking_events=m.ranking_events, **kw)
    got = ur.calc_all_from_events(data, ap, fx["min_events_per_user"], **kw)
    assert got == want
    if recs_model == "all":
        pop_want = ur.calc_pop_on_device(want, m.events, m.set_events, ap, ranking_events=m.ranking_events, **kw)
        pop = ur.calc_pop_from_events(want, data, ap, **kw)
        assert pop == pop_want
        assert ur.calc_pop_from_events(pop, data, ap, **kw) == pop   # the fixed point


def test_info_of_an_export(ctx):
    rows = [{"event": "buy", "entityType": "user", "entityId": "u1", "targetEntityType": "item", "targetEntityId": "i1", "eventTime": "2020-01-01T00:00:00Z"},
            {"event": "view", "entityType": "user", "entityId": "u2", "eventTime": "2020-01-01T00:00:03Z"},
            {"event": "$set", "entityType": "item", "entityId": "i1", "properties": {"c": 1}, "eventTime": "2020-01-01T00:00:04Z"},
            {"event": "buy", "entityType": "shop", "entityId": "s", "targetEntityType": "item", "targetEntityId": "i2", "eventTime": "2020-01-01T00:00:05Z"}]
    data = b"\n".join(json.dumps(r).encode() for r in rows)
    with ctx.read_events(data) as log:
        info = log.info()
        assert (info.n_lines, info.names, info.n_training, info.n_ranking) == (4, ["buy", "view", "$set"], [1, 0, 0], [2, 0, 0])
        assert (info.n_property_events, info.n_property_items, info.n_property_fields, info.n_ignored) == (1, 1, 1, 1)


def ingest_both(ctx, m, names, min_events):
    by = {n: [(u, i) for u, e, i, _ in m.events if e == n] for n in names}
    cols = [(*ur.encode_ids([u for u, _ in by[n]]), *ur.encode_ids([i for _, i in by[n]])) for n in names]
    a = ctx.ingest_strings(cols, min_events)
    return a


@pytest.mark.parametrize("min_events", [0, 2])
def test_log_ingest_equals_string_ingest(ctx, tmp_path, min_events):
    rng = random.Random(3)
    rows = []
    for k in range(3000):
        n = rng.choice(["buy", "view", "like"])
        u = f"u{rng.randint(0, 300)}" if n != "like" else f"w{rng.randint(0, 50)}"   # "like" users are not buyers
        rows.append({"event": n, "entityType": "user", "entityId": u, "targetEntityType": "item",
                     "targetEntityId": f"i{rng.randint(0, 400)}", "eventTime": iso_ms(1_600_000_000_000 + k)})
    data = b"".join(json.dumps(r).encode() + b"\n" for r in rows)
    path = tmp_path / "export.json"
    path.write_bytes(data)
    m = E.read_export(data)
    names = ["buy", "view", "nothing", "like"]
    (ds_a, users_a, items_a) = ingest_both(ctx, m, names, min_events)
    with ctx.read_events(str(path)) as log:
        ds_b, users_b, items_b = ctx.ingest_event_log(log, names, min_events)
    try:
        assert users_a == users_b and items_a == items_b
        for t in range(len(names)):
            a, b = ctx.dataset_to_host(ds_a, t), ctx.dataset_to_host(ds_b, t)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        ctx.free_dataset(ds_a)
        ctx.free_dataset(ds_b)


def esc(s: str, rng) -> str:
    """a JSON string literal with some characters written as \\u escapes (surrogate pairs for astral ones)"""
    out = []
    for ch in s:
        cp = ord(ch)
        if rng.random() < 0.3 or ch in '"\\':
            if cp >= 0x10000:
                v = cp - 0x10000
                out.append("\\u%04x\\u%04x" % (0xD800 + (v >> 10), 0xDC00 + (v & 0x3FF)))
            else:
                out.append("\\u%04X" % cp)
        else:
            out.append(ch)
    return '"' + "".join(out) + '"'


def random_export(seed: int) -> bytes:
    rng = random.Random(seed)
    ids = ["u" + str(k) for k in range(40)] + ["ü" + str(k) for k in range(10)] + ["😀" + str(k) for k in range(5)] + ['q"\\' + str(k) for k in range(3)]
    items = ["i" + str(k) for k in range(60)] + ["é" + str(k) for k in range(10)] + ["𝄞" + str(k) for k in range(5)]
    offsets = ["Z", "+05:30", "-0800", "+01", "-00:00"]
    lines = []
    for k in range(1500):
        kind = rng.random()
        t = rng.randint(-10 ** 11, 2 * 10 ** 12)
        if kind < 0.1:
            t = rng.choice([0, -1, 1000])   # ties and pre-1970
        off = rng.choice(offsets)
        sign = -1 if off[0] == "-" else 1
        mins = 0 if off == "Z" else (int(off[1:3]) * 60 + (int(off.lstrip("+-")[2:].lstrip(":") or 0))) * sign
        local = t + mins * 60_000
        txt = iso_ms(local)[:-1]
        frac = rng.choice(["", "." + txt[-3:], "." + txt[-3:] + "999"])
        when = txt[:-4] + frac + off
        if not frac and txt[-3:] != "000":   # no fraction: the time has whole seconds
            continue
        m = {}
        if kind < 0.7:
            m = {"event": rng.choice(["buy", "view", "like"]), "entityType": rng.choice(["user"] * 8 + ["shop"]),
                 "entityId": rng.choice(ids), "targetEntityType": rng.choice(["item"] * 8 + ["brand"]), "targetEntityId": rng.choice(items)}
        elif kind < 0.9:
            m = {"event": rng.choice(["$set", "$set", "$unset", "$delete"]), "entityType": rng.choice(["item"] * 5 + ["user"]),
                 "entityId": rng.choice(items), "properties": {rng.choice(["cat", "color", "size"]): rng.choice([1, "x", [1, 2], None, 2.5])}}
        else:
            m = {"event": "rate", "entityType": "user", "entityId": rng.choice(ids), "targetEntityType": None, "targetEntityId": None}
        m["eventTime"] = when
        mem = [(json.dumps(k_), esc(v, rng) if isinstance(v, str) else json.dumps(v)) for k_, v in m.items()]
        mem += [('"eventId"', '"%d"' % k), ('"creationTime"', '"x"'), ('"tags"', '[1,{"a":"}"}]')]
        rng.shuffle(mem)
        ws = lambda: rng.choice(["", " ", "\t", "  "])
        lines.append("{" + ws() + ",".join(f"{ws()}{a}{ws()}:{ws()}{b}{ws()}" for a, b in mem) + "}")
    return ("\r\n".join(lines)).encode()   # no final newline


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_exports_match_the_mirror(ctx, seed):
    data = random_export(seed)
    m = E.read_export(data)
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy", "view", "like"], "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": ["buy", "view"], "duration": 10 ** 9},
        {"name": "uniqueRank", "type": "random", "duration": 10 ** 9}]})
    now = 2 * 10 ** 12
    want = ur.calc_all_on_device(m.events, m.set_events, ap, 0, now_ms=now, ctx=ctx, ranking_events=m.ranking_events)
    assert ur.calc_all_from_events(data, ap, 0, now_ms=now, ctx=ctx) == want
    with ctx.read_events(data) as log:
        info = log.info()
        assert info.names == m.names and info.n_ignored == m.n_ignored
        assert info.n_ranking == [len(m.ranking_events[n]) for n in m.names]
        assert info.n_property_items == len(m.set_events)
        assert info.n_property_fields == len({f for _, d in m.set_events for f in d})


def test_property_values_are_spliced_as_written_and_a_fieldless_item_keeps_a_document(ctx):
    rows = [b'{"event":"buy","entityType":"user","entityId":"u%d","targetEntityType":"item","targetEntityId":"i%d",'
            b'"eventTime":"2020-01-01T00:00:0%dZ"}' % (u, i, u) for u in range(3) for i in range(3)]
    rows += [b'{"event":"$set","entityType":"item","entityId":"i0","eventTime":"2020-01-01T00:00:00Z",'
             b'"properties":{"a" : 1e3,"b":7.50, "popRank":"3","c":[1, 2]}}',
             b'{"event":"$set","entityType":"item","entityId":"x","eventTime":"2020-01-01T00:00:00Z","properties":{"a":-0.0}}',
             b'{"event":"$unset","entityType":"item","entityId":"x","eventTime":"2020-01-01T00:00:00Z","properties":{"a":null}}',
             b'{"event":"$delete","entityType":"item","entityId":"y","eventTime":"2020-01-01T00:00:01Z"}',
             b'{"event":"$set","entityType":"item","entityId":"y","eventTime":"2020-01-01T00:00:00Z","properties":{"a":5}}']
    data = b"\n".join(rows) + b"\n"
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy"], "seed": 1, "rankings": [
        {"name": "uniqueRank", "type": "random", "duration": 10 ** 6}]})
    now = 1_577_836_900_000
    body = ur.calc_all_from_events(data, ap, 0, now_ms=now, ctx=ctx)
    docs = [json.loads(x) for x in body.decode().splitlines()[1::2]]
    i0 = body.decode().splitlines()[1::2][0]
    assert '"a":1e3,"b":7.50,"popRank":"3","c":[1, 2]' in i0
    x = [d for d in docs if d["id"] == "x"]
    assert len(x) == 1 and set(x[0]) == {"id", "uniqueRank"}   # no field left, still a document and a random-rank candidate
    assert not [d for d in docs if d["id"] == "y"]            # deleted after its $set
    m = E.read_export(data)
    assert body == ur.calc_all_on_device(m.events, m.set_events, ap, 0, now_ms=now, ctx=ctx, ranking_events=m.ranking_events)


GOOD = b'{"event":"v","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z"}'


@pytest.mark.parametrize("bad", [
    b'{"event":"buy","entityType":"user","entityId":"","targetEntityType":"item","targetEntityId":"i","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","targetEntityType":"item","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","eventTime":"2020-01-01"}',
    b'{"event":"buy","entityType":"user","entityId":5,"eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z","properties":[]}',
    b'{"event":"buy","entityType":"user","eventTime":"2020-01-01T00:00:00Z"}',
    b'[1]', b'', b'{"event":"buy"', b'{"event":"b\\x"}',
    b'{"event":"$set","entityType":"item","entityId":"i","eventTime":"2020-01-01T00:00:00Z","properties":{"a" 1}}',
])
def test_bad_lines_are_invalid_arguments_naming_the_line(ctx, bad):
    with pytest.raises(N.CcoInvalidArgument, match="line 2"):
        ctx.read_events(GOOD + b"\n" + GOOD + b"\n" + bad + b"\n" + GOOD)
    with pytest.raises(ValueError, match="line 2"):
        E.read_export(GOOD + b"\n" + GOOD + b"\n" + bad + b"\n" + GOOD)


def test_group_context_is_refused():
    g = ur.CcoContext(devices=[0])
    try:
        with pytest.raises(N.CcoError) as e:
            g.read_events(GOOD)
        assert e.value.status == N.E_UNSUPPORTED
    finally:
        g.close()
