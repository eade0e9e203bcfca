"""The host mirror of the DataSource over a PredictionIO event export (universal_recommender_b200/events.py): time parser,
selection, property aggregation, and a round trip through the model fixtures rendered as exports."""
import datetime
import json
import random

import pytest

from conftest import load_golden
from test_model_docs import MODEL_FIXTURES
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200.ur_model import RawJson

UTC = datetime.timezone.utc
EPOCH = datetime.datetime(1970, 1, 1, tzinfo=UTC)


def iso_ms(t_ms: int) -> str:
    dt = EPOCH + datetime.timedelta(milliseconds=t_ms)
    return dt.strftime("%Y-%m-%dT%H:%M:%S.") + "%03dZ" % (dt.microsecond // 1000)


def export_of(fx) -> bytes:
    """a model fixture as `pio export` lines: its events, then its `$set` events"""
    out = []
    for u, e, i, t in fx["events"]:
        out.append({"eventId": "x", "event": e, "entityType": "user", "entityId": u, "targetEntityType": "item",
                    "targetEntityId": i, "properties": {}, "eventTime": iso_ms(t), "creationTime": iso_ms(t)})
    for item, props, t in fx["set_events"]:
        out.append({"event": "$set", "entityType": "item", "entityId": item, "properties": props, "eventTime": iso_ms(t)})
    return b"".join(json.dumps(o).encode() + b"\n" for o in out)


def test_time_parser_agrees_with_datetime():
    rng = random.Random(7)
    special = [datetime.datetime(y, m, d, tzinfo=UTC) for y, m, d in
               [(1, 1, 1), (1969, 12, 31), (1970, 1, 1), (9999, 12, 31), (2000, 2, 29), (1600, 2, 29), (2024, 2, 29)]]
    for k in range(100_000):
        if k < len(special):
            dt = special[k]
        else:
            y = rng.choice([1, 1969, 1970, 9999, rng.randint(1, 9999)])
            m = rng.randint(1, 12)
            leap = y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)
            dmax = [31, 29 if leap else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31][m - 1]
            dt = datetime.datetime(y, m, rng.choice([1, dmax, rng.randint(1, dmax)]), rng.randint(0, 23), rng.randint(0, 59),
                                   rng.randint(0, 59), rng.randint(0, 999999))
        nd = rng.randint(0, 9)
        digits = "%06d" % dt.microsecond + "".join(rng.choice("0123456789") for _ in range(3))
        frac = "." + digits[:nd] if nd else ""
        oh, om = rng.randint(0, 23), rng.choice([0, 30, 45, rng.randint(0, 59)])
        sign = rng.choice("+-")
        form = rng.randint(0, 3)
        off = [("Z", 0), (f"{sign}{oh:02d}:{om:02d}", 1), (f"{sign}{oh:02d}{om:02d}", 1), (f"{sign}{oh:02d}", 2)][form]
        minutes = 0 if form == 0 else (oh * 60 + (om if form != 3 else 0)) * (-1 if sign == "-" else 1)
        text = dt.strftime("%Y-%m-%dT%H:%M:%S").rjust(19, "0") if dt.year >= 1000 else "%04d" % dt.year + dt.strftime("-%m-%dT%H:%M:%S")
        text += frac + off[0]
        us = int(digits[:nd].ljust(6, "0")[:6]) if nd else 0
        local = dt.replace(microsecond=us, tzinfo=datetime.timezone(datetime.timedelta(minutes=minutes)))
        want = (local - EPOCH) // datetime.timedelta(milliseconds=1)
        assert E.parse_event_time(text) == want, text


@pytest.mark.parametrize("text", ["2017-05-01T12:34:56", "2017-05-01 12:34:56Z", "2017-5-01T12:34:56Z", "2017-02-29T00:00:00Z",
                                  "2017-05-01T24:00:00Z", "2017-05-01T12:60:00Z", "2017-05-01T12:34:60Z", "2017-05-01T12:34:56.Z",
                                  "2017-05-01T12:34:56.1234567890Z", "2017-05-01T12:34:56+24:00", "2017-05-01T12:34:56+05:3",
                                  "2017-05-01T12:34:56+5", "2017-05-01T12:34:56z", "2017-05-01T12:34:56Z ", "+2017-05-01T12:34:56Z",
                                  "２017-05-01T12:34:56Z", "2017-13-01T00:00:00Z", "2017-00-10T00:00:00Z", "1900-02-29T00:00:00Z"])
def test_time_parser_rejects(text):
    with pytest.raises(ValueError):
        E.parse_event_time(text)


def ev(i, name, item, t, props=None, etype="item"):
    return E.Event(i, name, etype, item, None, None, t, props or {})


def test_aggregation_with_equal_times_and_an_item_without_fields():
    seq = [ev(0, "$set", "a", 5, {"x": 1, "y": 2}), ev(1, "$unset", "a", 5, {"x": None}), ev(2, "$set", "b", 1, {"z": 3}),
           ev(3, "$delete", "b", 5), ev(4, "$set", "b", 5, {"w": 4}), ev(5, "$set", "c", 2, {"q": 1}), ev(6, "$unset", "c", 3, {"q": 0}),
           ev(7, "$delete", "d", 1), ev(8, "$unset", "e", 1, {"k": 1}), ev(9, "$set", "a", 4, {"x": 9, "v": 0}),
           ev(10, "$delete", "f", 9), ev(11, "$set", "f", 9, {"f": 1})]
    got = E.aggregate_property_events(seq)
    # (time, line) order: b@1 set, d@1 delete, e@1 unset, c@2, c@3, a@4 (x, v), a@5 set (x, y merged), a@5 unset x, b@5 delete,
    # b@5 set w, f@9 delete then set
    # items in order of their first property event (line order), fields in order of first appearance among the members
    assert [(i, list(d.items())) for i, d in got] == [("a", [("y", 2), ("v", 0)]), ("b", [("w", 4)]), ("c", []), ("f", [("f", 1)])]
    # an item ending with no field keeps a state (the reference's fieldsRDD lists it)
    assert ("c", {}) in got


def line(obj) -> bytes:
    return json.dumps(obj).encode()


def test_selection_rules():
    rows = [
        {"event": "buy", "entityType": "user", "entityId": "u1", "targetEntityType": "item", "targetEntityId": "i1", "eventTime": "2020-01-01T00:00:00Z"},
        {"event": "buy", "entityType": "shop", "entityId": "s1", "targetEntityType": "item", "targetEntityId": "i2", "eventTime": "2020-01-01T00:00:01Z"},
        {"event": "buy", "entityType": "user", "entityId": "u1", "targetEntityType": "brand", "targetEntityId": "b1", "eventTime": "2020-01-01T00:00:02Z"},
        {"event": "view", "entityType": "user", "entityId": "u2", "eventTime": "2020-01-01T00:00:03Z"},
        {"event": "$set", "entityType": "item", "entityId": "i1", "properties": {"c": ["x"]}, "eventTime": "2020-01-01T00:00:04Z"},
        {"event": "$set", "entityType": "user", "entityId": "u1", "properties": {"c": ["x"]}, "eventTime": "2020-01-01T00:00:05Z"},
    ]
    data = b"\r\n".join(line(r) for r in rows)   # '\r' is whitespace, no final newline
    got = E.read_export(data)
    assert got.names == ["buy", "view", "$set"]
    assert got.events == [("u1", "buy", "i1", 1577836800000)]
    assert got.ranking_events == {"buy": [("i1", 1577836800000), ("i2", 1577836801000), ("b1", 1577836802000)], "view": [], "$set": []}
    assert got.set_events == [("i1", {"c": RawJson('["x"]')})]
    assert got.n_ignored == 2


def test_repeated_members_and_nulls():
    raw = (b'{"event":"a","event":"buy","entityType":"user","entityId":"u0","entityId":"u1","targetEntityType":null,'
           b'"targetEntityId":null,"targetEntityType":"item","targetEntityId":"i\\u00e9","eventTime":"bad","eventTime":"2020-01-01T00:00:00Z"}')
    got = E.read_export(raw)
    assert got.events == [("u1", "buy", "ié", 1577836800000)]


@pytest.mark.parametrize("bad", [
    b'{"event":"buy","entityType":"user","entityId":"","targetEntityType":"item","targetEntityId":"i","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","targetEntityType":"item","targetEntityId":"","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","targetEntityType":"item","eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","eventTime":"2020-01-01"}',
    b'{"event":"buy","entityType":"user","entityId":5,"eventTime":"2020-01-01T00:00:00Z"}',
    b'{"event":"buy","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z","properties":[]}',
    b'{"event":"buy","entityType":"user","eventTime":"2020-01-01T00:00:00Z"}',
    b'[1]', b'', b'{"event":"buy"',
])
def test_bad_lines_raise_and_name_the_line(bad):
    good = b'{"event":"v","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z"}'
    with pytest.raises(ValueError, match="line 1"):
        E.read_export(good + b"\n" + bad + b"\n" + good + b"\n")


@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_round_trip_of_the_model_fixtures(name):
    fx = load_golden(name)
    got = E.read_export(export_of(fx))
    assert got.events == [tuple(e) for e in fx["events"]]
    assert got.names == list(dict.fromkeys([e[1] for e in fx["events"]] + (["$set"] if fx["set_events"] else [])))
    want = um.aggregate_properties([(s[0], s[1]) for s in sorted(fx["set_events"], key=lambda s: s[2])])
    assert [(i, f, json.loads(v.text)) for i, f, v in um.aggregate_properties(got.set_events)] == want


def test_property_values_keep_their_text():
    raw = (b'{"event":"$set","entityType":"item","entityId":"i","eventTime":"2020-01-01T00:00:00Z",'
           b'"properties":{ "a" : 1e3 , "b":7.50,"popRank":"3","c":[1, 2],"a":1E3}}')
    got = E.read_export(raw)
    assert got.set_events == [("i", {"a": RawJson("1E3"), "b": RawJson("7.50"), "popRank": RawJson('"3"'), "c": RawJson("[1, 2]")})]
    assert um.property_json(got.set_events[0][1]["b"]) == "7.50"


def test_line_numbers_of_property_events_are_file_lines():
    good = b'{"event":"v","entityType":"user","entityId":"u","eventTime":"2020-01-01T00:00:00Z"}'
    prop = b'{"event":"$set","entityType":"item","entityId":"i","eventTime":"2020-01-01T00:00:00Z","properties":{"a":1}}'
    got = E.read_export(good + b"\n" + good + b"\n" + prop)
    assert [e.line for e in got.property_events] == [2]
