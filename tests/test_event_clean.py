"""Clean write-back off the GPU: the host statement events.clean_export against the independent restatement clean_ref,
byte for byte, and its contract -- reading the compacted export under any later window gives what reading the original
export under that window gives -- on random exports at every cutoff step, with and without removeDuplicates and
compressProperties, plus directed cases of the fold."""
import json

import pytest

from clean_ref import clean_ref
from test_event_window import DAY, NOW, random_export
from test_events_mirror import iso_ms
from universal_recommender_b200 import events as E

WINDOWS = [None, E.EventWindow("5 days"), E.EventWindow(None, True), E.EventWindow("5 days", True)]


def view(d: E.DataSourceEvents, compress: bool):
    """what the contract compares of a read"""
    rank = {n: v for n, v in d.ranking_events.items() if v}
    props = {item: {f: v.text for f, v in fields.items()} for item, fields in d.set_events}
    out = [d.events, rank, props]
    if not compress:
        out += [d.n_ignored, [item for item, _ in d.set_events]]
    return out


def later(window, now):
    """w' = window's removeDuplicates with cutoffs at and after window's: every eventTime step of the random exports past
    the cutoff (a cutoff moves what expires only when it passes an eventTime), and past all of them"""
    dedup = window is not None and window.removeDuplicates
    if window is None or window.duration is None:
        yield None if not dedup else E.EventWindow(None, True), now
        base = NOW - 9 * DAY - 1
    else:
        base = window.cutoff_ms(now)
    steps = sorted({base, base + 1, NOW - 5 * DAY - 1, NOW - 5 * DAY, NOW - 5 * DAY + 1, NOW - 2 * DAY, NOW - DAY, NOW, NOW + 1})
    for c in steps:
        if c >= base:
            yield E.EventWindow("1 day", dedup), c + DAY


def check_contract(data: bytes, window, now, compress: bool):
    out = E.clean_export(data, window, now, compress)
    for w2, now2 in later(window, now):
        assert view(E.read_export(out, w2, now2), compress) == view(E.read_export(data, w2, now2), compress), (w2, now2)
    return out


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("window", WINDOWS, ids=["none", "duration", "dedup", "both"])
@pytest.mark.parametrize("compress", [False, True], ids=["plain", "compress"])
def test_mirror_against_ref_and_contract(seed, window, compress):
    data = random_export(seed, 400)
    out = check_contract(data, window, NOW, compress)
    assert out == clean_ref(data, window, NOW, compress)
    if not compress:   # the kept lines, verbatim, in order
        kept, _, _ = E.clean_events([E.parse_line(i, r) for i, r in enumerate(E.export_lines(data))], window, NOW)
        assert out == b"".join(E.export_lines(data)[e.line] + b"\n" for e in kept)


def test_compressed_export_is_a_fixed_point():
    """cleaning the compacted export again under the same window changes nothing"""
    for seed in range(3):
        w = E.EventWindow("5 days", True)
        once = E.clean_export(random_export(seed, 400), w, NOW, True)
        assert E.clean_export(once, w, NOW, True) == once


def line(**kv) -> bytes:
    return json.dumps(kv).encode()


def export(*lines: bytes) -> bytes:
    return b"\n".join(lines) + b"\n"


def t(days_ago: float) -> str:
    return iso_ms(NOW - int(days_ago * DAY))


def test_last_line_without_newline_gets_one():
    data = line(event="view", entityType="user", entityId="u", targetEntityType="item", targetEntityId="i", eventTime=t(1))
    assert E.clean_export(data, None, NOW) == data + b"\n"
    assert E.clean_export(data + b"\r\n", None, NOW) == data + b"\r\n"


def test_delete_between_sets_is_not_folded_and_can_expire_later():
    data = export(line(event="$set", entityType="item", entityId="a", properties={"x": 1}, eventTime=t(4)),
                  line(event="$delete", entityType="item", entityId="a", eventTime=t(3)),
                  line(event="$set", entityType="item", entityId="a", properties={"y": 2}, eventTime=t(2)),
                  line(event="$set", entityType="item", entityId="b", properties={"x": 1}, eventTime=t(2)),
                  line(event="$set", entityType="item", entityId="b", properties={"x": 3}, eventTime=t(1)))
    w = E.EventWindow("5 days")
    out = check_contract(data, w, NOW, True)
    lines = E.export_lines(out)
    assert lines[:3] == E.export_lines(data)[:3]   # entity a: verbatim in place
    assert lines[3] == b'{"event":"$set","entityType":"item","entityId":"b","properties":{"x":3},"eventTime":"%s"}' % t(1).encode()
    # a cutoff 3.5 days ago expires the $delete: the first $set counts again, in the read of either export
    w2, now2 = E.EventWindow("1 day"), NOW + int(2.5 * DAY)
    props = lambda d: {i: {k: v.text for k, v in f.items()} for i, f in E.read_export(d, w2, now2).set_events}
    assert props(out) == props(data) and props(out)["a"] == {"x": "1", "y": "2"}


def test_unset_before_set_only_unset_and_empty():
    data = export(line(event="$unset", entityType="item", entityId="a", properties={"x": None}, eventTime=t(4)),
                  line(event="$set", entityType="item", entityId="a", properties={"x": 1, "y": 2}, eventTime=t(3)),
                  line(event="$unset", entityType="item", entityId="b", properties={"x": None}, eventTime=t(4)),
                  line(event="$unset", entityType="item", entityId="b", properties={"y": 1, "x": 0}, eventTime=t(3)),
                  line(event="$set", entityType="item", entityId="c", properties={"x": 1}, eventTime=t(4)),
                  line(event="$unset", entityType="item", entityId="c", properties={"x": None}, eventTime=t(3)),
                  line(event="$set", entityType="item", entityId="d", properties={"x": 1, "y": 2}, eventTime=t(4)),
                  line(event="$unset", entityType="item", entityId="d", properties={"x": None}, eventTime=t(3)),
                  line(event="$set", entityType="item", entityId="d", properties={"x": 5}, eventTime=t(2)))
    out = check_contract(data, None, NOW, True)
    assert out == clean_ref(data, None, NOW, True)
    got = E.export_lines(out)
    assert got[0] == b'{"event":"$set","entityType":"item","entityId":"a","properties":{"x":1,"y":2},"eventTime":"%s"}' % t(3).encode()
    assert got[1] == b'{"event":"$unset","entityType":"item","entityId":"b","properties":{"x":0,"y":1},"eventTime":"%s"}' % t(3).encode()
    assert got[2] == b'{"event":"$set","entityType":"item","entityId":"c","properties":{},"eventTime":"%s"}' % t(3).encode()
    # an unset name set again moves to the end
    assert got[3] == b'{"event":"$set","entityType":"item","entityId":"d","properties":{"y":2,"x":5},"eventTime":"%s"}' % t(2).encode()


def test_users_targets_duplicates_and_repeated_names():
    rep = line(event="$set", entityType="item", entityId="r", properties={"a": 1}, eventTime=t(2)).replace(
        b'"properties": {', b'"properties": {"a": "old", "b": 7, ', 1)
    data = export(line(event="$set", entityType="user", entityId="u", properties={"age": 3}, eventTime=t(3)),
                  line(event="$set", entityType="user", entityId="u", properties={"city": "x"}, eventTime=t(2)),
                  line(event="$set", entityType="item", entityId="i", targetEntityType="item", targetEntityId="j",
                       properties={"a": 1}, eventTime=t(3)),
                  line(event="$set", entityType="item", entityId="i", properties={"a": 2}, eventTime=t(2)),
                  line(event="$set", entityType="item", entityId="i", properties={"b": 2}, eventTime=t(4)),
                  line(event="$set", entityType="item", entityId="k", properties={"a": 1}, eventTime=t(2)),
                  line(event="$set", entityType="item", entityId="k", properties={"a": 1}, eventTime=t(1)),
                  line(event="$set", entityType="item", entityId="r", properties={"c": 1}, eventTime=t(3)),
                  rep)
    for w in (None, E.EventWindow(None, True)):
        out = check_contract(data, w, NOW, True)
        assert out == clean_ref(data, w, NOW, True)
        got = E.export_lines(out)
        # a user's $set lines stay verbatim, and item i has a targeted $set: none of its lines is folded
        assert got[:5] == E.export_lines(data)[:5]
        assert b'"entityId":"r","properties":{"c":1,"a":1,"b":7}' in out
    # removeDuplicates leaves one of k's equal $sets, which then stays verbatim
    assert E.export_lines(E.clean_export(data, E.EventWindow(None, True), NOW, True)).count(E.export_lines(data)[6]) == 1


def test_escaped_non_ascii_and_long_ids():
    long_id = "é" * 750   # 1 500 bytes of UTF-8
    ent = long_id + "\" \x85"   # through json4s' quote: \"   \u0085
    data = export(line(event="$set", entityType="item", entityId=ent, properties={"näme\n": 1, " ": "ÿ", " ": 2}, eventTime=t(3)),
                  line(event="$set", entityType="item", entityId=ent, properties={"q": [1, {"z": None}]}, eventTime=t(2)),
                  line(event="$set", entityType="it\"em", entityId=long_id, properties={"x": 1}, eventTime=t(3)),
                  line(event="$set", entityType="it\"em", entityId=long_id, properties={"x": 2}, eventTime=t(2)),
                  line(event="$set", entityType="item", entityId="i" * 1500, properties={"a": 1}, eventTime=t(3)),
                  line(event="$unset", entityType="item", entityId="i" * 1500, properties={"a": None}, eventTime=t(2)))
    out = check_contract(data, E.EventWindow("5 days"), NOW, True)
    assert out == clean_ref(data, E.EventWindow("5 days"), NOW, True)
    lines = E.export_lines(out)
    assert lines[:2] == E.export_lines(data)[2:4]   # not an item: verbatim
    o = json.loads(lines[2])
    assert o["entityId"] == ent and list(o["properties"]) == ["näme\n", " ", " ", "q"]
    assert b'\\u2028\\u0085"' in lines[2] and b'"\\u2003":2' in lines[2]

def test_window_without_now_raises():
    with pytest.raises(ValueError):
        E.clean_export(b"", E.EventWindow("1 day"), None)
