"""The DataSource's eventWindow off the GPU: the host mirror (events.read_export(window=...)) against an independent brute
force, Scala's Duration(...).toMillis (ur_model.duration_ms), DataSourceParams from engine.json, and the C entries."""
import json
import os
import random
import subprocess

import pytest

import universal_recommender_b200 as ur
from conftest import ROOT
from test_events_mirror import iso_ms
from universal_recommender_b200 import events as E
from universal_recommender_b200.ur_model import duration_ms

NOW = 1_700_000_000_000
DAY = 86_400_000


def random_export(seed: int, n: int = 600) -> bytes:
    """events over few ids, so that many repeat; copies of earlier events with a new eventId / eventTime / creationTime,
    member order, null for absent, repeated property names; some old, some at the cutoff"""
    rng = random.Random(seed)
    rows, raw = [], []
    cut = NOW - 5 * DAY
    for k in range(n):
        if rows and rng.random() < 0.35:
            r = dict(rng.choice(rows))
            r["eventId"] = f"e{k}"
            r["creationTime"] = iso_ms(NOW - rng.randint(0, 9 * DAY))
            if rng.random() < 0.7:
                r["eventTime"] = iso_ms(rng.choice([cut, cut + 1, cut - 1, NOW - rng.randint(0, 9 * DAY)]))
            if "properties" in r and rng.random() < 0.5:
                r["properties"] = dict(reversed(list(r["properties"].items())))
            if rng.random() < 0.2 and "targetEntityId" not in r:
                r["targetEntityId"] = None
                r["targetEntityType"] = None
            if rng.random() < 0.2 and "prId" not in r:
                r["prId"] = None
            items = list(r.items())
            rng.shuffle(items)
            r = dict(items)
        else:
            name = rng.choice(["buy", "view", "$set", "$unset", "$delete", "like"])
            t = rng.choice([cut, cut + 1, cut - 1, NOW - rng.randint(0, 9 * DAY)])
            if name.startswith("$"):
                r = {"event": name, "entityType": rng.choice(["item", "item", "user"]), "entityId": f"i{rng.randint(0, 5)}"}
                if name != "$delete":
                    r["properties"] = {f: rng.choice([1, "x", [1, 2], {"a": 1}]) for f in rng.sample("abcd", rng.randint(0, 3))}
            else:
                r = {"event": name, "entityType": "user", "entityId": f"u{rng.randint(0, 6)}"}
                if name != "like":
                    r.update(targetEntityType="item", targetEntityId=f"i{rng.randint(0, 5)}")
                if rng.random() < 0.2:
                    r["prId"] = rng.choice(["p1", "p2", ""])
                if rng.random() < 0.2:
                    r["tags"] = rng.choice([[], ["a"], ["a", "b"], None])
                if rng.random() < 0.2:
                    r["properties"] = {"q": rng.randint(0, 1)}
            r["eventTime"] = iso_ms(t)
        rows.append(r)
        line = json.dumps(r)
        if "properties" in r and r["properties"] and rng.random() < 0.1:   # a repeated name: the last one wins
            f = next(iter(r["properties"]))
            line = line.replace('"properties": {', '"properties": {"%s": "old", ' % f, 1)
        raw.append(line.encode())
    return b"\n".join(raw) + b"\n"


def brute_force(data: bytes, window: E.EventWindow, now: int) -> tuple[list, int, int]:
    """kept lines, expired, duplicates: json.loads, a canonical tuple per event, a sort"""
    cutoff = None if window.duration is None else now - duration_ms(window.duration)
    evs = []
    for i, line in enumerate(data.splitlines()):
        o = json.loads(line, object_pairs_hook=dict)
        t = E.parse_event_time(o["eventTime"])
        if cutoff is not None and t <= cutoff and o["event"] not in ("$set", "$unset"):
            continue
        tags = o.get("tags")
        key = json.dumps([o["event"], o["entityType"], o["entityId"], o.get("targetEntityType"), o.get("targetEntityId"), o.get("prId"),
                          [] if tags is None else tags, sorted((k, json.dumps(v)) for k, v in (o.get("properties") or {}).items())])
        evs.append((key, t, i))
    n_lines = len(data.splitlines())
    expired = n_lines - len(evs)
    if not window.removeDuplicates:
        return sorted(i for _, _, i in evs), expired, 0
    evs.sort(key=lambda x: (x[0], -x[1], -x[2]))
    kept = [x[2] for k, x in enumerate(evs) if k == 0 or x[0] != evs[k - 1][0]]
    return sorted(kept), expired, len(evs) - len(kept)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("window", [E.EventWindow("5 days", True), E.EventWindow("5 days"), E.EventWindow(None, True),
                                    E.EventWindow("120 h", True, True)])
def test_mirror_against_brute_force(seed, window):
    data = random_export(seed)
    m = E.read_export(data, window, NOW)
    kept, expired, dups = brute_force(data, window, NOW)
    assert (m.n_expired, m.n_duplicates) == (expired, dups)
    parsed = [E.parse_line(i, raw) for i, raw in enumerate(E.export_lines(data))]
    assert [e.line for e in E.clean_events(parsed, window, NOW)[0]] == kept
    assert (dups > 0) == window.removeDuplicates and (expired > 0) == (window.duration is not None)
    # the selections read only what is kept
    plain = E.read_export(b"\n".join(data.splitlines()[i] for i in kept) + b"\n")
    assert (m.events, m.set_events, m.n_ignored) == ([(u, e, i, t) for u, e, i, t in plain.events], plain.set_events, plain.n_ignored)
    assert {k: v for k, v in m.ranking_events.items() if v} == {k: v for k, v in plain.ranking_events.items() if v}


def test_no_window_is_the_plain_read():
    data = random_export(9)
    a, b = E.read_export(data), E.read_export(data, E.EventWindow(), NOW)
    assert (a.events, a.ranking_events, a.set_events, a.n_ignored) == (b.events, b.ranking_events, b.set_events, b.n_ignored)
    assert (b.n_expired, b.n_duplicates) == (0, 0)


def test_an_expired_delete_revives_the_sets_before_it():
    rows = [{"event": "$set", "entityType": "item", "entityId": "i", "properties": {"a": 1}, "eventTime": iso_ms(NOW - 9 * DAY)},
            {"event": "$delete", "entityType": "item", "entityId": "i", "eventTime": iso_ms(NOW - 8 * DAY)},
            {"event": "$unset", "entityType": "item", "entityId": "j", "properties": {"a": 0}, "eventTime": iso_ms(NOW - 8 * DAY)}]
    data = b"\n".join(json.dumps(r).encode() for r in rows)
    assert E.read_export(data).set_events == []
    m = E.read_export(data, E.EventWindow("7 days"), NOW)
    assert [(i, {k: v.text for k, v in d.items()}) for i, d in m.set_events] == [("i", {"a": "1"})] and m.n_expired == 1


def test_a_bad_line_still_raises_when_it_would_be_dropped():
    old = iso_ms(NOW - 9 * DAY)
    empty = json.dumps({"event": "buy", "entityType": "user", "entityId": "", "targetEntityType": "item", "targetEntityId": "i",
                        "eventTime": old}).encode()
    with pytest.raises(ValueError, match="line 0: Empty user or item ID"):
        E.read_export(empty, E.EventWindow("1 day", True), NOW)
    with pytest.raises(ValueError, match="needs now_ms"):
        E.read_export(b"", E.EventWindow("1 day"))


@pytest.mark.parametrize("text,ms", [
    ("1 day", DAY), ("2days", 2 * DAY), ("3 d", 3 * DAY), (" 1 0 days ", 10 * DAY), ("1.5 days", 36 * 3_600_000),
    ("12 hours", 43_200_000), ("1h", 3_600_000), ("90 min", 5_400_000), ("1 minute", 60_000), ("2 minutes", 120_000),
    ("30 s", 30_000), ("1 sec", 1000), ("5 secs", 5000), ("1 second", 1000), ("0.0015 seconds", 1), ("7 ms", 7),
    ("7 millis", 7), ("1 millisecond", 1), ("1999999 ns", 1), ("2000000 nanos", 2), ("1500 micros", 1), ("1500 µs", 1),
    ("-1 day", -DAY + 1),   # (nanos + 0.5).toLong rounds -86400e12 up by one nanosecond ("+2 h", 7_200_000), (".5 s", 500), ("1e3 ms", 1000), ("0.9999999 ms", 1), ("0.0000004 ms", 0),
    ("-0.0000006 ms", 0), ("9007199254740993 ns", 9007199254),
])
def test_duration_ms(text, ms):
    assert duration_ms(text) == ms


@pytest.mark.parametrize("text", ["", "day", "1", "259200", "1 mins", "1 m", "1 hrs", "1 weeks", "Inf", "PlusInf", "-Inf", "MinusInf",
                                  "1,5 days", "1..5 s", "0x10 s", "NaN s", "1 day 2 h", "106752 days", "9223372036854775808 ns"])
def test_bad_durations(text):
    with pytest.raises(ValueError):
        duration_ms(text)


def test_data_source_params_from_engine_json():
    engine = json.loads("""{"datasource": {"params": {"appName": "shop", "eventNames": ["buy", "view"], "minEventsPerUser": 3,
                         "eventWindow": {"duration": "28 days", "removeDuplicates": true, "compressProperties": true}}}}""")
    p = ur.DataSourceParams.from_engine_json(engine["datasource"]["params"])
    assert (p.appName, p.eventNames, p.minEventsPerUser) == ("shop", ["buy", "view"], 3)
    assert p.eventWindow == ur.EventWindow("28 days", True, True)
    assert p.eventWindow.cutoff_ms(NOW) == NOW - 28 * DAY
    bare = ur.DataSourceParams.from_engine_json({"appName": "a"})
    assert bare.eventWindow is None and bare.eventNames is None and bare.minEventsPerUser is None
    w = ur.DataSourceParams.from_engine_json({"eventWindow": {"duration": "1 day"}}).eventWindow
    assert (w.removeDuplicates, w.compressProperties, w.cutoff_ms(NOW)) == (False, False, NOW - DAY)
    assert ur.EventWindow(removeDuplicates=True).cutoff_ms(NOW) is None


def test_c_program_links_against_the_event_window_entries(tmp_path):
    from universal_recommender_b200 import _native
    exe = tmp_path / "event_window_abi_check"
    libdir = os.path.dirname(_native.LIB_PATH)
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "abi", "event_window_abi_check.c"), "-o", str(exe), "-L", libdir, "-lcco_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    p = subprocess.run([str(exe)], capture_output=True, text=True)
    assert p.returncode == 0 and p.stdout == "ok\n", (p.returncode, p.stdout, p.stderr)


def test_window_entries_refuse_bad_arguments_without_a_gpu():
    import ctypes
    from universal_recommender_b200 import _native as N
    L = N.lib()
    h = ctypes.c_void_p()
    x, d = ctypes.c_int64(), ctypes.c_int64()
    assert L.cco_event_log_begin_window(None, 1, None, ctypes.byref(h)) == N.E_INVALID_ARG
    assert L.cco_event_log_window_stats(None, ctypes.byref(x), ctypes.byref(d)) == N.E_INVALID_ARG
