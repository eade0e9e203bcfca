"""Host mirror of the DataSource (DataSource.scala:65-102) over a PredictionIO event export (`pio export`: JSON lines, one
event per line), the restatement cco_event_log_read (include/cco_b200.h) is held to.  It selects what the reference reads:

  training events  entityType "user" and targetEntityType "item", by event name (an empty id raises, as the reference's
                   require(..., "Empty user or item ID"));
  ranking events   every event with a targetEntityId, of any entity types, by event name (PopModel.eventsRDD reads the
                   store without an entity-type filter);
  property events  "$set" / "$unset" / "$delete" of entityType "item", aggregated as PEventStore.aggregateProperties does:
                   in (eventTime, line) order -- ties in eventTime go to the later line, the store's order for them being
                   undefined -- "$set" merges its members, "$unset" removes the fields it names, "$delete" drops the item.
                   Values stay the JSON text they were written in (ur_model.RawJson), as the device splices them.  Items
                   come in order of their first property event in line order, an item's fields in the order their names
                   first appear among the members of $set / $unset properties; an item whose final state exists without
                   a field is listed with an empty dict.

eventTime is Joda's extended date-time YYYY-MM-DDThh:mm:ss[.f{1,9}](Z|+hh:mm|+hhmm|+hh), fraction digits past the third
dropped, proleptic Gregorian years 0000-9999.  Anything else raises ValueError naming the 0-based line.

A line is strict UTF-8 text, as `pio export` writes it: a byte order mark is not whitespace, and a line that starts with
one raises here as it does on the device.

What the mirror accepts differs from the device in these ways:
  - every line goes through json.loads here, while the device checks nested values only for closed strings, valid
    escapes and bracket depth (and the members of a property event's properties object).  So a line such as
    {"event":"v",...,"tags":[tru]} raises here and is read by the device, and so does a nested value whose bracket kinds
    do not match, such as the property value {"a":{]}: the device splices its text verbatim;
  - a byte sequence that is not UTF-8 inside a string raises here; the device copies the bytes through, so an id holds
    them verbatim;
  - a \\u escape of a surrogate that is not part of a pair (a high surrogate not followed by a \\u escape of a low one, or a
    lone low one) is written by the device as the surrogate's 3-byte form (\\ud800 -> ED A0 80, Python's
    "surrogatepass").  Here it stays a lone surrogate in the str, which encode_ids (strict UTF-8) cannot encode: such an
    export cannot go through calc_all_on_device / calc_pop_on_device, only through the *_from_events paths."""
from __future__ import annotations

import json
import os
import re
from json.decoder import scanstring
from dataclasses import dataclass, field
from typing import Optional, Sequence

from .ur_model import RawJson

PROPERTY_EVENTS = ("$set", "$unset", "$delete")
_WS = re.compile(r"[ \t\n\r]*")
_DEC = json.JSONDecoder()


def _members(s: str, i: int) -> tuple[list, int]:
    """the members of the JSON object at s[i] ('{') as (name, value start, value end) -> (members, index after '}')"""
    out = []
    i = _WS.match(s, i + 1).end()
    if s[i] == "}":
        return out, i + 1
    while True:
        if s[i] != '"':
            raise ValueError("bad object")
        name, i = scanstring(s, i + 1)
        i = _WS.match(s, i).end()
        if s[i] != ":":
            raise ValueError("bad object")
        i = _WS.match(s, i + 1).end()
        _, j = _DEC.raw_decode(s, i)
        out.append((name, i, j))
        i = _WS.match(s, j).end()
        if s[i] == ",":
            i = _WS.match(s, i + 1).end()
        elif s[i] == "}":
            return out, i + 1
        else:
            raise ValueError("bad object")


def raw_properties(line: str) -> dict:
    """{name: RawJson(text)} of the last "properties" member of an event line (the last of a repeated name wins)"""
    top, _ = _members(line, _WS.match(line).end())
    spans = [(b, e) for n, b, e in top if n == "properties"]
    if not spans:
        return {}
    inner, _ = _members(line, spans[-1][0])
    out: dict = {}
    for n, b, e in inner:
        out[n] = RawJson(line[b:e])
    return out

_TIME = re.compile(rb"([0-9]{4})-([0-9]{2})-([0-9]{2})T([0-9]{2}):([0-9]{2}):([0-9]{2})(?:\.([0-9]{1,9}))?"
                   rb"(Z|[+-][0-9]{2}(?::?[0-9]{2})?)\Z")


def days_from_civil(y: int, m: int, d: int) -> int:
    """days since 1970-01-01 of a proleptic Gregorian date"""
    y -= m <= 2
    era = (y if y >= 0 else y - 399) // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + doy - 719468


def parse_event_time(text: str) -> int:
    """eventTime -> epoch milliseconds (floor); ValueError for any other spelling"""
    m = _TIME.match(text.encode("utf-8", "surrogatepass"))
    if not m:
        raise ValueError(f"bad eventTime {text!r}")
    y, mo, d, h, mi, s = (int(m.group(k)) for k in range(1, 7))
    leap = y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)
    mdays = 29 if mo == 2 and leap else 28 if mo == 2 else 30 if mo in (4, 6, 9, 11) else 31
    if not (1 <= mo <= 12 and 1 <= d <= mdays and h <= 23 and mi <= 59 and s <= 59):
        raise ValueError(f"bad eventTime {text!r}")
    frac = int((m.group(7) or b"").ljust(3, b"0")[:3] or 0)
    off = 0
    z = m.group(8)
    if z != b"Z":
        oh, om = int(z[1:3]), int(z[3:].lstrip(b":") or 0)
        if oh > 23 or om > 59:
            raise ValueError(f"bad eventTime {text!r}")
        off = (oh * 60 + om) * (-1 if z[:1] == b"-" else 1)
    return ((days_from_civil(y, mo, d) * 86400 + h * 3600 + mi * 60 + s) - off * 60) * 1000 + frac


@dataclass
class Event:
    line: int
    event: str
    entity_type: str
    entity_id: str
    target_type: Optional[str]
    target_id: Optional[str]
    time_ms: int
    properties: dict


def parse_line(i: int, raw: bytes) -> Event:
    """one export line -> Event, with the checks of cco_event_log_read (the last of a repeated member wins)"""
    try:   # strict UTF-8 first: json.loads(bytes) would take a leading byte order mark for utf-8-sig
        obj = json.loads(raw.decode("utf-8"))
    except ValueError as e:
        raise ValueError(f"line {i}: not one JSON object ({e})") from None
    if not isinstance(obj, dict):
        raise ValueError(f"line {i}: not a JSON object")
    for k in ("event", "entityType", "entityId", "eventTime"):
        if k not in obj:
            raise ValueError(f"line {i}: an event needs {k!r}")
        if not isinstance(obj[k], str):
            raise ValueError(f"line {i}: {k!r} is not a string")
    tt, ti = obj.get("targetEntityType"), obj.get("targetEntityId")
    for k, v in (("targetEntityType", tt), ("targetEntityId", ti)):
        if v is not None and not isinstance(v, str):
            raise ValueError(f"line {i}: {k!r} is not a string or null")
    props = obj.get("properties", {})
    if not isinstance(props, dict):
        raise ValueError(f"line {i}: 'properties' is not an object")
    if props:
        props = raw_properties(raw.decode("utf-8", "surrogatepass"))
    if (tt is None) != (ti is None):
        raise ValueError(f"line {i}: targetEntityType and targetEntityId must be given together")
    try:
        t = parse_event_time(obj["eventTime"])
    except ValueError as e:
        raise ValueError(f"line {i}: {e}") from None
    return Event(i, obj["event"], obj["entityType"], obj["entityId"], tt, ti, t, props)


def export_lines(data: bytes) -> list[bytes]:
    """lines end in '\\n'; the last one may not"""
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    return lines


def aggregate_property_events(events: Sequence[Event]) -> list[tuple[str, dict]]:
    """aggregateProperties over property events (in line order) -> [(item, fields)] of the items whose final state exists
    (fields may be empty), in order of their first property event; each item's fields in the order their names first
    appear among the members of $set / $unset properties"""
    state: dict = {e.entity_id: None for e in events}
    rank = {n: k for k, n in enumerate(dict.fromkeys(n for e in events if e.event != "$delete" for n in e.properties))}
    for e in sorted(events, key=lambda e: (e.time_ms, e.line)):
        cur = state[e.entity_id]
        if e.event == "$set":
            state[e.entity_id] = {**cur, **e.properties} if cur is not None else dict(e.properties)
        elif e.event == "$unset":
            if cur is not None:
                state[e.entity_id] = {k: v for k, v in cur.items() if k not in e.properties}
        else:
            state[e.entity_id] = None
    return [(item, dict(sorted(d.items(), key=lambda kv: rank[kv[0]]))) for item, d in state.items() if d is not None]


def is_property_event(e: Event) -> bool:
    return e.entity_type == "item" and e.event in PROPERTY_EVENTS


@dataclass
class DataSourceEvents:
    """what the DataSource and PopModel read from an export"""
    names: list                        # every event name, in order of first appearance
    events: list                       # training events (user, event name, item, time ms), line order
    ranking_events: dict               # {event name: [(item, time ms)]}, every name, line order
    set_events: list                   # aggregated properties [(item, {field: value})]
    n_ignored: int = 0
    property_events: list = field(default_factory=list)


def export_parts(directory) -> list[str]:
    """the part files of a `pio export` directory (Spark's saveAsTextFile: part-NNNNN files and a _SUCCESS marker) in name
    order; _SUCCESS, checksum (*.crc) and hidden files and empty parts are skipped"""
    names = sorted(n for n in os.listdir(directory) if n.startswith("part-") and not n.endswith(".crc"))
    paths = [os.path.join(directory, n) for n in names]
    return [p for p in paths if os.path.isfile(p) and os.path.getsize(p) > 0]


def part_lines(path) -> int:
    """lines of one part: every '\\n' ends one, and a last line without it counts too"""
    n, last = 0, b"\n"
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            n += block.count(b"\n")
            last = block[-1:]
    return n + (last != b"\n")


def locate_line(counts: Sequence[int], line: int) -> tuple[int, int]:
    """global 0-based line of parts read in order (each part's lines kept apart) -> (part index, line in that part)"""
    for k, n in enumerate(counts):
        if line < n:
            return k, line
        line -= n
    raise ValueError("line past the last part")


def join_parts(paths: Sequence) -> bytes:
    """the bytes of parts read in order; a part that does not end in '\\n' is followed by one, so that parts never join lines"""
    out = []
    for p in paths:
        with open(p, "rb") as f:
            b = f.read()
        out.append(b + b"\n" if b and not b.endswith(b"\n") else b)
    return b"".join(out)


def read_export(data) -> DataSourceEvents:
    """data: the export's bytes, or the directory `pio export` writes (its parts joined as join_parts does)"""
    if isinstance(data, (str, os.PathLike)):
        data = join_parts(export_parts(data))
    names: dict = {}
    events, ranking, props, ignored = [], {}, [], 0
    for i, raw in enumerate(export_lines(bytes(data))):
        e = parse_line(i, raw)
        names.setdefault(e.event, None)
        ranking.setdefault(e.event, [])
        used = False
        if e.target_id is not None:
            used = True
            ranking[e.event].append((e.target_id, e.time_ms))
            if e.entity_type == "user" and e.target_type == "item":
                if not e.entity_id or not e.target_id:
                    raise ValueError(f"line {i}: Empty user or item ID")
                events.append((e.entity_id, e.event, e.target_id, e.time_ms))
        if is_property_event(e):
            used = True
            props.append(e)
        ignored += not used
    return DataSourceEvents(list(names), events, ranking, aggregate_property_events(props), ignored, props)
