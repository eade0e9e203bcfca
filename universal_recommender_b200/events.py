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
    export cannot go through calc_all_on_device / calc_pop_on_device, only through the *_from_events paths.

The DataSource's eventWindow (read_export(window=...), cco_event_log_begin_window) cleans the events first, as PredictionIO's
SelfCleaningDataSource does before every read [RECALL, unverifiable here]: every line is still parsed and checked; then
an event at or before now - duration expires unless it is a $set or $unset; then, with removeDuplicates, events of equal
identity (event_identity) collapse to the one with the latest eventTime, ties to the later line.  The training, ranking
and property selections read what is left."""
from __future__ import annotations

import json
import os
import re
from json.decoder import scanstring
from dataclasses import dataclass, field
from typing import Optional, Sequence

from .ur_model import RawJson, duration_ms

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


def raw_member(line: str, name: str) -> Optional[str]:
    """the trimmed text of the last top-level member `name` of an event line, None when absent"""
    top, _ = _members(line, _WS.match(line).end())
    spans = [(b, e) for n, b, e in top if n == name]
    return line[spans[-1][0]:spans[-1][1]] if spans else None


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
    pr_id: object = None      # the decoded prId (a string), None when absent or null
    tags: str = "[]"          # the trimmed text of tags; absent and null are "[]"


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
    text = raw.decode("utf-8", "surrogatepass")
    tags = raw_member(text, "tags") if "tags" in obj else None
    return Event(i, obj["event"], obj["entityType"], obj["entityId"], tt, ti, t, props, obj.get("prId"),
                 "[]" if tags in (None, "null") else tags)


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
    n_expired: int = 0                 # lines the eventWindow dropped (EventLog.window_stats)
    n_duplicates: int = 0


@dataclass
class EventWindow:
    """engine.json datasource.params.eventWindow, PredictionIO's EventWindow(duration, removeDuplicates,
    compressProperties).  duration: a scala.concurrent.duration string (ur_model.duration_ms), None: nothing expires.
    compressProperties applies to the cleaned events written back (clean_export, ur.clean_export): each item's $set /
    $unset lines are folded into one where that leaves what aggregateProperties returns unchanged.  A read does not
    rewrite events, so it changes nothing in read_export or CcoContext.read_events."""
    duration: Optional[str] = None
    removeDuplicates: bool = False
    compressProperties: bool = False

    @staticmethod
    def from_json(d: Optional[dict]) -> Optional["EventWindow"]:
        if d is None:
            return None
        return EventWindow(d.get("duration"), bool(d.get("removeDuplicates", False)), bool(d.get("compressProperties", False)))

    def cutoff_ms(self, now_ms: int) -> Optional[int]:
        """events at or before it expire ($set / $unset excepted); None without a duration"""
        return None if self.duration is None else now_ms - duration_ms(self.duration)


@dataclass
class DataSourceParams:
    """DataSourceParams (DataSource.scala:36-41): engine.json's datasource.params"""
    appName: Optional[str] = None
    eventNames: Optional[Sequence[str]] = None
    eventWindow: Optional[EventWindow] = None
    minEventsPerUser: Optional[int] = None

    @staticmethod
    def from_engine_json(params: dict) -> "DataSourceParams":
        return DataSourceParams(params.get("appName"), params.get("eventNames"), EventWindow.from_json(params.get("eventWindow")),
                                params.get("minEventsPerUser"))


def event_identity(e: Event) -> tuple:
    """what removeDuplicates compares: the event without eventId, eventTime and creationTime.  Properties are the set of
    their top-level (name, trimmed value text) members, tags the trimmed text: nested values compare by text, as on the
    device (json4s would compare numbers by value and objects without regard to member order)."""
    return (e.event, e.entity_type, e.entity_id, e.target_type, e.target_id, e.pr_id, e.tags,
            frozenset((k, v.text) for k, v in e.properties.items()))


def clean_events(events: Sequence[Event], window: Optional[EventWindow], now_ms: Optional[int]) -> tuple[list, int, int]:
    """the events the window keeps, in line order -> (events, expired, duplicates)"""
    if window is None:
        return list(events), 0, 0
    cutoff = window.cutoff_ms(now_ms) if window.duration is not None else None
    kept = [e for e in events if cutoff is None or e.time_ms > cutoff or e.event in ("$set", "$unset")]
    expired = len(events) - len(kept)
    if not window.removeDuplicates:
        return kept, expired, 0
    best: dict = {}
    for e in kept:
        k = event_identity(e)
        if k not in best or (e.time_ms, e.line) > (best[k].time_ms, best[k].line):
            best[k] = e
    out = sorted(best.values(), key=lambda e: e.line)
    return out, expired, len(kept) - len(out)


@dataclass
class KeptEvents:
    """what an extendable log keeps of the lines read so far (CcoContext.read_events(extendable=True)): the events the window
    kept, the drop counts, and the eventTimes of the events removeDuplicates dropped that are neither $set nor $unset (a
    later cutoff turns those into expired events).  cutoff: the window's, None when nothing expires."""
    events: list = field(default_factory=list)
    n_expired: int = 0
    n_duplicates: int = 0
    dup_times: list = field(default_factory=list)
    cutoff: Optional[int] = None
    remove_duplicates: Optional[bool] = None   # None: nothing read yet


def extend_clean(kept: KeptEvents, new_events: Sequence[Event], window: Optional[EventWindow], now_ms: Optional[int]) -> KeptEvents:
    """the mirror of EventLog.extend: kept (the state after events A under an earlier window) with the events B that follow
    them (lines numbered after A's) under `window`.  The contract: extend_clean(clean_kept(A, w1), B, w2) gives the events
    and counts of clean_events(A + B, w2) whenever w2's cutoff is at or after w1's and removeDuplicates is the same.  It
    holds because an event dropped under the earlier cutoff is dropped under the later one: among equal events the kept
    one is the latest, so when it expires all of them have, and a duplicate drop at or before the new cutoff is an expired
    event of the whole read.  A cutoff before kept.cutoff raises: the events it would bring back are gone."""
    cutoff = window.cutoff_ms(now_ms) if window is not None and window.duration is not None else None
    if kept.cutoff is not None and (cutoff is None or cutoff < kept.cutoff):
        raise ValueError("the cutoff cannot move back: the events it expired are gone")
    dedup = window is not None and window.removeDuplicates
    if kept.remove_duplicates is not None and dedup != kept.remove_duplicates:
        raise ValueError("removeDuplicates cannot change between reads")
    exempt = lambda e: e.event in ("$set", "$unset")
    gone = lambda t: cutoff is not None and t <= cutoff
    old = [e for e in kept.events if exempt(e) or not gone(e.time_ms)]
    new = [e for e in new_events if exempt(e) or not gone(e.time_ms)]
    moved = sum(1 for t in kept.dup_times if gone(t))
    n_expired = kept.n_expired + (len(kept.events) - len(old)) + (len(new_events) - len(new)) + moved
    n_dup = kept.n_duplicates - moved
    dup_times = [t for t in kept.dup_times if not gone(t)]
    out = old + new
    if dedup:
        best: dict = {}
        for e in out:
            k = event_identity(e)
            if k not in best or (e.time_ms, e.line) > (best[k].time_ms, best[k].line):
                best[k] = e
        stay = {id(e) for e in best.values()}
        dropped = [e for e in out if id(e) not in stay]
        n_dup += len(dropped)
        dup_times += [e.time_ms for e in dropped if not exempt(e)]
        out = [e for e in out if id(e) in stay]
    return KeptEvents(out, n_expired, n_dup, dup_times, cutoff, dedup)


def clean_kept(events: Sequence[Event], window: Optional[EventWindow], now_ms: Optional[int]) -> KeptEvents:
    """clean_events as the state an extendable log keeps: the extend of nothing"""
    return extend_clean(KeptEvents(), events, window, now_ms)


def erased_line(e: Event, users, items) -> bool:
    """whether EventLog.erase(users, items) takes the line out (cco_event_log_erase): a training event (entityType "user",
    targetEntityType "item") of one of the users; any line whose targetEntityId is one of the items, whatever its types, as
    PopModel reads ranking events by id; an item property event ($set / $unset / $delete) of one of the items.  Ids are
    the decoded strings.  A user's lines without an item target and lines naming an item only as a non-property entityId
    are never erased: the log holds no id for them."""
    if e.target_id is not None and e.entity_type == "user" and e.target_type == "item" and e.entity_id in users:
        return True
    if e.target_id is not None and e.target_id in items:
        return True
    return is_property_event(e) and e.entity_id in items


def erase_kept(kept: KeptEvents, users, items) -> tuple[KeptEvents, int]:
    """the mirror of EventLog.erase: kept without its erased events -> (state, lines erased).  dup_times, n_expired and
    n_duplicates stay: they count lines read, and the log holds no id for a dropped duplicate.

    The contract: the rule is made of whole removeDuplicates groups (event_identity holds entityId and targetEntityId),
    so erasing E from clean_kept(X, w) keeps the events clean_events(X - E, w) keeps, X - E being X without E's lines, and
    an extend after it keeps what clean_events((X - E) + B, w') keeps.  Lines read = retained + expired + duplicates +
    erased holds across erases and extends."""
    users, items = set(users), set(items)
    out = [e for e in kept.events if not erased_line(e, users, items)]
    return (KeptEvents(out, kept.n_expired, kept.n_duplicates, list(kept.dup_times), kept.cutoff, kept.remove_duplicates),
            len(kept.events) - len(out))


def _fold_line(group: Sequence[Event], lines: Sequence[bytes]) -> bytes:
    """one $set / $unset line for a group of one entity's property lines (no $delete, no target): the fold in (eventTime,
    line) order.  With a $set, aggregate_property_events' state (None at first, so an $unset before the first $set does
    nothing) as a $set, members in dict insertion order; with only $unsets, one $unset of the union of the names, each with
    its last value text.  eventTime: the last folded event's eventTime text."""
    from .ur_query import json_string
    order = sorted(group, key=lambda e: (e.time_ms, e.line))
    if any(e.event == "$set" for e in order):
        state = None
        for e in order:
            if e.event == "$set":
                state = {**state, **e.properties} if state is not None else dict(e.properties)
            elif state is not None:
                state = {k: v for k, v in state.items() if k not in e.properties}
        name, props = "$set", state
    else:
        props: dict = {}
        for e in order:
            props.update(e.properties)
        name = "$unset"
    last = order[-1]
    time_text = raw_member(lines[last.line].decode("utf-8", "surrogatepass"), "eventTime")
    members = ",".join(f"{json_string(k)}:{v.text}" for k, v in props.items())
    text = (f'{{"event":{json_string(name)},"entityType":{json_string(last.entity_type)},"entityId":{json_string(last.entity_id)},'
            f'"properties":{{{members}}},"eventTime":{time_text}}}')
    return text.encode("utf-8", "surrogatepass") + b"\n"


def clean_export(data, window: Optional[EventWindow], now_ms: Optional[int], compress_properties: bool = False) -> bytes:
    """PredictionIO's cleanPersistedPEvents as a compacted export [RECALL, unverifiable here]: the lines clean_events keeps,
    in line order, each copied byte for byte and ending in '\\n' (as join_parts ends a part).  data: as read_export takes it.

    compress_properties: the kept $set / $unset lines of items (entityType "item", the property events a read aggregates)
    are grouped by decoded entityId.  Other entity types' lines stay verbatim: a resident log keeps the item property
    lines only, so those are what the device can group before the source streams past, and no read looks at the others.
    These stay verbatim in place: the property lines of an entity with a kept $delete line, of an entity with a kept
    $set / $unset that carries a target entity (that line is also a ranking event, and a fold around it would move it in
    the (eventTime, line) order), and the line of an entity with only one.  Every other group becomes one line (_fold_line),
    written after all verbatim lines in the order of each group's first line.

    The contract: for any later window w' (cutoff at or after this one's, the same removeDuplicates) and now',
    read_export(clean_export(X, w, now, p), w', now') gives the training events and the ranking events per name (names left
    without events aside) that read_export(X, w', now') gives, and the same aggregated properties as {item: {field: text}};
    without compress_properties also n_ignored and the order of the property-only items.  It holds because a line dropped
    under w is dropped under w' (extend_clean), $set / $unset never expire, and an entity whose $delete could expire
    later is never folded.

    Deviations from PredictionIO (whose compressPProperties is recalled, not read): PIO folds every entity type; PIO folds across $delete, which changes
    what aggregateProperties returns; PIO's fold keeps the first event's name and eventId, this one writes a new $set or
    $unset without eventId, creationTime, prId or tags; members are in insertion order, not Scala Map order; the folded
    lines come last, as an export has no order the store keeps."""
    if isinstance(data, (str, os.PathLike)):
        data = join_parts(export_parts(data))
    if window is not None and window.duration is not None and now_ms is None:
        raise ValueError("an eventWindow with a duration needs now_ms")
    lines = export_lines(bytes(data))
    kept, _, _ = clean_events([parse_line(i, raw) for i, raw in enumerate(lines)], window, now_ms)
    folded: dict = {}
    if compress_properties:
        ent = lambda e: (e.entity_type, e.entity_id)
        props = [e for e in kept if is_property_event(e)]
        pinned = {ent(e) for e in props if e.event == "$delete" or e.target_id is not None}
        for e in props:
            if e.event in ("$set", "$unset") and ent(e) not in pinned:
                folded.setdefault(ent(e), []).append(e)
        folded = {k: g for k, g in folded.items() if len(g) > 1}
    gone = {e.line for g in folded.values() for e in g}
    out = [lines[e.line] + b"\n" for e in kept if e.line not in gone]
    out += [_fold_line(g, lines) for g in folded.values()]
    return b"".join(out)


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


def read_export(data, window: Optional[EventWindow] = None, now_ms: Optional[int] = None) -> DataSourceEvents:
    """data: the export's bytes, or the directory `pio export` writes (its parts joined as join_parts does); window: the
    eventWindow, its duration counted back from now_ms (required with a duration).  Event names are listed for every line
    read, expired and duplicate ones included, as the device numbers them while it parses."""
    if isinstance(data, (str, os.PathLike)):
        data = join_parts(export_parts(data))
    if window is not None and window.duration is not None and now_ms is None:
        raise ValueError("an eventWindow with a duration needs now_ms")
    names: dict = {}
    parsed = []
    for i, raw in enumerate(export_lines(bytes(data))):
        e = parse_line(i, raw)
        if e.target_id is not None and e.entity_type == "user" and e.target_type == "item" and (not e.entity_id or not e.target_id):
            raise ValueError(f"line {i}: Empty user or item ID")
        names.setdefault(e.event, None)
        parsed.append(e)
    kept, n_expired, n_dup = clean_events(parsed, window, now_ms)
    events, ranking, props, ignored = [], {n: [] for n in names}, [], 0
    for e in kept:
        used = False
        if e.target_id is not None:
            used = True
            ranking[e.event].append((e.target_id, e.time_ms))
            if e.entity_type == "user" and e.target_type == "item":
                events.append((e.entity_id, e.event, e.target_id, e.time_ms))
        if is_property_event(e):
            used = True
            props.append(e)
        ignored += not used
    return DataSourceEvents(list(names), events, ranking, aggregate_property_events(props), ignored, props, n_expired, n_dup)
