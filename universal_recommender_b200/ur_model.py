"""Host mirror of what calcAll writes besides the correlators (SURVEY.md 8f-2, 8f-3): the item properties and PopModel ranks
of `propertiesRDD` (URAlgorithm.scala:351-367), joined into one document per item by URModel.save's groupAll
(URModel.scala:57-102).  This is the definition cco_format_model is held to; the device builds the same documents from id
strings with CcoContext.format_model.

Precedence inside a document, lowest to highest (Scala `++` and `+`: the later source wins):
  correlator fields < properties (fieldsPropMap ++ rankPropMap) < ranks (a later ranking beats an earlier one of the same
  name, getRanksRDD's foldLeft) < "id" (propsMap + ("id" -> itemId)).

Random rankings (uniqueRank, PopModel.calcRandom): every item of an event in the window, of any event name, plus every item
with a property, valued n · 10^-15 with n a hash of the id bytes and the window (random_rank) instead of the reference's
unseeded Random.nextDouble.  The values change with the window, so with "now" as its end from train to train, as the
reference's do; unlike the reference's, they repeat when a fixed offsetDate repeats the window.
"""
from __future__ import annotations

import datetime
import json
import re
from collections import Counter
from dataclasses import dataclass
from decimal import Decimal
from typing import Iterable, Optional, Sequence


class RankingFieldName:
    """PopModel.scala:31-41"""
    UserRank, UniqueRank, PopRank, TrendRank, HotRank, UnknownRank = "userRank", "uniqueRank", "popRank", "trendRank", "hotRank", "unknownRank"
    ALL = (UserRank, UniqueRank, PopRank, TrendRank, HotRank)


class RankingType:
    """PopModel.scala:43-51"""
    Popular, Trending, Hot, UserDefined, Random = "popular", "trending", "hot", "userDefined", "random"


NAME_BY_TYPE = {RankingType.Popular: RankingFieldName.PopRank, RankingType.Trending: RankingFieldName.TrendRank,
                RankingType.Hot: RankingFieldName.HotRank, RankingType.UserDefined: RankingFieldName.UserRank,
                RankingType.Random: RankingFieldName.UniqueRank}   # PopModel.scala:205-210, default unknownRank

BACKFILL_FIELD_NAME = RankingFieldName.PopRank   # URAlgorithm.scala:64-66
BACKFILL_TYPE = RankingType.Popular
BACKFILL_DURATION = "3650 days"


@dataclass
class RankingParams:
    """URAlgorithm.scala:110-117 (one entry of the engine.json `rankings` list)"""
    name: Optional[str] = None
    type: Optional[str] = None
    eventNames: Optional[Sequence[str]] = None
    offsetDate: Optional[str] = None
    endDate: Optional[str] = None
    duration: Optional[str] = None

    @staticmethod
    def from_json(d: dict) -> "RankingParams":
        return RankingParams(d.get("name"), d.get("type"), d.get("eventNames"), d.get("offsetDate"), d.get("endDate"), d.get("duration"))

    def ranking_type(self) -> str:
        return self.type or BACKFILL_TYPE

    def field_name(self) -> str:
        return self.name or NAME_BY_TYPE.get(self.ranking_type(), RankingFieldName.UnknownRank)


def rankings_params(rankings: Optional[Sequence[RankingParams]], model_event_names: Sequence[str]) -> list[RankingParams]:
    """URAlgorithm.scala:249-256: the configured rankings, or one `popRank` popular ranking over the first model event name
    for "3650 days"; then one ranking per type, the first of each.  Scala's groupBy gives no order; this mirror keeps the
    types in order of first appearance."""
    rs = list(rankings) if rankings is not None else [
        RankingParams(BACKFILL_FIELD_NAME, BACKFILL_TYPE, list(model_event_names[:1]), None, None, BACKFILL_DURATION)]
    by_type: dict = {}
    for r in rs:
        by_type.setdefault(r.type, r)
    return list(by_type.values())


_UNITS = {"d": 86400, "day": 86400, "days": 86400, "h": 3600, "hour": 3600, "hours": 3600,
          "min": 60, "mins": 60, "minute": 60, "minutes": 60, "m": 60,
          "s": 1, "sec": 1, "secs": 1, "second": 1, "seconds": 1,
          "ms": Decimal("0.001"), "milli": Decimal("0.001"), "millis": Decimal("0.001"), "millisecond": Decimal("0.001"),
          "milliseconds": Decimal("0.001")}


def duration_seconds(duration) -> int:
    """`Duration(durationAsString).toSeconds.toInt` for "<n> <unit>" strings (units of scala.concurrent.duration, day to
    millisecond).  A bare number, as examples/pop-engine.json writes it (259200), is read as seconds."""
    if isinstance(duration, (int, float)) and not isinstance(duration, bool):
        return int(duration)
    m = re.fullmatch(r"\s*([0-9]+(?:\.[0-9]+)?)\s*([A-Za-z]*)\s*", str(duration))
    if not m or (m.group(2) and m.group(2) not in _UNITS):
        raise ValueError(f"bad duration {duration!r}")
    return int(Decimal(m.group(1)) * (_UNITS[m.group(2)] if m.group(2) else 1))


_NANOS = {**{u: 86_400_000_000_000 for u in ("d", "day", "days")}, **{u: 3_600_000_000_000 for u in ("h", "hour", "hours")},
          **{u: 60_000_000_000 for u in ("min", "minute", "minutes")}, **{u: 1_000_000_000 for u in ("s", "sec", "secs", "second", "seconds")},
          **{u: 1_000_000 for u in ("ms", "milli", "millis", "millisecond", "milliseconds")},
          **{u: 1_000 for u in ("µs", "micro", "micros", "microsecond", "microseconds")},
          **{u: 1 for u in ("ns", "nano", "nanos", "nanosecond", "nanoseconds")}}
_DOUBLE = re.compile(r"[+-]?(?:[0-9]+\.?[0-9]*|\.[0-9]+)(?:[eE][+-]?[0-9]+)?")
_LONG_MAX = (1 << 63) - 1


def duration_ms(duration: str) -> int:
    """Scala's `Duration(duration).toMillis`, as PredictionIO's EventWindow reads its duration [RECALL, unverifiable here]:
    whitespace is removed; the unit is the trailing letters, one of scala.concurrent.duration's labels (d day, h hour,
    min minute, s sec second, ms milli millisecond, µs micro microsecond, ns nano nanosecond; each word also with an "s");
    the number before it is a Java double.  Up to 2^53 it is scaled to nanoseconds in double arithmetic and rounded (x +
    0.5, truncated), beyond that it must be an integer and is scaled exactly; either way |nanoseconds| <= 2^63 - 1.  The
    result is truncated toward zero to milliseconds.  "Inf" and the other infinite durations have no millisecond value:
    like everything else that does not parse, they raise ValueError."""
    s = "".join(str(duration).split())
    unit = re.search(r"[^\W\d_]*\Z", s).group(0)
    num = s[:len(s) - len(unit)]
    if unit not in _NANOS or not _DOUBLE.fullmatch(num):
        raise ValueError(f"bad duration {duration!r}")
    value = float(num)
    if abs(value) <= 2.0 ** 53:
        nanos = float(_NANOS[unit]) * value
        if not -_LONG_MAX - 1 <= nanos <= _LONG_MAX:
            raise ValueError(f"duration {duration!r} is out of range")
        nanos = int(nanos + 0.5)
    else:
        if not re.fullmatch(r"[+-]?[0-9]+", num):
            raise ValueError(f"bad duration {duration!r}")
        nanos = int(num) * _NANOS[unit]
        if not -_LONG_MAX <= nanos <= _LONG_MAX:
            raise ValueError(f"duration {duration!r} is out of range")
    ms = abs(nanos) // 1_000_000
    return ms if nanos >= 0 else -ms


def ranking_window(rp: RankingParams, now_ms: int) -> tuple[int, int]:
    """PopModel.calc (PopModel.scala:57-77): end = offsetDate (ISO 8601; 'now' if it does not parse, as the reference
    warns and does), start = end - duration seconds.  Events count in [start, end)."""
    end = now_ms
    if rp.offsetDate is not None:
        try:
            dt = datetime.datetime.fromisoformat(rp.offsetDate.replace("Z", "+00:00"))
            if dt.tzinfo is None:
                dt = dt.replace(tzinfo=datetime.timezone.utc)
            end = int(dt.timestamp() * 1000)
        except ValueError:
            end = now_ms
    return end - duration_seconds(rp.duration if rp.duration is not None else BACKFILL_DURATION) * 1000, end


_M64 = (1 << 64) - 1


def _mix64(z: int) -> int:
    """mix64 of cco_kernels.cuh on one Python int (synth._mix64 is the numpy form)"""
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & _M64
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def id_hash(item: str) -> int:
    """the 64-bit hash k_str_hash (cco_strings.cuh, mask ~0) gives an id: mix64 over its UTF-8 bytes as little-endian 8-byte
    words, the last one zero-padded, then over the length"""
    b = item.encode("utf-8")
    h = 0x243F6A8885A308D3
    for k in range(0, len(b), 8):
        h = (_mix64(h ^ int.from_bytes(b[k:k + 8], "little")) + 0x9E3779B97F4A7C15) & _M64
    return _mix64(h ^ len(b))


def random_rank(item: str, start_ms: int, end_ms: int) -> int:
    """n of an item's random rank n · 10^-15 (0 <= n < 10^15) over the window [start_ms, end_ms):
    r = mix64(id_hash ^ mix64(start ^ mix64(end))) as uint64, n = floor(r · 10^15 / 2^64)"""
    window = _mix64((start_ms & _M64) ^ _mix64(end_ms & _M64))
    return (_mix64(id_hash(item) ^ window) * 10**15) >> 64


def pop_scores(mode: str, items: Sequence[str], times_ms: Sequence[int], start_ms: int, end_ms: int) -> dict:
    """PopModel.calcPopular / calcTrending / calcHot (PopModel.scala:113-182) per item id: {item: score} for the items the
    reference's RDD holds.  Same rules as cco_pop_model, including the empty-bucket ones."""
    def count(lo, hi):
        return Counter(j for j, t in zip(items, times_ms) if lo <= t < hi)
    dur = end_ms - start_ms
    if mode == RankingType.Popular:
        return {j: float(c) for j, c in count(start_ms, end_ms).items()}
    if mode == RankingType.Trending:
        half = dur // 2
        older = count(start_ms, start_ms + half)
        if not older:
            return {}
        newer = count(start_ms + half, end_ms)
        return {j: float(newer[j] - older[j]) for j in newer if j in older}
    if mode == RankingType.Hot:
        third = dur // 3
        older = count(start_ms, start_ms + third)
        middle = count(start_ms + third, start_ms + 2 * third)
        if not older or not middle:
            return {}
        newer = count(start_ms + 2 * third, end_ms)
        return {j: float((newer[j] - middle[j]) - (middle[j] - older[j])) for j in newer if j in middle and j in older}
    raise ValueError(mode)


@dataclass
class Ranking:
    """One ranking ready for the model: its field, PopModel mode, window and per-event-name streams of (item, time)."""
    field: str
    mode: str
    start_ms: int
    end_ms: int
    streams: list   # [(item ids list[str], times list[int])] one per event name

    def scores(self, property_items: Iterable[str] = ()) -> dict:
        """{item: score}; a random ranking also scores the items that have a property"""
        items = [i for s in self.streams for i in s[0]]
        times = [t for s in self.streams for t in s[1]]
        if self.mode == RankingType.Random:
            keep = [i for i, t in zip(items, times) if self.start_ms <= t < self.end_ms] + list(property_items)
            return {i: random_rank(i, self.start_ms, self.end_ms) / 1e15 for i in dict.fromkeys(keep)}
        return pop_scores(self.mode, items, times, self.start_ms, self.end_ms)


def rankings_for(params: Sequence[RankingParams], events_by_name: dict, now_ms: int, model_event_names: Sequence[str]) -> list[Ranking]:
    """getRanksRDD (URAlgorithm.scala:537-560): one Ranking per histogram or random ranking.  A ranking reads the event store
    (every user's events of its event names, {name: [(item, time ms)]}), not the Preparator output; without eventNames it
    reads the first model event name.  A random ranking reads every event name, in the order of events_by_name, and ignores
    its eventNames (calcRandom, PopModel.scala:98-110).  userDefined rankings produce nothing (PopModel returns an empty RDD;
    the field comes from the item's own properties)."""
    out = []
    for rp in params:
        t = rp.ranking_type()
        if t not in (RankingType.Popular, RankingType.Trending, RankingType.Hot, RankingType.Random):
            continue   # userDefined, or an unknown type the reference warns about and skips
        start, end = ranking_window(rp, now_ms)
        if t == RankingType.Random:
            names = list(events_by_name)
        else:
            names = rp.eventNames if rp.eventNames is not None else list(model_event_names[:1])
        streams = [([i for i, _ in events_by_name.get(n, [])], [tm for _, tm in events_by_name.get(n, [])]) for n in names]
        out.append(Ranking(rp.field_name(), t, start, end, streams or [([], [])]))
    return out


def aggregate_properties(set_events: Iterable[tuple[str, dict]]) -> list[tuple[str, str, object]]:
    """`$set` events in event-time order -> (item, field, value) triples, one per (item, field): later sets of a key win.
    Items and fields keep the order of their first `$set`.  `$unset` / `$delete` stay with the event store."""
    props: dict = {}
    for item, fields in set_events:
        d = props.setdefault(item, {})
        for k, v in fields.items():
            d[k] = v
    return [(item, k, v) for item, d in props.items() for k, v in d.items()]


def extract_jvalue(key: str, value):
    """URModel.extractJvalue (URModel.scala:126-140) without the date conversion: a string under a RankingFieldName becomes a
    double, lists convert elementwise, everything else stays."""
    if isinstance(value, list):
        return [extract_jvalue(key, v) for v in value]
    if isinstance(value, str) and key in RankingFieldName.ALL:
        return float(value)
    return value


def java_double(x: float) -> str:
    """Java's Double.toString: plain decimal with at least one fraction digit for 1e-3 <= |x| < 1e7, else computerised
    scientific notation (1.0E7, 1.5E-4), over the shortest digits that round-trip (Python's repr digits, as JDK 19+ prints
    them).  Not checked against a JVM here."""
    x = float(x)
    if x != x or x in (float("inf"), float("-inf")):
        raise ValueError(f"{x} has no JSON text")
    sign = "-" if str(x).startswith("-") else ""
    if x == 0:
        return sign + "0.0"
    _, digits, exp = Decimal(repr(abs(x))).normalize().as_tuple()
    ds = "".join(map(str, digits))   # significant digits, no leading or trailing zeros
    point = len(ds) + exp            # digits before the decimal point
    if 1e-3 <= abs(x) < 1e7:
        if point <= 0:
            return sign + "0." + "0" * (-point) + ds
        if point >= len(ds):
            return sign + ds + "0" * (point - len(ds)) + ".0"
        return sign + ds[:point] + "." + ds[point:]
    return sign + ds[0] + "." + (ds[1:] or "0") + "E" + str(point - 1)


def json_string(s: str) -> str:
    """the repo's JSON string escaping (cco_format_es_bulk): '"' and '\\' get a backslash, code points below 0x20 become
    \\u00xx, everything else passes through"""
    out = []
    for ch in s:
        if ch in '"\\':
            out.append("\\" + ch)
        elif ord(ch) < 0x20:
            out.append("\\u%04x" % ord(ch))
        else:
            out.append(ch)
    return '"' + "".join(out) + '"'


class RawJson:
    """a property value kept as the JSON text it was written in (an event export's member value, trimmed): spliced as is"""
    __slots__ = ("text",)

    def __init__(self, text: str):
        self.text = text

    def __eq__(self, other):
        return isinstance(other, RawJson) and other.text == self.text

    def __repr__(self):
        return f"RawJson({self.text!r})"


def property_json(value) -> str:
    """a property value -> the JSON text the device splices verbatim (floats as Java's Double.toString; RawJson as written)"""
    if isinstance(value, RawJson):
        return value.text
    if value is None:
        return "null"
    if isinstance(value, bool):
        return "true" if value else "false"
    if isinstance(value, int):
        return str(value)
    if isinstance(value, float):
        return java_double(value)
    if isinstance(value, str):
        return json_string(value)
    if isinstance(value, (list, tuple)):
        return "[" + ",".join(property_json(v) for v in value) + "]"
    if isinstance(value, dict):
        return "{" + ",".join(json_string(str(k)) + ":" + property_json(v) for k, v in value.items()) + "}"
    raise TypeError(f"no JSON text for {type(value).__name__}")


def model_documents(row_ids: Sequence[str], indicators: Sequence[tuple[str, Sequence[Sequence[str]]]],
                    properties: Sequence[tuple[str, str, object]], rankings: Sequence[Ranking]) -> list[dict]:
    """URModel.save's groupAll / getRanksRDD's fullOuterJoin as one dict per item, in the documents' order: the rows first
    (row order), then the items without a row that have a property or a score, by first appearance (property triples, then
    the ranking streams in order).  A random ranking scores the property items too.  indicators = [(event name, correlator
    ids per row)]; properties = (item, field, value) triples, the last of a repeated (item, field) wins."""
    props: dict = {}
    for item, f, v in properties:
        props.setdefault(item, {})[f] = v
    scored = [(r.field, r.scores([i for i, _, _ in properties])) for r in rankings]
    rows = set(row_ids)
    order = list(row_ids)
    seen = set()
    candidates = [i for i, _, _ in properties] + [i for r in rankings for s in r.streams for i in s[0]]
    for item in candidates:
        if item in rows or item in seen:
            continue
        seen.add(item)
        if item in props or any(item in sc for _, sc in scored):
            order.append(item)
    docs = []
    for d, item in enumerate(order):
        doc: dict = {}
        if d < len(row_ids):
            for name, lists in indicators:
                doc[name] = list(lists[d])
        doc.update(props.get(item, {}))
        for name, sc in scored:
            if item in sc:
                doc[name] = sc[item]
        doc["id"] = item
        docs.append(doc)
    return docs


def rerank_documents(old_docs: Sequence[tuple[str, dict]], properties: Sequence[tuple[str, str, object]],
                     rankings: Sequence[Ranking]) -> list[dict]:
    """calcPop's documents (URAlgorithm.scala:375-399): the current index `old_docs` = [(item id, {member: value})] in index
    order joined with fresh properties and rankings the way calcPop + URModel.save join them, one dict per item in the
    order cco_rerank_model writes the documents: the old documents first, then the items without one that have a property
    or a score, by first appearance (property triples, then the ranking streams in order).
    propertiesRDD = current.fullOuterJoin(ranks) gives meta ++ rank, and save's groupAll puts the fresh fields under it,
    so per document, lowest to highest: fresh properties < old members < rankings (a later one beats an earlier one of the
    same name) < "id".  A fresh `$set` value loses to an old member of the same name, and an old rank member survives when
    the item has no score in the new ranking.  Random rankings cover the property items, not items only in the index."""
    props: dict = {}
    for item, f, v in properties:
        props.setdefault(item, {})[f] = v
    scored = [(r.field, r.scores([i for i, _, _ in properties])) for r in rankings]
    have = {item for item, _ in old_docs}
    order = list(old_docs)
    seen = set()
    for item in [i for i, _, _ in properties] + [i for r in rankings for s in r.streams for i in s[0]]:
        if item in have or item in seen:
            continue
        seen.add(item)
        if item in props or any(item in sc for _, sc in scored):
            order.append((item, {}))
    docs = []
    for item, meta in order:
        doc = dict(props.get(item, {}))
        doc.update(meta)
        for name, sc in scored:
            if item in sc:
                doc[name] = sc[item]
        doc["id"] = item
        docs.append(doc)
    return docs


# ---- the index read back from Elasticsearch -------------------------------------------------------------------------------
# EsClient.getRDD (esJsonRDD, EsClient.scala:464-470) scrolls the index for calcPop, EsClient.getSource (EsClient.scala:
# 394-442) reads one document for the item queries.  index_from_pages is the host mirror of cco_index_pages_*: the pages
# of a _search / _search/scroll turned back into the bulk body above, one `{"index":{"_id":"<id>"}}\n<_source>\n` per hit.
_WS = b" \t\n\r"
_STRING = re.compile(rb'"(?:[^"\\]|\\.)*"', re.S)
_STRUCT = re.compile(rb'"(?:[^"\\]|\\.)*"|\\.|"|[{}\[\]]', re.S)       # a string, an escape pair outside one, a lone quote, a bracket
_GOOD_STRING = re.compile(rb'"(?:[^"\\\x00-\x1f]|\\["\\/bfnrt]|\\u[0-9a-fA-F]{4})*"')
_NUMBER = re.compile(rb"-?(?:0|[1-9][0-9]*)(?:\.[0-9]+)?(?:[eE][+-]?[0-9]+)?\Z")
_INTEGER = re.compile(rb"-?(?:0|[1-9][0-9]*)\Z")
_COMPACT = re.compile(rb'("(?:[^"\\]|\\.)*")|[ \t\n\r]+', re.S)


class _PageError(ValueError):
    pass


def _string_bad(b: bytes, i: int, e: int) -> int:
    """the first bad byte of the raw string inside b[i:e] (a raw byte < 0x20, a bad escape), -1"""
    while i < e:
        c = b[i]
        if c < 0x20:
            return i
        if c != 0x5C:
            i += 1
        elif b[i + 1:i + 2] in (b'"', b"\\", b"/", b"b", b"f", b"n", b"r", b"t"):
            i += 2
        elif b[i + 1:i + 2] == b"u" and re.fullmatch(rb"[0-9a-fA-F]{4}", b[i + 2:min(i + 6, e)]):
            i += 6
        else:
            return i
    return -1


class _Walk:
    """one page: the levels the reader reads are parsed strictly, every other value is skipped by its brackets"""

    def __init__(self, b: bytes, page: int):
        self.b, self.page = b, page

    def fail(self, at: int, what: str):
        raise _PageError(f"page {self.page}, byte {at}: {what}")

    def ws(self, i: int) -> int:
        while i < len(self.b) and self.b[i] in _WS:
            i += 1
        return i

    def string(self, i: int) -> int:
        """b[i] is a quote: the end of the string (its raw inside checked)"""
        m = _STRING.match(self.b, i)
        if not m:
            self.fail(len(self.b), "a string is not closed")
        if _string_bad(self.b, i + 1, m.end() - 1) >= 0:
            self.fail(i + 1, "a string holds a bad escape or a raw byte < 0x20")
        return m.end()

    def skip(self, i: int) -> int:
        """b[i] opens an object or an array: the end of its matching close, which must be of its kind"""
        depth = 0
        for m in _STRUCT.finditer(self.b, i):
            t = m.group()
            if t in (b"{", b"["):
                depth += 1
            elif t in (b"}", b"]"):
                depth -= 1
                if depth == 0:
                    if t != (b"}" if self.b[i] == 0x7B else b"]"):
                        self.fail(m.start(), "unbalanced or mismatched brackets")
                    return m.end()
        self.fail(len(self.b), "unbalanced or mismatched brackets")

    def value(self, i: int):
        """a member value at b[i] (not whitespace) -> (kind, start, end): 'string' (the quotes included), 'object',
        'array' or 'scalar' (true, false, null or a number)"""
        c = self.b[i:i + 1]
        if c == b'"':
            return "string", i, self.string(i)
        if c in (b"{", b"["):
            return ("object" if c == b"{" else "array"), i, self.skip(i)
        j = i
        while j < len(self.b) and self.b[j] not in b',}]{["' and self.b[j] not in _WS:
            j += 1
        t = self.b[i:j]
        if not (t in (b"true", b"false", b"null") or _NUMBER.match(t)):
            self.fail(i, "malformed JSON")
        return "scalar", i, j

    def members(self, i: int) -> list:
        """the object opening at b[i] -> [(decoded name, kind, start, end)]"""
        out = []
        j = self.ws(i + 1)
        if self.b[j:j + 1] == b"}":
            return out
        while True:
            if self.b[j:j + 1] != b'"':
                self.fail(j, "malformed JSON")
            ne = self.string(j)
            name = json.loads(self.b[j:ne].decode("utf-8", "surrogatepass"))
            j = self.ws(ne)
            if self.b[j:j + 1] != b":":
                self.fail(j, "malformed JSON")
            j = self.ws(j + 1)
            if j >= len(self.b) or self.b[j] in b",}]":
                self.fail(j, "malformed JSON")
            kind, vb, ve = self.value(j)
            out.append((name, kind, vb, ve))
            j = self.ws(ve)
            if self.b[j:j + 1] == b"}":
                return out
            if self.b[j:j + 1] != b",":
                self.fail(j, "unbalanced or mismatched brackets" if self.b[j:j + 1] == b"]" else "malformed JSON")
            j = self.ws(j + 1)

    def elements(self, i: int) -> list:
        """the array opening at b[i], every element an object -> [(start, end)]"""
        out = []
        j = self.ws(i + 1)
        if self.b[j:j + 1] == b"]":
            return out
        while True:
            c = self.b[j:j + 1]
            if c != b"{":
                self.fail(j, "malformed JSON" if c in (b",", b"]") else "a hits.hits element is not an object")
            e = self.skip(j)
            out.append((j, e))
            j = self.ws(e)
            if self.b[j:j + 1] == b"]":
                return out
            if self.b[j:j + 1] != b",":
                self.fail(j, "a hits.hits element is not an object" if self.b[j:j + 1] != b"}" else "malformed JSON")
            j = self.ws(j + 1)


def _first(members, name):
    for m in members:
        if m[0] == name:
            return m
    return None


def _structure(b: bytes, page: int) -> None:
    """the whole page: no closing bracket without an opening one, every string closed, the brackets balanced"""
    depth = 0
    for m in _STRUCT.finditer(b):
        t = m.group()
        if t == b'"':
            raise _PageError(f"page {page}, byte {len(b)}: a string is not closed")
        if t in (b"{", b"["):
            depth += 1
        elif t in (b"}", b"]"):
            depth -= 1
            if depth < 0:
                raise _PageError(f"page {page}, byte {m.start()}: unbalanced or mismatched brackets")
    if depth:
        raise _PageError(f"page {page}, byte {len(b)}: unbalanced or mismatched brackets")


def index_page(b: bytes, page: int = 0):
    """one _search / _search/scroll response page -> (documents as bytes, n_hits, scroll_id or None, hits.total when
    exact else -1); ValueError names the page, and the hit or the byte offset"""
    b = bytes(b)
    _structure(b, page)
    w = _Walk(b, page)
    first = w.ws(0)
    if b[first:first + 1] != b"{":
        raise _PageError(f"page {page}: the top level is not an object")
    end = w.skip(first)
    if w.ws(end) != len(b):
        w.fail(end, "malformed JSON")
    top = w.members(first)
    scroll_id, total, status, hits_arr = None, -1, None, None
    timed_out = shards_failed = hits_bad = False
    seen = set()
    for name, kind, vb, ve in top:   # the nested levels in member order, the first of a repeated member
        if name in seen:
            continue
        seen.add(name)
        if name == "_shards" and kind == "object":
            f = _first(w.members(vb), "failed")
            shards_failed = f is not None and not (f[1] == "scalar" and _INTEGER.match(b[f[2]:f[3]]) and int(b[f[2]:f[3]]) == 0)
        elif name == "hits" and kind == "object":
            inner = w.members(vb)
            t = _first(inner, "total")
            if t is not None and t[1] == "scalar":
                text = b[t[2]:t[3]]
                total = int(text) if _INTEGER.match(text) and -2 ** 63 < int(text) < 2 ** 63 else -1
            elif t is not None and t[1] == "object":   # ES 7: {"value": n, "relation": "eq" | "gte"}
                tm = w.members(t[2])
                v, r = _first(tm, "value"), _first(tm, "relation")
                exact = v is not None and v[1] == "scalar" and _INTEGER.match(b[v[2]:v[3]]) is not None \
                    and -2 ** 63 < int(b[v[2]:v[3]]) < 2 ** 63
                if r is not None:
                    exact = exact and r[1] == "string" and json.loads(b[r[2]:r[3]].decode("utf-8", "surrogatepass")) == "eq"
                total = int(b[v[2]:v[3]]) if exact else -1
            h = _first(inner, "hits")
            if h is not None and not (h[1] == "scalar" and b[h[2]:h[3]] == b"null"):
                hits_arr = h if h[1] == "array" else None
                hits_bad = h[1] != "array"
    sid = _first(top, "_scroll_id")
    if sid is not None and sid[1] == "string":
        scroll_id = json.loads(b[sid[2]:sid[3]].decode("utf-8", "surrogatepass"))
    st = _first(top, "status")
    if st is not None and st[1] == "scalar" and _INTEGER.match(b[st[2]:st[3]]) and -2 ** 31 <= int(b[st[2]:st[3]]) < 2 ** 31:
        status = int(b[st[2]:st[3]])
    to = _first(top, "timed_out")
    timed_out = to is not None and to[1] == "scalar" and b[to[2]:to[3]] == b"true"
    if _first(top, "error") is not None:
        raise _PageError(f"page {page}: Elasticsearch returned an error" + (f" (status {status})" if status is not None else ""))
    if timed_out:
        raise _PageError(f"page {page}: the search timed out (timed_out is true)")
    if shards_failed:
        raise _PageError(f"page {page}: _shards.failed is not 0")
    if hits_bad:
        raise _PageError(f"page {page}: hits.hits is neither an array nor absent")
    hits = [w.members(hb) for hb, _ in w.elements(hits_arr[2])] if hits_arr is not None else []
    docs = []
    for k, hit in enumerate(hits):
        ids = [m for m in hit if m[0] == "_id"]
        if not ids or any(m[1] != "string" for m in ids):
            raise _PageError(f"page {page}, hit {k}: the hit has no string _id")
        if len(ids) > 1:
            raise _PageError(f"page {page}, hit {k}: a repeated _id")
        src = _first(hit, "_source")
        if src is None:
            raise _PageError(f"page {page}, hit {k}: the hit has no _source")
        if src[1] != "object":
            raise _PageError(f"page {page}, hit {k}: _source is not an object")
        docs.append((json.loads(b[ids[0][2]:ids[0][3]].decode("utf-8", "surrogatepass")), src[2], src[3]))
    out = bytearray()
    for k, (item, sb, se) in enumerate(docs):
        for m in re.finditer(rb'"(?:[^"\\]|\\.)*"|\\', b[sb:se], re.S):   # the source's strings, and backslashes outside them
            bad = sb + m.start() if m.group() == b"\\" else _string_bad(b, sb + m.start() + 1, sb + m.end() - 1)
            if bad >= 0:
                raise _PageError(f"page {page}, hit {k}, byte {bad}: a _source string holds a bad escape or a raw byte < 0x20")
        out += b'{"index":{"_id":' + json_string(item).encode("utf-8", "surrogatepass") + b'}}\n'
        out += _COMPACT.sub(lambda m: m.group(1) or b"", b[sb:se]) + b"\n"
    return bytes(out), len(docs), scroll_id, total


def index_from_pages(pages) -> tuple:
    """the model index read back from the pages of an Elasticsearch _search / scroll (each bytes), in order -> (bulk body,
    n_docs, total): one `{"index":{"_id":"<_id>"}}\\n<_source>\\n` per hit, the _id decoded and escaped as format_model
    escapes ids (json_string), _source with the whitespace outside strings dropped; total is the first page's hits.total
    when exact, else -1"""
    body, n_docs, total = bytearray(), 0, -1
    for p, page in enumerate(pages):
        docs, n, _, t = index_page(page, p)
        body += docs
        n_docs += n
        if p == 0:
            total = t
    return bytes(body), n_docs, total


# ---- the index written into Elasticsearch -----------------------------------------------------------------------------------
# URModel.save (URModel.scala:47-84) hands EsClient.hotSwap (EsClient.scala:257-362) the documents and esFields;
# createIndex (EsClient.scala:168-246) PUTs the mapping, saveToEs sends the _bulk requests, _aliases swaps the alias.  The
# bodies below restate the Scala string construction; index_fields, bulk_requests and bulk_item_statuses are the host mirrors
# of cco_index_write_*, written over json.
def index_mapping(fields: Sequence[str], ap, type_name: str) -> bytes:
    """the mapping createIndex PUTs for the fields (each as IndexWrite.fields / index_fields spell it: escaped), typed by
    getMappings (URAlgorithm.scala:955-967): its Map `++` order lets the date names override the event names and those
    the ranking names; every other field is a keyword.  The tail's unused "last" property closes the object without a
    trailing comma, so a field really named "last" is written twice, as the reference writes it."""
    types = index_field_types(ap)
    out = '{ "mappings": {    "%s": {      "properties": {            ' % type_name
    for f in fields:
        out += '"%s"    : {      "type": "%s"    },            ' % (f, types.get(f, "keyword"))
    out += '    "last": {      "type": "keyword"    }}}}}            '
    return out.encode("utf-8", "surrogatepass")


def index_field_types(ap) -> dict:
    """getMappings' types by escaped field name (index_mapping's rule): date names over event names over ranking names; a
    field not listed is a keyword"""
    names = ap.model_event_names()
    dates = list(dict.fromkeys(d for d in (ap.dateName, ap.availableDateName, ap.expireDateName) if d is not None))
    types = {**{rp.field_name(): "float" for rp in rankings_params(ap.rankings, names)}, **{e: "keyword" for e in names},
             **{d: "date" for d in dates}}
    return {json_string(k)[1:-1]: v for k, v in types.items()}


def mapping_additions(fields: Sequence[str], ap) -> bytes:
    """the body of PUT /<index>/_mapping/<type> that adds the fields (escaped, as IndexWrite.fields gives them) to a live
    index, typed as index_mapping types them"""
    types = index_field_types(ap)
    return ('{"properties":{' + ",".join('"%s":{"type":"%s"}' % (f, types.get(f, "keyword")) for f in fields)
            + "}}").encode("utf-8", "surrogatepass")


def alias_actions(alias: str, new_index: str, old_index: Optional[str] = None) -> bytes:
    """hotSwap's _aliases body: add the alias to the new index and, when the alias names an existing index, remove that
    index (remove_index)"""
    remove = ',{ "remove_index": { "index": "%s"}}' % old_index if old_index is not None else ""
    return ('{    "actions" : [        { "add":  { "index": "%s", "alias": "%s" } }        %s    ]}      '
            % (new_index, alias, remove)).encode("utf-8", "surrogatepass")


def new_index_name(index_name: str, now_ms: int) -> str:
    """hotSwap's new index: the alias, '_', the wall clock in milliseconds"""
    return f"{index_name}_{now_ms}"


class _Obj(list):
    """a JSON object as its (name, value) pairs in order, repeated names kept"""


def _pairs(text: bytes):
    return json.loads(text.decode("utf-8", "surrogatepass"), object_pairs_hook=_Obj)


def bulk_documents(body: bytes) -> list:
    """the documents of a model index body -> [(decoded _id, first byte, end byte, [(decoded name, value)])]"""
    body = bytes(body)
    if body and not body.endswith(b"\n"):
        raise ValueError("the body does not end in a newline")
    docs, at = [], 0
    lines = body.split(b"\n")[:-1] if body else []
    if len(lines) % 2:
        raise ValueError(f"the body has {len(lines)} lines: lines come in (action, source) pairs")
    for d in range(0, len(lines), 2):
        action, source = _pairs(lines[d]), _pairs(lines[d + 1])
        end = at + len(lines[d]) + len(lines[d + 1]) + 2
        if not isinstance(action, _Obj) or not isinstance(source, _Obj):
            raise ValueError(f"document {d // 2}: a line is not a JSON object")
        index = [v for k, v in action if k == "index"]
        ids = [v for k, v in index[0] if k == "_id"] if index and isinstance(index[0], _Obj) else []
        if not ids or not isinstance(ids[0], str):
            raise ValueError(f"document {d // 2}: the action line is not {{\"index\":{{...}}}} with a string \"_id\" member")
        docs.append((ids[0], at, end, source))
        at = end
    return docs


def index_fields(body: bytes) -> list:
    """esFields (URModel.scala:78) as cco_index_write_fields gives them: the distinct decoded member names of the document
    lines in first-appearance order, escaped as format_model escapes names; "id", which save adds to every document, last
    when no document line has it"""
    docs = bulk_documents(body)
    seen = dict.fromkeys(name for _, _, _, members in docs for name, _ in members)
    if docs and "id" not in seen:
        seen["id"] = None
    return [json_string(n)[1:-1] for n in seen]


def bulk_requests(body: bytes, max_docs: int, max_bytes: int) -> tuple:
    """elasticsearch-hadoop's batching of the documents into _bulk requests of at most max_docs documents and max_bytes
    bytes, a larger document alone -> (doc_begin, byte_begin), each with one entry past the last request"""
    docs = bulk_documents(body)
    doc_begin, byte_begin, n, size = [0], [0], 0, 0
    for d, (_, b, e, _) in enumerate(docs):
        if n and (n == max_docs or size + (e - b) > max_bytes):
            doc_begin.append(d)
            byte_begin.append(b)
            n = size = 0
        n += 1
        size += e - b
    if n:
        doc_begin.append(len(docs))
        byte_begin.append(docs[-1][2])
    return doc_begin, byte_begin


def bulk_item_statuses(response: bytes, ids: Sequence[str], action: str = "index") -> list:
    """one _bulk response for the documents of `ids` -> [(status, error.type, error.reason)] per item ("" where the item
    has no such string).  ValueError for the errors cco_index_write_response reports.  action="delete" reads the response
    to `delete` actions, whose items are {"delete":{...}} with the same members."""
    top = _pairs(bytes(response))
    if not isinstance(top, _Obj):
        raise ValueError("the top level is not an object")
    if any(k == "error" for k, _ in top):
        status = _first_pair(top, "status")
        ok = isinstance(status, int) and not isinstance(status, bool) and -2 ** 31 <= status < 2 ** 31
        raise ValueError("Elasticsearch returned an error" + (f" (status {status})" if ok else ""))
    items = _first_pair(top, "items", None)
    if not isinstance(items, list) or isinstance(items, _Obj):
        raise ValueError('the response has no "items" array')
    if any(not isinstance(x, _Obj) for x in items):
        raise ValueError("an items element is not an object")
    if len(items) != len(ids):
        raise ValueError(f"{len(items)} items for {len(ids)} documents")
    out = []
    for i, item in enumerate(items):
        if len(item) != 1 or item[0][0] != action or not isinstance(item[0][1], _Obj):
            raise ValueError(f"item {i}: the item is not {{\"{action}\":{{...}}}}")
        members = item[0][1]
        got_id = [v for k, v in members if k == "_id"]
        status = [v for k, v in members if k == "status"]
        if not got_id or any(not isinstance(v, str) for v in got_id):
            raise ValueError(f"item {i}: the item has no string _id")
        if len(got_id) > 1:
            raise ValueError(f"item {i}: a repeated _id")
        if not status:
            raise ValueError(f"item {i}: the item has no status")
        if len(status) > 1:
            raise ValueError(f"item {i}: a repeated status")
        if not (isinstance(status[0], int) and not isinstance(status[0], bool) and -2 ** 31 <= status[0] < 2 ** 31):
            raise ValueError(f"item {i}: the status is not a 32-bit integer")
        if got_id[0] != ids[i]:
            raise ValueError(f"item {i}: the item's _id is not the document's _id")
        err = _first_pair(members, "error")
        kind = reason = ""
        if isinstance(err, _Obj):
            t, r = _first_pair(err, "type"), _first_pair(err, "reason")
            kind = t if isinstance(t, str) else ""
            reason = r if isinstance(r, str) else ""
        out.append((status[0], kind, reason))
    return out


def _first_pair(pairs: list, name: str, default=None):
    for k, v in pairs:
        if k == name:
            return v
    return default


# ---- item properties refreshed in the live index ----------------------------------------------------------------------------
# The host mirror of cco_refresh_properties (include/cco_b200.h states the rule): fresh properties win, the correlator and
# computed ranking members of an old document are kept verbatim, every other old member is dropped.
@dataclass
class RefreshedIndex:
    """A refresh of the model index: body = the refreshed full index; delta = the changed and new documents (a bulk body);
    deletes = one {"delete":{"_id":...}} line per deleted document; changed / deleted = their old document numbers."""
    body: bytes
    delta: bytes
    deletes: bytes
    n_docs: int
    n_changed: int
    n_new: int
    n_deleted: int
    n_unchanged: int
    changed: list
    deleted: list

    @property
    def changed_ids(self) -> list:
        """the decoded ids of the changed documents (the first n_changed documents of the delta)"""
        lines = self.delta.split(b"\n")
        return [_pairs(lines[2 * k])[0][1][0][1] for k in range(self.n_changed)]

    @property
    def deleted_ids(self) -> list:
        return [_pairs(line)[0][1][0][1] for line in self.deletes.split(b"\n")[:-1]]


def _raw_members(line: bytes) -> list:
    """the members of a source line -> [(decoded name, raw name bytes between the quotes, trimmed raw value bytes)]"""
    w = _Walk(line, 0)
    i = w.ws(0)
    out = []
    j = w.ws(i + 1)
    if line[j:j + 1] == b"}":
        return out
    while True:
        name_b, ne = j, w.string(j)
        name = json.loads(line[j:ne].decode("utf-8", "surrogatepass"))
        j = w.ws(ne)
        _, vb, ve = w.value(w.ws(j + 1))
        out.append((name, line[name_b + 1:ne - 1], line[vb:ve]))
        j = w.ws(ve)
        if line[j:j + 1] == b"}":
            return out
        j = w.ws(j + 1)


def refresh_documents(body: bytes, correlators: Sequence[str], rankings: Sequence[str],
                      triples: Sequence[tuple[str, str, object]]) -> RefreshedIndex:
    """cco_refresh_properties on the host.  body: the current index (bulk_documents' grammar, an _id in two documents is a
    ValueError); correlators: the model's event names; rankings: the field names of the computed (popular, trending, hot,
    random) rankings; triples: the fresh (item, field, value) properties, values as property_json writes them, fields
    numbered by first appearance, the last triple of an (item, field) wins.  An old document becomes "id", its members
    named like a correlator, the item's fresh properties (not "id", not named like a computed ranking), its members named
    like a computed ranking; "id" and a member followed by one of the same name are skipped.  A document with neither a
    triple nor a kept member is deleted; an item with a triple and no document is new.  ValueError for a property named
    like a correlator."""
    body = bytes(body)
    docs = bulk_documents(body)
    corr, rank = set(correlators), set(rankings) - set(correlators)
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    for f in fields:
        if f in corr:
            raise ValueError(f'property field "{f}" is named like a correlator: a refresh keeps the correlator arrays')
    fnum = {f: k for k, f in enumerate(fields)}
    props: dict = {}
    for item, f, v in triples:
        props.setdefault(item, {})[f] = v
    enc = lambda s: s.encode("utf-8", "surrogatepass")

    def prop_bytes(item) -> bytes:
        d = props.get(item, {})
        return b"".join(b"," + enc(json_string(f)) + b":" + enc(property_json(d[f]))
                        for f in sorted(d, key=fnum.get) if f != "id" and f not in rank)

    def doc_bytes(item, src: bytes) -> bytes:
        return b'{"index":{"_id":' + enc(json_string(item)) + b"}}\n" + src + b"\n"

    first: dict = {}
    full, delta, deletes = bytearray(), bytearray(), bytearray()
    changed, deleted = [], []
    for d, (_, b, e, _) in enumerate(docs):
        index = _first_pair(_pairs(body[b:e].split(b"\n")[0]), "index")
        item = [v for k, v in index if k == "_id"][-1]   # of a repeated _id the last, as cco_rerank_model reads it
        if item in first:
            raise ValueError(f"document {d}: its _id is the _id of document {first[item]}")
        first[item] = d
        old = body[b:e].split(b"\n")[1]
        members = _raw_members(old)
        kept = [m for k, m in enumerate(members) if m[0] != "id" and all(m2[0] != m[0] for m2 in members[k + 1:])]
        cm = b"".join(b',"' + raw + b'":' + val for name, raw, val in kept if name in corr)
        rm = b"".join(b',"' + raw + b'":' + val for name, raw, val in kept if name in rank)
        if item not in props and not cm and not rm:
            deleted.append(d)
            deletes += b'{"delete":{"_id":' + enc(json_string(item)) + b"}}\n"
            continue
        src = b'{"id":' + enc(json_string(item)) + cm + prop_bytes(item) + rm + b"}"
        full += doc_bytes(item, src)
        if src != old:
            changed.append(d)
            delta += doc_bytes(item, src)
    new = [item for item in props if item not in first]
    for item in new:
        doc = doc_bytes(item, b'{"id":' + enc(json_string(item)) + prop_bytes(item) + b"}")
        full += doc
        delta += doc
    return RefreshedIndex(bytes(full), bytes(delta), bytes(deletes), len(docs) - len(deleted) + len(new), len(changed), len(new),
                          len(deleted), len(docs) - len(deleted) - len(changed), changed, deleted)
