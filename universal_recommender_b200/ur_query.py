"""URAlgorithm.buildQuery for user queries (Query.user set; item, itemSet and withRanks absent), item queries and
item-set queries (both below), restated from
src/main/scala/URAlgorithm.scala:195-267 (parameters), :563-767 (should / must / must_not / sort), :795-839
(getBiasedRecentUserActions) and :872-953 (date filters).  The query is the text the reference posts to Elasticsearch;
scoring stays with Elasticsearch.

plan() renders what every user's query shares (the fragments CcoContext.user_queries hands to the device);
user_queries() is the host mirror over events.read_export's output, the whole body built here.

Quirks of the reference, kept on purpose:
  * the per-name history limit is DefaultIndicatorParams().maxItemsPerUser = 100 whenever `eventNames` is given, even
    next to `indicators`, and otherwise the indicator's maxItemsPerUser or 500 (:213-224); a query event name without an
    entry raises KeyError, as the reference throws NoSuchElementException;
  * maxQueryEvents with indicators is the sum of their maxItemsPerUser (100 each by default) times 10 (:202-210), and
    only the first maxQueryEvents - 1 *names* get a terms clause: the slice is over names, not events (:575, :665);
  * the should / must choice tests the algorithm's userBias, not the query's (:572, :660); the boost itself is the
    query's userBias, else the algorithm's, written only when b > 0 and b != 1 (:823-824);
  * the metadata signs are inverted between query and engine.json: boosts are query fields with bias > 0 plus params
    fields with bias < 0, filters the other way round, exclusions bias == 0 of both (:844-867), each list distinct;
  * a dateRange whose `after` or `before` is given writes one range clause even when the value is "", and leaves the
    empty bound out (:878-918); otherwise availableDateName and expireDateName both set give the lte / gt pair against
    currentDate, the query's or "now" as Joda's DateTime.toDateTimeISO.toString in UTC (yyyy-MM-ddTHH:mm:ss.SSSZ)
    [RECALL: Joda 2.9];
  * the history is the latest `limit` events of each name, prepended one by one (oldest first) and then `distinct`: an
    item stays at its oldest position among them; a name without history still writes [] (:826-836);
  * the blacklist is the targets of *all* the user's events of the query names that are also blacklistEvents (default:
    the first model event name; [] means none), newest first, then blacklistItems, distinct (:742-767);
  * sort is [] under recsModel "collabFiltering" (:730-738).
Rendering is json4s 3.2.x compact(render(...)) [RECALL]: a Float is widened to Double and printed by Double.toString (a
bias of 1.05 prints 1.0499999523162842, 2 prints 2.0), ints print plainly, and strings escape '"' and '\\', use the short
forms \\b \\f \\n \\r \\t, and write every other code point below U+0020, in U+0080..U+009F and in U+2000..U+20FF as
\\u%04x in lowercase hex.  Any valid escaping gives Elasticsearch the same query; the rule is fixed so that bytes compare.
Date values and sort field names are interpolated into JSON text and parsed again by the reference; here they are written
as escaped strings, the same text for every value that needs no escape.
LEventStore.findByEntity is taken to read every event of the user, unlimited, latest first [RECALL: PredictionIO 0.12].

Deviations:
  * the history is the log's training events (entityType "user" -> targetEntityType "item"); findByEntity has no
    target-type filter, so events aimed at other entity types, which the reference would read, are not read here;
  * where the reference would throw on a target-less event of a query name, no such event exists here.

Item queries (Query.item set; user, itemSet and withRanks absent): item_plan() renders what every item's query shares (the
fragments CcoContext.item_queries hands to the device); item_queries() is the host mirror over a model index body (what
CcoContext.format_model / rerank_model write).  Quirks of the reference, kept on purpose:
  * history clauses are still written: getBiasedRecentUserActions (:795-839) evaluates query.user.get inside its try, the
    NoSuchElementException is caught, and every query event name (query eventNames, else the model names) gets a terms
    clause with [] -- the first maxQueryEvents - 1 names (:624, :690), in should with the user boost or in must with
    "boost":0 when the algorithm's userBias < 0, as plan() renders them for a user without history.  No event is read, so
    indicatorParams is never consulted: a query event name without an entry raises nothing here;
  * similar items (getBiasedSimilarItems, :770-792) are one clause per *model* event name, not per query eventName; the
    document is EsClient.getSource by _id (EsClient.scala:394-442), and a missing document (a 404 reaches Map.empty
    through the caught ResponseException [RECALL: ES 5 low-level client]) or a source without members (m.nonEmpty, :776)
    adds no clause at all, while a document without the name's field writes {"terms":{"<name>":[]}} (an item with only
    $set events has such a document);
  * a list with size <= maxQueryEvents is kept whole, a longer one keeps its first maxQueryEvents - 1 (:782); elements
    keep the document's order, no distinct;
  * the should / must choice tests the algorithm's itemBias (:630, :695-697); the boost is the query's itemBias, else the
    algorithm's, written only when > 0 and != 1, a Float widened to Double (:777-779); in must it is "boost":0;
  * clause order: should = history, similar items, boosted metadata, constant_score (:653, :681); must = history filter,
    similar-items filter, filtering metadata, date filters (:703-709);
  * must_not ids (:741-767): blacklistItems, then the item itself unless query.returnSelf.getOrElse(ap.returnSelf)
    (default false, :237, :759), then distinct -- an item already in blacklistItems is not repeated;
  * getSource casts the source unchecked to Map[String, List[String]] (EsClient.scala:435): a queried document whose
    model-name member is not an array of strings makes that query fail; here it raises, naming the document.
Deviation: the reference's GET for an empty item id addresses the type, not a document; here "" is looked up as any id.

Item-set queries (Query.itemSet set: "shopping cart" recommendations; user, item and withRanks absent): item_set_plan()
renders what every set's query shares (the fragments CcoContext.item_set_queries hands to the device); item_set_queries()
is the host mirror over a list of sets.  Nothing is read: the set is the caller's.  Quirks of the reference, kept on purpose:
  * history clauses are still written, empty, exactly as for item queries (getBiasedRecentUserActions, :795-839): the
    first maxQueryEvents - 1 query event names (query eventNames, else the model names), in should with the user boost or
    in must with "boost":0 when the algorithm's userBias < 0; indicatorParams is never consulted;
  * no similar items (query.item is empty, :630, :695);
  * the set clause is BoostableCorrelators(modelEventNames.head, itemSet, query.itemSetBias) (:640-648): its field is the
    *first model event name*, not a query eventName, and with no model event name the reference's .head throws (here
    ValueError); its elements are the set exactly as given -- order and repeats kept, no maxQueryEvents slice;
  * its boost is query.itemSetBias only, a Float widened to Double, with no algorithm-level fallback (Engine.scala:38's
    comment says otherwise) and no > 0 / != 1 test: None writes no "boost", 1 writes "boost":1.0, -1 writes "boost":-1.0
    in should; boost.getOrElse(1f) != 0f (:656-659) drops the clause for 0 and -0.0; an empty set ("itemSet": [] is
    Some(Nil)) still writes {"terms":{"<name>":[]}};
  * clause order: should = history, boosted metadata, the set clause, constant_score (:653, :681); must = history filter,
    filtering metadata, date filters (:703-709); the set clause never goes to must;
  * must_not ids (getExcludedItems, :741-767): distinct(blacklistItems ++ itemSet) -- the blacklist first, each once, then
    each set element not among them and not earlier in the set: a repeated element is written twice in the set clause and
    once here.

Mixed queries (any subset of Query.user, Query.item and Query.itemSet in one query; withRanks absent): mixed_plan()
renders what every row's query shares (the fragments CcoContext.mixed_queries hands to the device); mixed_queries() is the
host mirror over an event export, an index body and three columns in which an absent member is None.  buildQuery composes
the three shapes above; quirks of the reference, kept on purpose:
  * history (getBiasedRecentUserActions, :795-839): a row with a user gets that user's lists, exactly as a user query (the
    per-name limits, latest first then reversed, distinct); a row without one evaluates query.user.get, the
    NoSuchElementException is caught, and each of the first maxQueryEvents - 1 query names still writes [] -- as an
    unknown user does.  Per-name limits are consulted exactly when the batch has a user column (mixed_plan's with_limits):
    then a query event name without an indicatorParams entry raises KeyError, as plan() does, even for rows without a user;
  * should (:653): the history (the algorithm's userBias >= 0), the similar items (the algorithm's itemBias >= 0; one
    clause per model name from the item's document, sliced, none for a missing document or a {} source), the boosted
    metadata, the set clause (the first model name, the set as given, boost = the query's itemSetBias only, dropped for 0
    and -0.0, [] for an empty set, nothing for an absent one), constant_score;
  * must (:703-709): the history filter (userBias < 0), the similar-items filter (itemBias < 0), the filtering metadata,
    the date filters;
  * must_not ids (getExcludedItems, :741-767): distinct(userBlacklisted ++ blacklistItems :+ item (unless returnSelf) ++
    itemSet), where userBlacklisted is the items of the user's events of blacklisted query names, latest first; distinct
    keeps each id's first position across the four sources;
  * "ItemSets should not be mixed with user or item queries" (:641-644) is only a log line: the query is built anyway.
Query files (a batchpredict input: one Query object per line, each with its own template): query_file() is the host
mirror of CcoContext.query_file, mixed_queries() for each line as a one-row batch; the extraction rules are listed above
parse_query_line().
Out of scope: withRanks (it only changes how results are read).
"""
from __future__ import annotations

import datetime as _dt
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from .ur_model import java_double, rankings_params

MAX_QUERY_EVENTS = 100          # DefaultURAlgoParams.MaxQueryEvents (URAlgorithm.scala:57)
MAX_EVENTS_PER_EVENT_TYPE = 500
NUM_RESULTS = 20
CONSTANT_SCORE = '{"constant_score":{"filter":{"match_all":{}},"boost":0}}'


@dataclass
class Field:
    """Engine.scala:53-58: bias > 0 boosts, < 0 filters, 0 excludes (signs inverted for engine.json fields)"""
    name: str
    values: Sequence[str]
    bias: float

    @staticmethod
    def from_json(d: dict) -> "Field":
        return Field(d["name"], list(d["values"]), float(d["bias"]))


@dataclass
class DateRange:
    """Engine.scala:61-65"""
    name: str
    before: Optional[str] = None
    after: Optional[str] = None


@dataclass
class UserQuery:
    """the user-query members of Query (Engine.scala:32-50); the user itself is the record's"""
    userBias: Optional[float] = None
    fields: Optional[Sequence[Field]] = None
    currentDate: Optional[str] = None
    dateRange: Optional[DateRange] = None
    blacklistItems: Optional[Sequence[str]] = None
    num: Optional[int] = None
    from_: Optional[int] = None
    eventNames: Optional[Sequence[str]] = None

    @staticmethod
    def from_json(d: dict) -> "UserQuery":
        dr = d.get("dateRange")
        return UserQuery(d.get("userBias"), None if d.get("fields") is None else [Field.from_json(f) for f in d["fields"]],
                         d.get("currentDate"), None if dr is None else DateRange(dr["name"], dr.get("before"), dr.get("after")),
                         d.get("blacklistItems"), d.get("num"), d.get("from"), d.get("eventNames"))


@dataclass
class ItemQuery(UserQuery):
    """the item-query members of Query (Engine.scala:32-50); the item itself is the record's"""
    itemBias: Optional[float] = None
    returnSelf: Optional[bool] = None

    @staticmethod
    def from_json(d: dict) -> "ItemQuery":
        u = UserQuery.from_json(d)
        return ItemQuery(**{k: getattr(u, k) for k in u.__dataclass_fields__}, itemBias=d.get("itemBias"), returnSelf=d.get("returnSelf"))


@dataclass
class ItemSetQuery(UserQuery):
    """the item-set-query members of Query (Engine.scala:32-50); the set itself is the record's"""
    itemSetBias: Optional[float] = None

    @staticmethod
    def from_json(d: dict) -> "ItemSetQuery":
        u = UserQuery.from_json(d)
        return ItemSetQuery(**{k: getattr(u, k) for k in u.__dataclass_fields__}, itemSetBias=d.get("itemSetBias"))


@dataclass
class MixedQuery(ItemQuery):
    """the template members of Query (Engine.scala:32-50) for rows that may have a user, an item and an item set: the union
    of UserQuery, ItemQuery and ItemSetQuery; the user, item and set themselves are the row's"""
    itemSetBias: Optional[float] = None

    @staticmethod
    def from_json(d: dict) -> "MixedQuery":
        i = ItemQuery.from_json(d)
        return MixedQuery(**{k: getattr(i, k) for k in i.__dataclass_fields__}, itemSetBias=d.get("itemSetBias"))


def f32(x: float) -> float:
    return float(np.float32(x))


def json_string(s: str) -> str:
    """json4s 3.2's quote, quotes included"""
    out = ['"']
    for ch in s:
        c = ord(ch)
        if ch in '"\\':
            out.append("\\" + ch)
        elif ch in "\b\f\n\r\t":
            out.append({"\b": "\\b", "\f": "\\f", "\n": "\\n", "\r": "\\r", "\t": "\\t"}[ch])
        elif c < 0x20 or 0x80 <= c < 0xA0 or 0x2000 <= c < 0x2100:
            out.append("\\u%04x" % c)
        else:
            out.append(ch)
    out.append('"')
    return "".join(out)


def jfloat(x: float) -> str:
    """a Scala Float rendered by json4s: widened to Double, Double.toString"""
    return java_double(f32(x))


def iso_utc(ms: int) -> str:
    """Joda DateTime.toDateTimeISO.toString in UTC"""
    t = _dt.datetime(1970, 1, 1, tzinfo=_dt.timezone.utc) + _dt.timedelta(milliseconds=int(ms))
    return t.strftime("%Y-%m-%dT%H:%M:%S.") + "%03dZ" % (t.microsecond // 1000)


def terms(name: str, values: Sequence[str], boost: Optional[str]) -> str:
    b = "" if boost is None else ',"boost":' + boost
    return '{"terms":{' + json_string(name) + ":[" + ",".join(json_string(v) for v in values) + "]" + b + "}}"


def _distinct(xs):
    out = []
    for x in xs:
        if x not in out:
            out.append(x)
    return out


@dataclass
class Plan:
    """what every user's query shares"""
    names: list                 # query event names
    limits: list                # per name
    blacklist: list             # blacklistEvents
    boost: Optional[str]        # the history boost's text, None: no "boost"
    in_must: bool               # the algorithm's userBias < 0
    n_history: int              # names with a terms clause: maxQueryEvents - 1, clamped
    head: str                   # {"from":F,"size":N
    should: str                 # should elements after the history
    must: str                   # must elements after the history
    must_not: str               # must_not elements after the ids clause
    sort: str
    blacklist_items: list = field(default_factory=list)
    boosted: str = ""           # the boosted metadata clauses of `should`, without the constant_score clause


def query_event_limits(ap, names: Sequence[str]) -> list:
    """indicatorParams(action).maxItemsPerUser (URAlgorithm.scala:213-224)"""
    if ap.eventNames is not None:
        table = {n: MAX_QUERY_EVENTS for n in ap.eventNames}
    elif ap.indicators:
        table = {i.name: i.maxItemsPerUser or MAX_EVENTS_PER_EVENT_TYPE for i in ap.indicators}
    else:
        raise ValueError('Must have either "eventNames" or "indicators" in algorithm parameters.')
    out = []
    for n in names:
        if n not in table:
            raise KeyError(f"key not found: {n}")   # NoSuchElementException
        out.append(table[n])
    return out


def max_query_events(ap) -> int:
    if not ap.indicators:
        return ap.maxQueryEvents if ap.maxQueryEvents is not None else MAX_QUERY_EVENTS
    return sum(i.maxItemsPerUser or MAX_QUERY_EVENTS for i in ap.indicators) * 10


def plan(ap, query: UserQuery, now_ms: Optional[int] = None, with_limits: bool = True) -> Plan:
    """with_limits=False: no per-name limits (an item query reads no history, so indicatorParams is never consulted)"""
    model_names = ap.model_event_names()
    names = list(query.eventNames) if query.eventNames is not None else list(model_names)
    limits = query_event_limits(ap, names) if with_limits else []
    blacklist = list(ap.blacklistEvents) if ap.blacklistEvents is not None else list(model_names[:1])
    algo_bias = f32(ap.userBias) if ap.userBias is not None else 1.0
    b = f32(query.userBias) if query.userBias is not None else algo_bias
    boost = java_double(b) if b > 0 and b != 1 else None
    n_history = max(0, min(max_query_events(ap) - 1, len(names)))
    size = query.num if query.num is not None else (ap.num if ap.num is not None else NUM_RESULTS)
    head = '{"from":%d,"size":%d' % (query.from_ or 0, size)
    qf, pf = list(query.fields or []), list(ap.fields or [])
    boosted = _distinct([(f.name, list(f.values), f32(f.bias)) for f in [f for f in qf if f32(f.bias) > 0] + [f for f in pf if f32(f.bias) < 0]])
    filters = _distinct([(f.name, list(f.values)) for f in [f for f in qf if f32(f.bias) < 0] + [f for f in pf if f32(f.bias) > 0]])
    excluded = _distinct([(f.name, list(f.values)) for f in [f for f in qf if f32(f.bias) == 0] + [f for f in pf if f32(f.bias) == 0]])
    should = [terms(n, v, java_double(x)) for n, v, x in boosted] + [CONSTANT_SCORE]
    must = [terms(n, v, "0") for n, v in filters] + date_filters(ap, query, now_ms)
    must_not = ['{"terms":{' + json_string(n) + ":[" + ",".join(json_string(x) for x in v) + "]}}" for n, v in excluded]
    if ap.recsModel in ("all", "backfill"):
        ranks = [rp.field_name() for rp in rankings_params(ap.rankings, model_names)]
        sort = "[" + ",".join(['{"_score":{"order":"desc"}}'] + ["{" + json_string(r) + ':{"unmapped_type":"double","order":"desc"}}'
                                                                  for r in ranks]) + "]"
    else:
        sort = "[]"
    return Plan(names, limits, blacklist, boost, algo_bias < 0, n_history, head, ",".join(should), ",".join(must), ",".join(must_not),
                sort, list(query.blacklistItems or []), ",".join(should[:-1]))


def _range(name: str, bounds: Sequence[tuple[str, str]]) -> str:
    return ('{"constant_score":{"filter":{"range":{' + json_string(name) + ":{" + ",".join(json_string(k) + ":" + json_string(v) for k, v in bounds)
            + '}}},"boost":0}}')


def date_filters(ap, query: UserQuery, now_ms: Optional[int]) -> list:
    """getFilteringDateRange (URAlgorithm.scala:872-953)"""
    dr = query.dateRange
    if dr is not None and (dr.after is not None or dr.before is not None):
        bounds = []
        if dr.after:
            bounds.append(("gt", dr.after))
        if dr.before:
            bounds.append(("lt", dr.before))
        return [_range(dr.name, bounds)]
    if ap.availableDateName is not None and ap.expireDateName is not None:
        if query.currentDate is not None:
            current = query.currentDate
        else:
            if now_ms is None:
                raise ValueError("the available / expire date filter needs now_ms or the query's currentDate")
            current = iso_utc(now_ms)
        return [_range(ap.availableDateName, [("lte", current)]), _range(ap.expireDateName, [("gt", current)])]
    return []


def user_history(recent: Sequence[tuple[str, str]], p: Plan) -> tuple[list, list]:
    """getBiasedRecentUserActions + getExcludedItems on one user's events [(event name, item)], latest first:
    -> ([items per query name], blacklist)"""
    hist = []
    for name, limit in zip(p.names, p.limits):
        items: list = []
        for ev, item in recent:
            if ev == name and len(items) < limit:
                items = [item] + items
        hist.append(list(dict.fromkeys(items)))
    black = [item for ev, item in recent if ev in p.blacklist] + list(p.blacklist_items)
    return hist, list(dict.fromkeys(black))


def render(p: Plan, hist: Sequence[Sequence[str]], black: Sequence[str]) -> str:
    """buildQuery's document (URAlgorithm.scala:599-610) in json4s' compact rendering"""
    h = [terms(n, items, "0" if p.in_must else p.boost) for n, items in zip(p.names[:p.n_history], hist)]
    should = ([] if p.in_must else h) + [p.should]
    must = (h if p.in_must else []) + ([p.must] if p.must else [])
    must_not = ['{"ids":{"values":[' + ",".join(json_string(x) for x in black) + '],"boost":0}}'] + ([p.must_not] if p.must_not else [])
    return (p.head + ',"query":{"bool":{"should":[' + ",".join(should) + '],"must":[' + ",".join(must) + '],"must_not":['
            + ",".join(must_not) + '],"minimum_should_match":1}},"sort":' + p.sort + "}")


def user_queries(events, ap, query: Optional[UserQuery] = None, users: Optional[Sequence[str]] = None, now_ms: Optional[int] = None,
                 header: str = "{}"):
    """the host mirror of CcoContext.user_queries over events.read_export's output (its training events, line order):
    -> (body, offsets), or (body, offsets, users) for users=None (every user with a training event of a query event
    name, in order of their first such line)"""
    p = plan(ap, query or UserQuery(), now_ms)
    qn = set(p.names)
    by_user: dict = {}
    for line, (u, ev, item, t) in enumerate(events.events):
        if ev in qn:
            by_user.setdefault(u, []).append((t, line, ev, item))
    who = list(by_user) if users is None else list(users)
    recs = []
    for u in who:
        recent = [(ev, item) for _, _, ev, item in sorted(by_user.get(u, []), key=lambda x: (-x[0], -x[1]))]
        hist, black = user_history(recent, p)
        recs.append((header + "\n" + render(p, hist, black) + "\n").encode("utf-8", "surrogatepass"))
    offsets = np.zeros(len(recs) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in recs], out=offsets[1:])
    body = b"".join(recs)
    return (body, offsets) if users is not None else (body, offsets, who)


@dataclass
class ItemPlan:
    """what every item's query shares"""
    names: list                 # model event names: one similar-items clause each
    max_query_events: int       # slice bound: a longer list keeps its first max_query_events - 1
    in_must: bool               # the algorithm's itemBias < 0
    boost: Optional[str]        # the similar items' boost text, None: no "boost"
    exclude_self: bool          # not returnSelf
    head: str
    should_head: str            # the empty history clauses when they go to should, else ""
    should: str
    must_head: str              # the same in must
    must: str
    must_not: str
    sort: str
    blacklist_items: list = field(default_factory=list)


def item_plan(ap, query: Optional[ItemQuery] = None, now_ms: Optional[int] = None) -> ItemPlan:
    query = query or ItemQuery()
    p = plan(ap, query, now_ms, with_limits=False)
    history = ",".join(terms(n, [], "0" if p.in_must else p.boost) for n in p.names[:p.n_history])
    algo_bias = f32(ap.itemBias) if ap.itemBias is not None else 1.0
    b = f32(query.itemBias) if query.itemBias is not None else algo_bias
    return_self = query.returnSelf if query.returnSelf is not None else bool(ap.returnSelf)
    return ItemPlan(list(ap.model_event_names()), max_query_events(ap), algo_bias < 0, java_double(b) if b > 0 and b != 1 else None,
                    not return_self, p.head, "" if p.in_must else history, p.should, history if p.in_must else "", p.must,
                    p.must_not, p.sort, p.blacklist_items)


def index_documents(index_body: bytes) -> list:
    """a model index bulk body -> [(decoded _id, source dict)] in body order; json's last-member-wins for repeated names"""
    if not index_body:
        return []
    if not index_body.endswith(b"\n"):
        raise ValueError("the body does not end in a newline")
    import json
    lines = index_body[:-1].decode("utf-8", "surrogatepass").split("\n")
    if len(lines) % 2:
        raise ValueError(f"the body has {len(lines)} lines: lines come in (action, source) pairs")
    docs, seen = [], {}
    for d in range(len(lines) // 2):
        action, source = json.loads(lines[2 * d]), json.loads(lines[2 * d + 1])
        if not isinstance(action, dict) or list(action) != ["index"] or not isinstance(action["index"], dict) \
                or not isinstance(action["index"].get("_id"), str):
            raise ValueError(f"document {d}: the action line is not {{\"index\":{{...}}}} with a string \"_id\" member")
        if not isinstance(source, dict):
            raise ValueError(f"document {d}: the source line is not a JSON object")
        i = action["index"]["_id"]
        if i in seen:
            raise ValueError(f"document {d}: its _id is the _id of document {seen[i]}")
        seen[i] = d
        docs.append((i, source))
    return docs


def similar_items(p: ItemPlan, d: int, source: dict) -> list:
    """getBiasedSimilarItems on one document's source -> [terms clause per model name]"""
    out = []
    for n in p.names:
        v = source.get(n, [])
        if not isinstance(v, list) or not all(isinstance(x, str) for x in v):
            raise ValueError(f'document {d}: its "{n}" member is not an array of strings')
        v = v if len(v) <= p.max_query_events else v[:p.max_query_events - 1]
        out.append(terms(n, v, "0" if p.in_must else p.boost))
    return out


def item_render(p: ItemPlan, similar: Sequence[str], excluded: Sequence[str]) -> str:
    """buildQuery's document for an item query (URAlgorithm.scala:594-606) in json4s' compact rendering"""
    should = [x for x in [p.should_head] if x] + ([] if p.in_must else list(similar)) + [x for x in [p.should] if x]
    must = [x for x in [p.must_head] if x] + (list(similar) if p.in_must else []) + [x for x in [p.must] if x]
    must_not = ['{"ids":{"values":[' + ",".join(json_string(x) for x in excluded) + '],"boost":0}}'] + ([p.must_not] if p.must_not else [])
    return (p.head + ',"query":{"bool":{"should":[' + ",".join(should) + '],"must":[' + ",".join(must) + '],"must_not":['
            + ",".join(must_not) + '],"minimum_should_match":1}},"sort":' + p.sort + "}")


def item_queries(index_body: bytes, ap, query: Optional[ItemQuery] = None, items: Optional[Sequence[str]] = None,
                 now_ms: Optional[int] = None, header: str = "{}"):
    """the host mirror of CcoContext.item_queries over a model index bulk body -> (body, offsets), or (body, offsets, items)
    for items=None (every document, in body order)"""
    p = item_plan(ap, query, now_ms)
    docs = index_documents(bytes(index_body))
    by_id = {i: (d, src) for d, (i, src) in enumerate(docs)}
    who = [i for i, _ in docs] if items is None else list(items)
    recs = []
    for it in who:
        d, src = by_id.get(it, (-1, {}))
        similar = similar_items(p, d, src) if src else []
        excluded = _distinct(list(p.blacklist_items) + ([it] if p.exclude_self else []))
        recs.append((header + "\n" + item_render(p, similar, excluded) + "\n").encode("utf-8", "surrogatepass"))
    offsets = np.zeros(len(recs) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in recs], out=offsets[1:])
    body = b"".join(recs)
    return (body, offsets) if items is not None else (body, offsets, who)


@dataclass
class ItemSetPlan:
    """what every item set's query shares"""
    name: Optional[str]         # the set clause's field: the first model event name
    with_set: bool              # itemSetBias != 0: the set clause is written
    boost: Optional[str]        # the set clause's boost text (the query's itemSetBias), None: no "boost"
    head: str
    should_head: str            # the empty history clauses when they go to should, then the boosted metadata
    should_tail: str            # the constant_score clause
    must: str                   # the empty history clauses when they go to must, the filtering metadata, the date filters
    must_not: str
    sort: str
    blacklist_items: list = field(default_factory=list)


def item_set_plan(ap, query: Optional[ItemSetQuery] = None, now_ms: Optional[int] = None) -> ItemSetPlan:
    query = query or ItemSetQuery()
    model_names = ap.model_event_names()
    if not model_names:
        raise ValueError("an item-set query needs a model event name: the set clause's field is the first one")
    p = plan(ap, query, now_ms, with_limits=False)
    history = [terms(n, [], "0" if p.in_must else p.boost) for n in p.names[:p.n_history]]
    b = None if query.itemSetBias is None else f32(query.itemSetBias)
    should_head = ([] if p.in_must else history) + ([p.boosted] if p.boosted else [])
    must = (history if p.in_must else []) + ([p.must] if p.must else [])
    return ItemSetPlan(model_names[0], b is None or b != 0, None if b is None else java_double(b), p.head, ",".join(should_head),
                       CONSTANT_SCORE, ",".join(must), p.must_not, p.sort, p.blacklist_items)


def item_set_render(p: ItemSetPlan, item_set: Sequence[str]) -> str:
    """buildQuery's document for an item-set query (URAlgorithm.scala:594-606) in json4s' compact rendering"""
    should = [x for x in [p.should_head] if x] + ([terms(p.name, item_set, p.boost)] if p.with_set else []) + [x for x in [p.should_tail] if x]
    excluded = list(dict.fromkeys(list(p.blacklist_items) + list(item_set)))   # distinct, first position
    must_not = ['{"ids":{"values":[' + ",".join(json_string(x) for x in excluded) + '],"boost":0}}'] + ([p.must_not] if p.must_not else [])
    return (p.head + ',"query":{"bool":{"should":[' + ",".join(should) + '],"must":[' + p.must + '],"must_not":['
            + ",".join(must_not) + '],"minimum_should_match":1}},"sort":' + p.sort + "}")


def item_set_queries(sets: Sequence[Sequence[str]], ap, query: Optional[ItemSetQuery] = None, now_ms: Optional[int] = None,
                     header: str = "{}"):
    """the host mirror of CcoContext.item_set_queries: one record per set, in order -> (body, offsets)"""
    p = item_set_plan(ap, query, now_ms)
    recs = [(header + "\n" + item_set_render(p, list(s)) + "\n").encode("utf-8", "surrogatepass") for s in sets]
    offsets = np.zeros(len(recs) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in recs], out=offsets[1:])
    return b"".join(recs), offsets


@dataclass
class MixedPlan:
    """what every row of a mixed batch shares: the user-query plan (history, blacklist names, fragments), the item-query
    plan (similar items) and the set clause"""
    user: Plan
    item: ItemPlan
    set_name: Optional[str]     # the first model event name, None without one
    with_set: bool              # itemSetBias != 0: the set clause is written for a row with a set
    set_boost: Optional[str]    # the query's itemSetBias text, None: no "boost"


def mixed_plan(ap, query: Optional[MixedQuery] = None, now_ms: Optional[int] = None, with_limits: bool = True) -> MixedPlan:
    """with_limits: consult the per-name limits (indicatorParams), as plan() does; pass whether the batch has a user column,
    so a batch without users never raises KeyError for a query event name without an entry"""
    query = query or MixedQuery()
    model_names = ap.model_event_names()
    b = None if query.itemSetBias is None else f32(query.itemSetBias)
    return MixedPlan(plan(ap, query, now_ms, with_limits), item_plan(ap, query, now_ms), model_names[0] if model_names else None,
                     b is None or b != 0, None if b is None else java_double(b))


def mixed_render(p: MixedPlan, hist: Sequence[Sequence[str]], similar: Sequence[str], item_set: Optional[Sequence[str]],
                 excluded: Sequence[str]) -> str:
    """buildQuery's document for a row with any subset of user, item and item set (URAlgorithm.scala:594-606) in json4s'
    compact rendering: hist = the history list of each of the first n_history names, similar = the rendered similar-items
    clauses, item_set = None for a row without a set"""
    u, i = p.user, p.item
    h = [terms(n, items, "0" if u.in_must else u.boost) for n, items in zip(u.names[:u.n_history], hist)]
    if item_set is not None and p.with_set and p.set_name is None:
        raise ValueError("an item-set query needs a model event name: the set clause's field is the first one")
    set_clause = [terms(p.set_name, item_set, p.set_boost)] if item_set is not None and p.with_set else []
    should = ([] if u.in_must else h) + ([] if i.in_must else list(similar)) + ([u.boosted] if u.boosted else []) + set_clause + [CONSTANT_SCORE]
    must = (h if u.in_must else []) + (list(similar) if i.in_must else []) + ([u.must] if u.must else [])
    must_not = ['{"ids":{"values":[' + ",".join(json_string(x) for x in excluded) + '],"boost":0}}'] + ([u.must_not] if u.must_not else [])
    return (u.head + ',"query":{"bool":{"should":[' + ",".join(should) + '],"must":[' + ",".join(must) + '],"must_not":['
            + ",".join(must_not) + '],"minimum_should_match":1}},"sort":' + u.sort + "}")


def mixed_queries(events, index_body: Optional[bytes], ap, query: Optional[MixedQuery] = None, users: Optional[Sequence] = None,
                  items: Optional[Sequence] = None, item_sets: Optional[Sequence] = None, now_ms: Optional[int] = None,
                  header: str = "{}"):
    """the host mirror of CcoContext.mixed_queries: one record per row -> (body, offsets).  users, items: a str or None per
    row; item_sets: a sequence of str or None per row; a column that is None has no member in any row.  events:
    events.read_export's output (None when no row has a user); index_body: a model index bulk body (None when no row has an
    item)."""
    cols = [c for c in (users, items, item_sets) if c is not None]
    n = len(cols[0]) if cols else 0
    if any(len(c) != n for c in cols):
        raise ValueError("the user, item and item-set columns have different lengths")
    p = mixed_plan(ap, query, now_ms, with_limits=users is not None)
    by_user: dict = {}
    if users is not None and any(x is not None for x in users):
        if events is None:
            raise ValueError("a row has a user: its history needs the events")
        qn = set(p.user.names)
        for line, (u, ev, item, t) in enumerate(events.events):
            if ev in qn:
                by_user.setdefault(u, []).append((t, line, ev, item))
    by_id: dict = {}
    if items is not None and any(x is not None for x in items):
        if index_body is None:
            raise ValueError("a row has an item: its similar items need an index body")
        by_id = {i: (d, src) for d, (i, src) in enumerate(index_documents(bytes(index_body)))}
    recs = []
    for r in range(n):
        u = None if users is None else users[r]
        it = None if items is None else items[r]
        s = None if item_sets is None or item_sets[r] is None else list(item_sets[r])
        if u is not None:
            recent = [(ev, item) for _, _, ev, item in sorted(by_user.get(u, []), key=lambda x: (-x[0], -x[1]))]
            hist, black = user_history(recent, p.user)   # black = distinct(userBlacklisted ++ blacklistItems)
        else:
            hist, black = [[] for _ in p.user.names[:p.user.n_history]], list(p.user.blacklist_items)
        similar = []
        if it is not None:
            d, src = by_id.get(it, (-1, {}))
            similar = similar_items(p.item, d, src) if src else []
        excluded = list(dict.fromkeys(list(black) + ([it] if it is not None and p.item.exclude_self else []) + (s or [])))
        recs.append((header + "\n" + mixed_render(p, hist, similar, s, excluded) + "\n").encode("utf-8", "surrogatepass"))
    offsets = np.zeros(len(recs) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in recs], out=offsets[1:])
    return b"".join(recs), offsets


# ---- batchpredict query files ----------------------------------------------------------------------------------------
# A query file (`pio batchpredict --input`) holds one Query JSON object per line, each with its own members.  Record r of
# its body is the buildQuery of line r: mixed_queries() for a one-row batch whose template is that line's members.
# Extraction restates PIO's json4s extract[Query] (Engine.scala:32-65); CcoContext.query_file applies the same rules on the
# device (cco_query_file_read) and decodes each distinct template with template_from_key:
#   * lines are separated by "\n"; a final "\n" opens no empty line; JSON whitespace ("\r" included) may surround the
#     object; an empty or whitespace-only line is an error, as json4s' parse("") fails and the batch job with it;
#   * members compare by their decoded name.  user, item, currentDate: a string; itemSet, blacklistItems, eventNames: an
#     array of strings; userBias, itemBias, itemSetBias: a JSON number, read as a double and rounded to float (JDouble ->
#     Float, f32(float(x))); num, from: an integer literal in Int32 range, a fraction or an exponent is an error [RECALL];
#     returnSelf, withRanks: true or false; fields: an array of {"name": string, "values": [strings], "bias": number}, all
#     three required; dateRange: {"name": string, "before"?: string, "after"?: string};
#   * null is an absent member (an Option is None); unknown members are ignored [RECALL: json4s extraction ignores extra
#     fields]; withRanks is checked and then ignored (it only changes how results are read);
#   * deviation: a repeated known member is an error (json4s keeps both, and which one it extracts is not verifiable here).
#   * the row members are user, item, itemSet and blacklistItems; every other known member is the line's template;
#   * deviations of the device reader (CcoContext.query_file): the inside of an unknown member's value is checked only for
#     its strings and bracket balance, and bytes are not checked as UTF-8; a template member's value that is not JSON is
#     an error naming the member.
ROW_MEMBERS = ("user", "item", "itemSet", "blacklistItems")
TEMPLATE_MEMBERS = ("fields", "dateRange", "currentDate", "returnSelf", "num", "from", "eventNames", "userBias", "itemBias", "itemSetBias")
KNOWN_MEMBERS = frozenset(ROW_MEMBERS + TEMPLATE_MEMBERS + ("withRanks",))


class _Obj(dict):
    """a decoded JSON object that remembers its member names in order (json's last-wins dict drops repeats)"""
    def __init__(self, pairs):
        super().__init__(pairs)
        self.names = [k for k, _ in pairs]


def _no_constant(x):
    raise ValueError(f"{x} is not JSON")


def query_file_lines(data) -> list:
    """the lines of a query file's bytes: "\\n"-separated, a final "\\n" opens no line"""
    data = bytes(data)
    if not data:
        return []
    lines = data.split(b"\n")
    return lines[:-1] if data.endswith(b"\n") else lines


def parse_query_line(raw: bytes, r: int):
    """one line of a query file -> (template key, MixedQuery, user, item, item set); ValueError naming line r"""
    import json
    def bad(what):
        return ValueError(f"line {r}: {what}")
    try:
        text = raw.decode("utf-8", "surrogatepass")
    except UnicodeDecodeError:
        raise bad("not UTF-8") from None
    if not text.strip(" \t\r"):
        raise bad("not a JSON object (an empty line is not a query)")
    try:
        d = json.loads(text, object_pairs_hook=_Obj, parse_constant=_no_constant)
    except ValueError as e:
        raise bad(f"not one JSON object ({e})") from None
    if not isinstance(d, _Obj):
        raise bad("not a JSON object")
    seen = set()
    for n in d.names:
        if n in KNOWN_MEMBERS and n in seen:
            raise bad(f'the member "{n}" is repeated')
        seen.add(n)
    m = {k: d[k] for k in KNOWN_MEMBERS if d.get(k) is not None}
    if "withRanks" in m and not isinstance(m["withRanks"], bool):
        raise bad('"withRanks" is not true or false')
    for k in ("user", "item"):
        if k in m and not isinstance(m[k], str):
            raise bad(f'"{k}" is not a string')
    for k in ("blacklistItems", "itemSet"):
        if k in m and (not isinstance(m[k], list) or not all(isinstance(x, str) for x in m[k])):
            raise bad(f'"{k}" is not an array of strings')
    q = template_query(m, r)
    q.blacklistItems = list(m["blacklistItems"]) if "blacklistItems" in m else None
    key = json.dumps([m.get(k) for k in TEMPLATE_MEMBERS])
    return key, q, m.get("user"), m.get("item"), None if "itemSet" not in m else list(m["itemSet"])


def template_query(m: dict, r: int) -> MixedQuery:
    """the template members of a line (decoded, null dropped) -> MixedQuery without blacklistItems; ValueError naming line r"""
    def bad(what):
        return ValueError(f"line {r}: {what}")

    def string(k, v):
        if not isinstance(v, str):
            raise bad(f'"{k}" is not a string')
        return v

    def strings(k, v):
        if not isinstance(v, list) or not all(isinstance(x, str) for x in v):
            raise bad(f'"{k}" is not an array of strings')
        return list(v)

    def number(k, v):
        if isinstance(v, bool) or not isinstance(v, (int, float)):
            raise bad(f'"{k}" is not a number')
        try:
            return float(v)
        except OverflowError:
            raise bad(f'"{k}" is out of the range of a double') from None

    def int32(k, v):
        if isinstance(v, bool) or not isinstance(v, int):
            raise bad(f'"{k}" is not an integer literal')
        if not -2**31 <= v < 2**31:
            raise bad(f'"{k}" is outside the Int32 range')
        return v

    def boolean(k, v):
        if not isinstance(v, bool):
            raise bad(f'"{k}" is not true or false')
        return v

    def fields(v):
        if not isinstance(v, list):
            raise bad('"fields" is not an array')
        out = []
        for f in v:
            if not isinstance(f, dict) or any(f.get(x) is None for x in ("name", "values", "bias")):
                raise bad('a "fields" element is not {"name": string, "values": [strings], "bias": number}')
            out.append(Field(string("fields.name", f["name"]), strings("fields.values", f["values"]), number("fields.bias", f["bias"])))
        return out

    def date_range(v):
        if not isinstance(v, dict) or v.get("name") is None:
            raise bad('"dateRange" is not {"name": string, "before"?: string, "after"?: string}')
        return DateRange(string("dateRange.name", v["name"]), *[None if v.get(x) is None else string("dateRange." + x, v[x]) for x in ("before", "after")])

    return MixedQuery(userBias=number("userBias", m["userBias"]) if "userBias" in m else None,
                   fields=fields(m["fields"]) if "fields" in m else None,
                   currentDate=string("currentDate", m["currentDate"]) if "currentDate" in m else None,
                   dateRange=date_range(m["dateRange"]) if "dateRange" in m else None,
                   num=int32("num", m["num"]) if "num" in m else None,
                   from_=int32("from", m["from"]) if "from" in m else None,
                   eventNames=strings("eventNames", m["eventNames"]) if "eventNames" in m else None,
                   itemBias=number("itemBias", m["itemBias"]) if "itemBias" in m else None,
                   returnSelf=boolean("returnSelf", m["returnSelf"]) if "returnSelf" in m else None,
                   itemSetBias=number("itemSetBias", m["itemSetBias"]) if "itemSetBias" in m else None)


def template_from_key(key: bytes, r: int) -> MixedQuery:
    """a template key of cco_query_file_read (the template members' raw values in TEMPLATE_MEMBERS order, '\\0' between
    them, an absent one empty) -> MixedQuery; ValueError naming line r (the template's first line)"""
    import json
    parts = key.split(b"\0")
    m = {}
    for k, raw in zip(TEMPLATE_MEMBERS, parts):
        if not raw:
            continue
        try:
            m[k] = json.loads(raw.decode("utf-8", "surrogatepass"), object_pairs_hook=_Obj, parse_constant=_no_constant)
        except ValueError:
            raise ValueError(f'line {r}: "{k}" is not JSON') from None
    return template_query(m, r)


def query_file_line_check(ap, q: MixedQuery, r: int, user, item, item_set, now_ms, have_events: bool, have_index: bool):
    """the errors mixed_queries() raises for line r as a one-row batch, with the line named; -> its MixedPlan"""
    try:
        p = mixed_plan(ap, q, now_ms, with_limits=user is not None)
    except KeyError as e:
        raise ValueError(f"line {r}: {e.args[0]}") from None
    except ValueError as e:
        raise ValueError(f"line {r}: {e}") from None
    if user is not None and not have_events:
        raise ValueError(f"line {r}: a row has a user: its history needs the events")
    if item is not None and not have_index:
        raise ValueError(f"line {r}: a row has an item: its similar items need an index body")
    if item_set is not None and p.with_set and p.set_name is None:
        raise ValueError(f"line {r}: an item-set query needs a model event name: the set clause's field is the first one")
    return p


def query_file(events, index_body: Optional[bytes], ap, lines, now_ms: Optional[int] = None, header: str = "{}"):
    """the host mirror of CcoContext.query_file: one record per line of a batchpredict query file (bytes), the line's
    buildQuery as mixed_queries() writes it for a one-row batch with the line's members as its template -> (body, offsets)"""
    recs = []
    for r, raw in enumerate(query_file_lines(lines)):
        _, q, u, it, s = parse_query_line(raw, r)
        query_file_line_check(ap, q, r, u, it, s, now_ms, events is not None, index_body is not None)
        try:
            # the set column is always given (a line may have no member), so the batch has its one row
            body, _ = mixed_queries(events, index_body, ap, q, None if u is None else [u], None if it is None else [it], [s], now_ms,
                                    header)
        except ValueError as e:
            raise ValueError(f"line {r}: {e}") from None
        recs.append(body)
    offsets = np.zeros(len(recs) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in recs], out=offsets[1:])
    return b"".join(recs), offsets
