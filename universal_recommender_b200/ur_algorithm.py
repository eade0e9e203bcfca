"""Mirror of the train half of URAlgorithm that reaches the hot path
(src/main/scala/URAlgorithm.scala:130-171 params, :310-369 calcAll).
calc_all_on_device runs the whole train half on the GPU, string events in and the Elasticsearch bulk body out.
calc_pop_on_device runs calcPop (recsModel "backfill") on the GPU: the current index's bulk body in, the same index with
fresh rankings out.  calc_all_from_events / calc_pop_from_events do the same from a PredictionIO event export parsed on the
device (CcoContext.read_events), the DataSource included.  user_queries_from_events builds buildQuery's user queries for a
whole user base from the same export (ur_query.py restates buildQuery); item_queries builds its item queries for every
item of a model index body; item_set_queries builds its item-set ("shopping cart") queries for a batch of sets;
mixed_queries_from_events builds its queries for rows with any subset of user, item and item set; queries_from_file
builds them for a batchpredict query file, each line with its own template; index_from_pages reads the model index back
from Elasticsearch's _search / scroll pages; write_index writes a model index body into Elasticsearch as hotSwap does, over a
request function the caller supplies.  Out of scope: Elasticsearch's scoring and the HTTP client."""
from __future__ import annotations

import json
import os
import time
from dataclasses import dataclass, field
from typing import Optional, Sequence

from .indexed_dataset import IndexedDataset
from .similarity_analysis import CcoContext, DownsamplableCrossOccurrenceDataset, SimilarityAnalysis, default_context, encode_ids
from .ur_query import Field, ItemQuery, ItemSetQuery, MixedQuery, UserQuery
from .ur_model import (RankingParams, RankingType, RefreshedIndex, alias_actions, bulk_item_statuses, extract_jvalue, index_mapping,
                       mapping_additions, new_index_name, property_json, ranking_window, rankings_for, rankings_params)


class DefaultURAlgoParams:
    """URAlgorithm.scala:53-57"""
    MaxEventsPerEventType = 500
    MaxCorrelatorsPerEventType = 50


@dataclass
class IndicatorParams:
    """URAlgorithm.scala:136-140"""
    name: str
    maxItemsPerUser: Optional[int] = None
    maxCorrelatorsPerItem: Optional[int] = None
    minLLR: Optional[float] = None


@dataclass
class URAlgorithmParams:
    """The subset of URAlgorithmParams (URAlgorithm.scala:142-171) that reaches the hot path."""
    eventNames: Optional[Sequence[str]] = None
    maxEventsPerEventType: Optional[int] = None
    maxCorrelatorsPerEventType: Optional[int] = None
    indicators: Optional[Sequence[IndicatorParams]] = None
    seed: Optional[int] = None
    recsModel: str = "all"
    rankings: Optional[Sequence[RankingParams]] = None
    # not an engine.json key of the reference: selects the literal Int/Int row sample rate recalled from Mahout 0.13.0's
    # sampleDownAndBinarize (SURVEY.md A.1; every interaction of a user above maxItemsPerUser is dropped) instead of the
    # real division min(m, d) / d this build defaults to (INTEGRATION.md "Deviation to know about")
    rowRateIntDiv: bool = False
    # query-side keys (buildQuery, ur_query.py); the train ignores them
    blacklistEvents: Optional[Sequence[str]] = None
    maxQueryEvents: Optional[int] = None
    num: Optional[int] = None
    userBias: Optional[float] = None
    itemBias: Optional[float] = None
    returnSelf: Optional[bool] = None
    fields: Optional[Sequence[Field]] = None
    availableDateName: Optional[str] = None
    expireDateName: Optional[str] = None
    dateName: Optional[str] = None
    indexName: Optional[str] = None
    typeName: Optional[str] = None   # the Elasticsearch type of the documents (write_index)

    @staticmethod
    def from_engine_json(algo_params: dict) -> "URAlgorithmParams":
        ind = algo_params.get("indicators")
        return URAlgorithmParams(
            eventNames=algo_params.get("eventNames"),
            maxEventsPerEventType=algo_params.get("maxEventsPerEventType"),
            maxCorrelatorsPerEventType=algo_params.get("maxCorrelatorsPerEventType"),
            indicators=None if ind is None else [IndicatorParams(i["name"], i.get("maxItemsPerUser"),
                                                                 i.get("maxCorrelatorsPerItem"), i.get("minLLR")) for i in ind],
            seed=algo_params.get("seed"), recsModel=algo_params.get("recsModel", "all"),
            rankings=None if algo_params.get("rankings") is None else [RankingParams.from_json(r) for r in algo_params["rankings"]],
            rowRateIntDiv=bool(algo_params.get("rowRateIntDiv", False)),
            blacklistEvents=algo_params.get("blacklistEvents"), maxQueryEvents=algo_params.get("maxQueryEvents"),
            num=algo_params.get("num"), userBias=algo_params.get("userBias"), itemBias=algo_params.get("itemBias"),
            returnSelf=algo_params.get("returnSelf"),
            fields=None if algo_params.get("fields") is None else [Field.from_json(f) for f in algo_params["fields"]],
            availableDateName=algo_params.get("availableDateName"), expireDateName=algo_params.get("expireDateName"),
            dateName=algo_params.get("dateName"), indexName=algo_params.get("indexName"),
            typeName=algo_params.get("typeName"))

    def model_event_names(self) -> list[str]:
        """URAlgorithm.scala:230-235: the indicator names if given, else eventNames"""
        return [i.name for i in self.indicators] if self.indicators else list(self.eventNames or [])


def calc_all(actions: Sequence[tuple[str, IndexedDataset]], ap: URAlgorithmParams,
             ctx: CcoContext | None = None, flags: int = 0) -> list[tuple[str, IndexedDataset]]:
    """URAlgorithm.calcAll up to `cooccurrenceCorrelators` (URAlgorithm.scala:310-349): picks the global-
    params call or the per-indicator call, then zips the event names back on positionally (:349).
    `indicators(i)` is indexed by POSITION in `actions` exactly like the reference (:334-340)."""
    _check_recs_model(ap)
    if ap.recsModel == "backfill":
        return []  # calcPop only: no CCO (URAlgorithm.scala:296)
    seed, flags = _seed_and_flags(ap, flags)
    ids = [d for _, d in actions]
    if not ap.indicators:
        out = SimilarityAnalysis.cooccurrencesIDSs(
            ids, randomSeed=seed,
            maxInterestingItemsPerThing=ap.maxCorrelatorsPerEventType or DefaultURAlgoParams.MaxCorrelatorsPerEventType,
            maxNumInteractions=ap.maxEventsPerEventType or DefaultURAlgoParams.MaxEventsPerEventType, ctx=ctx, flags=flags)
    else:
        inds = ap.indicators
        datasets = [DownsamplableCrossOccurrenceDataset(
            iD, inds[i].maxItemsPerUser or DefaultURAlgoParams.MaxEventsPerEventType,
            inds[i].maxCorrelatorsPerItem or DefaultURAlgoParams.MaxCorrelatorsPerEventType, inds[i].minLLR)
            for i, iD in enumerate(ids)]
        out = SimilarityAnalysis.crossOccurrenceDownsampled(datasets, seed, ctx=ctx, flags=flags)
    return [(name, o) for (name, _), o in zip(actions, out)]


def _check_recs_model(ap: URAlgorithmParams):
    if ap.recsModel not in ("all", "collabFiltering", "backfill"):
        raise ValueError(f"Bad algorithm param recsModel=[{ap.recsModel}] in engine definition params, possibly a bad json "
                         "value. Use one of the available parameter values (all, collabFiltering, backfill).")


def _seed_and_flags(ap: URAlgorithmParams, flags: int):
    seed = ap.seed if ap.seed is not None else int(time.time() * 1000)   # System.currentTimeMillis() (:325,345)
    if ap.rowRateIntDiv:
        flags |= 1   # CCO_FLAG_ROWRATE_INTDIV
    return seed, flags


def calc_all_on_device(events: Sequence[tuple[str, str, str, int]], set_events: Sequence[tuple[str, dict]], ap: URAlgorithmParams,
                       min_events_per_user: Optional[int] = None, now_ms: Optional[int] = None, ctx: CcoContext | None = None,
                       flags: int = 0, ranking_events: Optional[dict] = None) -> bytes:
    """URAlgorithm.calcAll (URAlgorithm.scala:310-369) through URModel.save's documents, on the GPU: string events in, the
    Elasticsearch bulk body out.  events = (user id, event name, item id, time ms); set_events = (item id, {field: value}) of
    the items' `$set` events in event-time order.  Steps: cco_ingest_strings (Preparator) -> cco_train_dataset -> the
    rankings' PopModel histograms (popular, trending, hot, and random over every event name) and the property join ->
    cco_format_model.  "collabFiltering" writes the correlators only (propertiesRDD is empty there); "backfill" raises:
    calcPop refreshes an existing index instead, see calc_pop_on_device.
    now_ms: the rankings' end when a ranking has no offsetDate (default: the wall clock).  A random ranking's values are a
    hash of the item id and the window (ur_model.random_rank): they change with now_ms and repeat for a fixed window.
    ranking_events: {event name: [(item id, time ms)]} the rankings read instead of `events` (PopModel reads events of every
    entity type; events.read_export gives both)."""
    _check_recs_model(ap)
    if ap.recsModel == "backfill":
        raise ValueError("recsModel=backfill runs calcPop against the live index: use calc_pop_on_device with its bulk body")
    ctx = ctx or default_context()
    seed, flags = _seed_and_flags(ap, flags)
    names = ap.model_event_names()
    by_name: dict = {}
    for u, e, i, t in events:
        by_name.setdefault(e, []).append((u, i, t))
    actions = [(n, by_name[n]) for n in names if by_name.get(n)]   # DataSource.scala:79-89 drops empty event RDDs
    if not actions:
        raise ValueError("no events of the model's event names")
    cols = [(*encode_ids([u for u, _, _ in ev]), *encode_ids([i for _, i, _ in ev])) for _, ev in actions]
    params = _indicator_params(ap, [n for n, _ in actions])
    props, rankings = None, None
    if ap.recsModel == "all":
        rank_by_name = ranking_events if ranking_events is not None else {n: [(i, t) for _, i, t in ev] for n, ev in by_name.items()}
        props, rankings = _properties_and_rankings(rank_by_name, set_events, ap, now_ms)
    ds, _, items = ctx.ingest_strings(cols, min_events_per_user or 0)
    try:
        _, h = ctx.train_dataset(ds, params, seed, flags, keep=True)
        try:
            return ctx.format_model(h, [n for n, _ in actions], items[0], items, props, rankings)
        finally:
            ctx.free_result(h)
    finally:
        ctx.free_dataset(ds)


def _indicator_params(ap: URAlgorithmParams, names: Sequence[str]) -> list:
    """(maxItemsPerUser, maxCorrelatorsPerItem, minLLR) per event name of the model (URAlgorithm.scala:323-346)"""
    if ap.indicators:
        ind = {i.name: i for i in ap.indicators}
        return [(ind[n].maxItemsPerUser or DefaultURAlgoParams.MaxEventsPerEventType,
                 ind[n].maxCorrelatorsPerItem or DefaultURAlgoParams.MaxCorrelatorsPerEventType, ind[n].minLLR) for n in names]
    return [(ap.maxEventsPerEventType or DefaultURAlgoParams.MaxEventsPerEventType,
             ap.maxCorrelatorsPerEventType or DefaultURAlgoParams.MaxCorrelatorsPerEventType, None)] * len(names)


def _with_presence(set_events: Sequence[tuple[str, dict]]) -> list:
    """ur_model.aggregate_properties, with an (item, "id", None) triple in the place of an item left with no field"""
    props: dict = {}
    for item, fields in set_events:
        props.setdefault(item, {}).update(fields)
    return [(item, k, v) for item, d in props.items() for k, v in (d.items() if d else [("id", None)])]


def _properties(set_events: Sequence[tuple[str, dict]]):
    """the `$set` properties as the JSON text triples of CcoContext.format_model.  An item given with no field stays a
    property item, as the reference's fieldsRDD lists it: a triple of the field "id" (never written, the document's own
    "id" wins) gives it an "id"-only document and makes it a random-rank candidate."""
    triples = [(i, f, extract_jvalue(f, v)) for i, f, v in _with_presence(set_events)]
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    fidx = {f: k for k, f in enumerate(fields)}
    return (fields, *encode_ids([i for i, _, _ in triples]), [fidx[f] for _, f, _ in triples],
            *encode_ids([property_json(v) for _, _, v in triples]))


def _properties_and_rankings(ev_by_name: dict, set_events: Sequence[tuple[str, dict]], ap: URAlgorithmParams, now_ms: Optional[int]):
    """propertiesRDD's inputs in the form of CcoContext.format_model: the `$set` properties as JSON text triples and the
    rankings of getRanksRDD over the events {event name: [(item, time ms)]}"""
    names = ap.model_event_names()
    now = now_ms if now_ms is not None else int(time.time() * 1000)
    rankings = [(r.field, r.mode, r.start_ms, r.end_ms, [(*encode_ids(items), times) for items, times in r.streams])
                for r in rankings_for(rankings_params(ap.rankings, names), ev_by_name, now, names)]
    return _properties(set_events), rankings


def _log_rankings(ap: URAlgorithmParams, now_ms: Optional[int]) -> list:
    """getRanksRDD's rankings as CcoContext.format_model(log=...) takes them: (field, mode, start, end, event names), the
    choices of ur_model.rankings_for (a random ranking reads every event name of the log)"""
    names = ap.model_event_names()
    now = now_ms if now_ms is not None else int(time.time() * 1000)
    out = []
    for rp in rankings_params(ap.rankings, names):
        t = rp.ranking_type()
        if t not in (RankingType.Popular, RankingType.Trending, RankingType.Hot, RankingType.Random):
            continue
        start, end = ranking_window(rp, now)
        out.append((rp.field_name(), t, start, end, [] if t == RankingType.Random else
                    list(rp.eventNames if rp.eventNames is not None else names[:1])))
    return out


def _read_log(export, ctx: CcoContext, window=None, now_ms: Optional[int] = None):
    """(log, owned): an EventLog as given, or one read by CcoContext.read_events (bytes, a buffer, a path, a `pio export`
    directory, a sequence of paths or an iterable of buffers), through the eventWindow when one is given"""
    from .similarity_analysis import EventLog
    if isinstance(export, EventLog):
        if window is not None:
            raise ValueError("the eventWindow applies while an export is read: pass the export, or read it with read_events(window=...)")
        return export, False
    return ctx.read_events(export, window=window, now_ms=now_ms), True


def _now(now_ms: Optional[int]) -> int:
    return now_ms if now_ms is not None else int(time.time() * 1000)


def calc_all_from_events(export, ap: URAlgorithmParams, min_events_per_user: Optional[int] = None, now_ms: Optional[int] = None,
                         ctx: CcoContext | None = None, flags: int = 0, event_window=None) -> bytes:
    """calc_all_on_device from a PredictionIO event export (any source CcoContext.read_events takes, or an EventLog of this
    context): the export is copied to the GPU and parsed there (the DataSource: include/cco_b200.h cco_event_log_read); the training
    events, the ranking streams and the items' properties, aggregated there from their $set / $unset / $delete events,
    stay in HBM.  Property values are spliced as written.  Same decisions as calc_all_on_device.
    event_window: the DataSource's eventWindow (events.EventWindow, DataSourceParams.eventWindow), applied to every
    selection on the device; its duration counts back from the same now_ms as the rankings."""
    _check_recs_model(ap)
    if ap.recsModel == "backfill":
        raise ValueError("recsModel=backfill runs calcPop against the live index: use calc_pop_from_events with its bulk body")
    ctx = ctx or default_context()
    seed, flags = _seed_and_flags(ap, flags)
    now_ms = _now(now_ms)
    log, owned = _read_log(export, ctx, event_window, now_ms)
    try:
        info = log.info()
        n_train = dict(zip(info.names, info.n_training))
        actions = [n for n in ap.model_event_names() if n_train.get(n)]   # DataSource.scala:79-89 drops empty event RDDs
        if not actions:
            raise ValueError("no events of the model's event names")
        params = _indicator_params(ap, actions)
        ds, _, items = ctx.ingest_event_log(log, actions, min_events_per_user or 0)
        try:
            _, h = ctx.train_dataset(ds, params, seed, flags, keep=True)
            try:
                if ap.recsModel == "collabFiltering":   # the correlators only: propertiesRDD is empty there
                    return ctx.format_model(h, actions, items[0], items)
                return ctx.format_model(h, actions, items[0], items, rankings=_log_rankings(ap, now_ms), log=log)
            finally:
                ctx.free_result(h)
        finally:
            ctx.free_dataset(ds)
    finally:
        if owned:
            log.free()


def calc_pop_on_device(body: bytes, events: Sequence[tuple[str, str, str, int]], set_events: Sequence[tuple[str, dict]],
                       ap: URAlgorithmParams, now_ms: Optional[int] = None, ctx: CcoContext | None = None,
                       ranking_events: Optional[dict] = None) -> bytes:
    """URAlgorithm.calcPop (URAlgorithm.scala:375-399, recsModel "backfill") on the GPU: the rankings of an existing index
    refreshed between trains, without a CCO train.  body = the current index as an Elasticsearch bulk body (what
    calc_all_on_device or format_model wrote, or index_from_pages read back from Elasticsearch); events and set_events as
    in calc_all_on_device, now_ms likewise.  The properties and rankings are built as calc_all_on_device builds them and
    joined into the old documents by cco_rerank_model: per document, fresh `$set` properties < old members < rankings <
    "id".  So a fresh `$set` value loses to an old member of the same name, and an old rank member survives when the item
    has no score in the new window.  Items with a property or a score and no old document are appended."""
    ctx = ctx or default_context()
    by_name: dict = {}
    for _, e, i, t in events:
        by_name.setdefault(e, []).append((i, t))
    props, rankings = _properties_and_rankings(ranking_events if ranking_events is not None else by_name, set_events, ap, now_ms)
    return ctx.rerank_model(body, props, rankings)


def calc_pop_from_events(body: bytes, export, ap: URAlgorithmParams, now_ms: Optional[int] = None, ctx: CcoContext | None = None,
                         event_window=None) -> bytes:
    """calc_pop_on_device from a PredictionIO event export (as in calc_all_from_events): the ranking streams and the
    properties of the log, both in HBM, joined into the old index by cco_rerank_model_log.  event_window as in
    calc_all_from_events."""
    ctx = ctx or default_context()
    now_ms = _now(now_ms)
    log, owned = _read_log(export, ctx, event_window, now_ms)
    try:
        return ctx.rerank_model(body, None, _log_rankings(ap, now_ms), log=log)
    finally:
        if owned:
            log.free()


def _refresh_names(ap: URAlgorithmParams) -> tuple:
    """(correlator names, computed ranking names) of a refresh: the model's event names, and the fields of the rankings
    _log_rankings lists (popular, trending, hot, random; a userDefined field is an ordinary property)"""
    return ap.model_event_names(), [r[0] for r in _log_rankings(ap, 0)]


def clean_export(src, out, window, now_ms: Optional[int] = None, chunk_bytes: Optional[int] = None, ctx: CcoContext | None = None):
    """PredictionIO's cleanPersistedPEvents in one call [RECALL, unverifiable here]: the export src read on the device with
    the eventWindow `window` (events.EventWindow; its cutoff counted back from now_ms, the wall clock by default) as an
    extendable log, its cleaned events written to out (EventLog.write_clean, compressProperties from the window), and the
    log freed.  src is read twice, so it must be a path, a part directory, a list of paths or a buffer, not a generator.
    The caller imports out into the event store (`pio import`).  -> CleanStats"""
    ctx = ctx or default_context()
    log = ctx.read_events(src, chunk_bytes, window, _now(now_ms), extendable=True)
    try:
        return log.write_clean(src, out, window is not None and window.compressProperties, chunk_bytes)
    finally:
        log.free()


def refresh_properties_from_events(body: bytes, export, ap: URAlgorithmParams, now_ms: Optional[int] = None, event_window=None,
                                   ctx: CcoContext | None = None) -> RefreshedIndex:
    """The item properties of the live index refreshed without a retrain (CcoContext.refresh_properties): the properties
    aggregated from a PredictionIO event export on the device (as in calc_all_from_events; an EventLog is used as given, not
    freed, so a resident log extended with new lines serves every refresh) written into the documents of the current index
    `body`.  Fresh properties win: a `$set` value replaces the old one, an `$unset` field leaves the document, a `$delete`d
    item loses its properties and, when it has no correlator or ranking member either, its document.  Correlators and
    rankings are kept as they are, never recomputed.  now_ms and event_window as in calc_all_from_events.  -> RefreshedIndex;
    update_index writes its delta and deletes in place."""
    ctx = ctx or default_context()
    now_ms = _now(now_ms)
    correlators, rankings = _refresh_names(ap)
    log, owned = _read_log(export, ctx, event_window, now_ms)
    try:
        return ctx.refresh_properties(body, correlators, rankings, log=log)
    finally:
        if owned:
            log.free()


def refresh_properties_on_device(body: bytes, set_events: Sequence[tuple[str, dict]], ap: URAlgorithmParams,
                                 ctx: CcoContext | None = None) -> RefreshedIndex:
    """refresh_properties_from_events with the properties given as calc_pop_on_device takes them: set_events = the `$set`
    events [(item, {field: value})] in event-time order, the later value of a field winning"""
    ctx = ctx or default_context()
    correlators, rankings = _refresh_names(ap)
    return ctx.refresh_properties(body, correlators, rankings, properties=_properties(set_events))


def user_queries_from_events(export, ap: URAlgorithmParams, query: Optional[UserQuery] = None, users=None, now_ms: Optional[int] = None,
                             ctx: CcoContext | None = None, event_window=None, header: str = "{}"):
    """buildQuery (URAlgorithm.scala:563-839) for every user of `users` (None: every user with a training event of a query
    event name, by first line) from a PredictionIO event export read on the device with history retention: one
    `header\nquery\n` record per user, the body of an Elasticsearch _msearch.  -> (body, offsets) as CcoContext.user_queries
    ((body, offsets, users) for users=None).  now_ms: "now" of the available / expire date filter and of the eventWindow.
    The query event names, limits, blacklist and fragments are ur_query.plan's."""
    ctx = ctx or default_context()
    now_ms = _now(now_ms)
    from .similarity_analysis import EventLog
    if isinstance(export, EventLog):
        if event_window is not None:
            raise ValueError("the eventWindow applies while an export is read")
        return ctx.user_queries(export, ap, query, users, now_ms, header)
    log = ctx.read_events(export, window=event_window, now_ms=now_ms, keep_history=True)
    try:
        return ctx.user_queries(log, ap, query, users, now_ms, header)
    finally:
        log.free()


def mixed_queries_from_events(export, index_body: Optional[bytes], ap: URAlgorithmParams, query: Optional[MixedQuery] = None, users=None,
                              items=None, item_sets=None, now_ms: Optional[int] = None, ctx: CcoContext | None = None, event_window=None,
                              header: str = "{}"):
    """buildQuery (URAlgorithm.scala:563-839) for rows that may each have a user, an item and an item set ("this user, on
    this product page", "this user, with this cart"): the users' histories from a PredictionIO event export read on the
    device with history retention (or an EventLog read with keep_history=True; None when no row has a user), the similar
    items from a model index body (None when no row has an item).  One `header\nquery\n` record per row, the body of an
    Elasticsearch _msearch.  users, items, item_sets as in CcoContext.mixed_queries: a column that is None has no member in
    any row, a row's None has none in that row.  -> (body, offsets).  now_ms: "now" of the available / expire date filter
    and of the eventWindow.  The fragments are ur_query.mixed_plan's."""
    ctx = ctx or default_context()
    now_ms = _now(now_ms)
    from .similarity_analysis import EventLog
    if export is None or isinstance(export, EventLog):
        if event_window is not None:
            raise ValueError("the eventWindow applies while an export is read")
        return ctx.mixed_queries(export, index_body, ap, query, users, items, item_sets, now_ms, header)
    log = ctx.read_events(export, window=event_window, now_ms=now_ms, keep_history=True)
    try:
        return ctx.mixed_queries(log, index_body, ap, query, users, items, item_sets, now_ms, header)
    finally:
        log.free()


def queries_from_file(query_file, export, index_body: Optional[bytes], ap: URAlgorithmParams, now_ms: Optional[int] = None,
                      ctx: CcoContext | None = None, event_window=None, header: str = "{}"):
    """buildQuery (URAlgorithm.scala:563-839) for every line of a batchpredict query file (`pio batchpredict --input`: one
    Query JSON object per line, each with its own members), as CcoContext.query_file: the bytes or a path; export: a
    PredictionIO event export read on the device with history retention, or an EventLog read with keep_history=True, or
    None when no line has a user; index_body: a model index body (None when no line has an item).  -> (body, offsets),
    record r is line r's.  now_ms: "now" of the available / expire date filter and of the eventWindow."""
    ctx = ctx or default_context()
    now_ms = _now(now_ms)
    from .similarity_analysis import EventLog
    if export is None or isinstance(export, EventLog):
        if event_window is not None:
            raise ValueError("the eventWindow applies while an export is read")
        return ctx.query_file(export, index_body, ap, query_file, now_ms, header)
    log = ctx.read_events(export, window=event_window, now_ms=now_ms, keep_history=True)
    try:
        return ctx.query_file(log, index_body, ap, query_file, now_ms, header)
    finally:
        log.free()


def predictions_from_responses(responses, ap: URAlgorithmParams, with_ranks=False, counts=None, ctx: CcoContext | None = None):
    """URAlgorithm.predict's second half (URAlgorithm.scala:484-529, Serving.scala:25-29) for every element of Elasticsearch
    _msearch response bodies -- the responses to the bodies the query builders write -- on the device, as
    CcoContext.search_results: one body or a list or generator of them (bytes or paths), with_ranks for every record or
    one per record, counts the elements of each body.  -> SearchResults: .records() are the PredictedResult JSON texts."""
    ctx = ctx or default_context()
    return ctx.search_results(responses, ap, with_ranks=with_ranks, counts=counts)


def index_from_pages(pages, ctx: CcoContext | None = None) -> bytes:
    """The model index read back from Elasticsearch, as calcPop (EsClient.getRDD, EsClient.scala:464-470) and the item
    queries (EsClient.getSource, EsClient.scala:394-442) read it, on the device (CcoContext.index_pages): one _search /
    _search/scroll response page, or a list or generator of them (bytes or paths), in order.  -> the bulk body
    format_model writes, which calc_pop_from_events, calc_pop_on_device and the query builders take.  Raises when the
    first page's hits.total is exact and differs from the documents read: the scroll ended early."""
    ctx = ctx or default_context()
    if isinstance(pages, (bytes, bytearray, memoryview, str, os.PathLike)):
        pages = [pages]
    with ctx.index_pages() as r:
        for page in pages:
            r.append(page)
        body = r.finish()
        if r.total >= 0 and r.total != r.n_docs:
            raise ValueError(f"hits.total is {r.total} but the pages hold {r.n_docs} documents: the scroll ended early")
    return body


def batchpredict_output(query_file, responses, ap: URAlgorithmParams, out=None, counts=None, ctx: CcoContext | None = None):
    """`pio batchpredict --output` on the device: line r of the query file (bytes or a path; one Query JSON object per
    line, as queries_from_file reads it) paired with record r of the _msearch responses to the body queries_from_file
    built from it (one body or a list or generator of bodies; counts the records of each when there are several).  Each
    record's withRanks is its line's.  -> the output lines as bytes, each ending in a newline ([RECALL] PredictionIO's
    {"query":...,"prediction":...}), or None after writing them to the path `out`."""
    ctx = ctx or default_context()
    text = ctx.search_results(responses, ap, counts=counts, query_lines=query_file).text()
    if out is None:
        return text
    with open(out, "wb") as f:
        f.write(text)
    return None


def item_queries(index_body: bytes, ap: URAlgorithmParams, query: Optional[ItemQuery] = None, items=None, now_ms: Optional[int] = None,
                 ctx: CcoContext | None = None, header: str = "{}"):
    """buildQuery (URAlgorithm.scala:563-792) for every item of `items` (None: every document of the index, in body order),
    the similar items read from the model index body (what calc_all_from_events, calc_all_on_device or a calcPop wrote,
    or index_from_pages read back from Elasticsearch) on the device: one `header\nquery\n` record per item, the body of
    an Elasticsearch _msearch.  -> (body, offsets) as CcoContext.item_queries ((body, offsets, items) for items=None).
    now_ms: "now" of the available / expire date filter (default: the wall clock).  The fragments are ur_query.item_plan's."""
    ctx = ctx or default_context()
    return ctx.item_queries(index_body, ap, query, items, _now(now_ms), header)


def item_set_queries(sets, ap: URAlgorithmParams, query: Optional[ItemSetQuery] = None, now_ms: Optional[int] = None,
                     ctx: CcoContext | None = None, header: str = "{}"):
    """buildQuery (URAlgorithm.scala:563-767) for every item set ("shopping cart") of `sets` on the device: one
    `header\nquery\n` record per set, the body of an Elasticsearch _msearch.  sets: a sequence of sequences of str, or the
    Arrow list<large_string> buffers (set_offsets, elem_offsets, elem_bytes).  -> (body, offsets) as
    CcoContext.item_set_queries.  now_ms: "now" of the available / expire date filter (default: the wall clock).  The
    fragments are ur_query.item_set_plan's; ValueError without a model event name (the set clause's field)."""
    ctx = ctx or default_context()
    return ctx.item_set_queries(sets, ap, query, _now(now_ms), header)


class IndexWriteError(RuntimeError):
    """write_index stopped before the alias swap: the alias still serves the old index; the new one is left in place"""

    def __init__(self, message: str, new_index: str, result=None):
        super().__init__(message)
        self.new_index = new_index
        self.result = result


def _bulk_ids(body: bytes, docs) -> dict:
    """{document index: decoded _id} of the given documents of a model index body"""
    want, out = set(int(d) for d in docs), {}
    at = 0
    for d in range(max(want) + 1 if want else 0):
        end = body.index(b"\n", at)
        if d in want:
            out[d] = json.loads(body[at:end].decode("utf-8", "surrogatepass"))["index"]["_id"]
        at = body.index(b"\n", end + 1) + 1
    return out


def write_index(body: bytes, ap: URAlgorithmParams, request, now_ms: Optional[int] = None, max_docs: int = 1000,
                max_bytes: int = 1 << 20, retries: int = 3, retry_wait_s: float = 10.0, ctx: CcoContext | None = None):
    """URModel.save -> EsClient.hotSwap (URModel.scala:47-84, EsClient.scala:168-246, 257-362) for a model index body
    (what calc_all_from_events or a calcPop wrote), over request(method, path, body bytes or None) -> (HTTP status, response
    bytes), one request at a time:
      1. HEAD /<new>, which must be 404 (new = <indexName>_<now_ms>);  2. PUT /<new> with index_mapping(esFields);
      3. POST /<new>/_refresh;  4. POST /<new>/<typeName>/_bulk for every request of at most max_docs documents and
      max_bytes bytes, each response read on the device (CcoContext.index_write);  5. up to `retries` rounds that send
      again the documents rejected with 429, retry_wait_s apart (elasticsearch-hadoop's es.batch.write.retry.count /
      .wait);  6. HEAD and GET /_alias/<indexName>, HEAD of its old index, POST /_aliases (add, remove_index), DELETE of
      the old indexes.
    An HTTP status other than 200 on steps 2-4, any item failure other than 429, or 429s left after the last round raise
    IndexWriteError before step 6, naming the first documents' ids with Elasticsearch's error type and reason: the alias
    keeps serving the old index and the new index is left in place.  -> (new index name, IndexWriteResult)."""
    if not ap.indexName or not ap.typeName:
        raise ValueError("write_index needs indexName and typeName in the algorithm params")
    ctx = ctx or default_context()
    body = bytes(body)
    alias, type_name = ap.indexName, ap.typeName
    new = new_index_name(alias, _now(now_ms))

    def call(method: str, path: str, data: Optional[bytes] = None, ok=(200,)):
        status, resp = request(method, path, data)
        if ok is not None and status not in ok:
            raise IndexWriteError(f"{method} {path} answered HTTP {status}: {bytes(resp or b'')[:500]!r}", new)
        return status, resp

    with ctx.index_write(body, max_docs, max_bytes) as w:
        mapping = index_mapping(w.fields(), ap, type_name)
        call("HEAD", f"/{new}", ok=(404,))
        call("PUT", f"/{new}", mapping)
        call("POST", f"/{new}/_refresh")
        bulk = f"/{new}/{type_name}/_bulk"
        for q, part in enumerate(w.requests()):
            w.response(q, call("POST", bulk, part)[1])
        for _ in range(retries):
            first, parts = w.retry()
            if not parts:
                break
            time.sleep(retry_wait_s)
            for k, (_, part) in enumerate(parts):
                w.response(first + k, call("POST", bulk, part)[1])
        result = w.finish()
    if result.errors:
        shown = result.errors[:5]
        ids = _bulk_ids(body, [d for d, _, _ in shown])
        lines = "; ".join(f"{ids[d]!r}: {t or '-'}: {r or '-'}" for d, t, r in shown)
        raise IndexWriteError(f"{len(result.errors)} documents were not written to {new} ({result.n_rejected} still rejected "
                              f"with 429, {result.n_failed} failed), the alias {alias} is unchanged: {lines}", new, result)
    old_set, old = [], None
    if call("HEAD", f"/_alias/{alias}", ok=None)[0] == 200:
        old_set = list(json.loads(bytes(call("GET", f"/_alias/{alias}")[1]).decode("utf-8")).keys())
        if old_set and call("HEAD", f"/{old_set[0]}", ok=None)[0] == 200:
            old = old_set[0]
        else:
            old_set = []
    call("POST", "/_aliases", alias_actions(alias, new, old))
    for name in old_set:   # deleteIndex: HEAD, then DELETE when it still exists
        st = call("HEAD", f"/{name}", ok=None)[0]
        if st == 200:
            call("DELETE", f"/{name}", ok=None)
        elif st != 404:
            raise IndexWriteError(f"HEAD /{name} answered HTTP {st}", new, result)
    return new, result


def _delete_requests(deletes: bytes, max_docs: int, max_bytes: int) -> list:
    """the delete lines cut as bulk_requests cuts documents -> [(decoded ids, request bytes)]"""
    lines = [ln + b"\n" for ln in bytes(deletes).split(b"\n")[:-1]]
    out, cur = [], []
    for ln in lines:
        if cur and (len(cur) == max_docs or sum(map(len, cur)) + len(ln) > max_bytes):
            out.append(cur)
            cur = []
        cur.append(ln)
    if cur:
        out.append(cur)
    ids = lambda part: [json.loads(ln.decode("utf-8", "surrogatepass"))["delete"]["_id"] for ln in part]
    return [(ids(part), b"".join(part)) for part in out]


def update_index(refresh: RefreshedIndex, ap: URAlgorithmParams, request, max_docs: int = 1000, max_bytes: int = 1 << 20,
                 retries: int = 3, retry_wait_s: float = 10.0, ctx: CcoContext | None = None):
    """A refresh (refresh_properties_from_events) written into the live index in place, over request(method, path, body
    bytes or None) -> (HTTP status, response bytes), as for write_index:
      1. GET /_alias/<indexName>, which must name exactly one index;  2. GET /<index>/_mapping/<typeName>, then one PUT of
      the same path adding the delta's fields the mapping lacks, typed as index_mapping types them (Elasticsearch would
      map a new property as analysed text);  3. POST /<index>/<typeName>/_bulk for the delta, at most max_docs documents
      and max_bytes bytes per request, the responses read on the device with up to `retries` rounds for 429s, retry_wait_s
      apart (write_index's steps 4-5);  4. the delete lines as _bulk requests cut by the same limits, a delete answered 200
      or 404 (already gone) being success;  5. POST /<index>/_refresh.
    No index is created, no alias moves, nothing but the deleted documents is removed.  Every action writes or deletes a
    whole document, so running the update again after a partial failure converges on the same index.  A status other
    than 200, an item failure or 429s left after the last round raise IndexWriteError naming the index.
    -> (index name, IndexWriteResult of the delta, or None when the delta is empty)."""
    if not ap.indexName or not ap.typeName:
        raise ValueError("update_index needs indexName and typeName in the algorithm params")
    ctx = ctx or default_context()
    alias, type_name = ap.indexName, ap.typeName
    index = None

    def call(method: str, path: str, data: Optional[bytes] = None, ok=(200,)):
        status, resp = request(method, path, data)
        if status not in ok:
            raise IndexWriteError(f"{method} {path} answered HTTP {status}: {bytes(resp or b'')[:500]!r}", index)
        return bytes(resp or b"")

    names = list(json.loads(call("GET", f"/_alias/{alias}").decode("utf-8")).keys())
    if len(names) != 1:
        raise IndexWriteError(f"the alias {alias} names {len(names)} indexes ({', '.join(names) or 'none'}): an update writes into one", None)
    index = names[0]
    mapping_path = f"/{index}/_mapping/{type_name}"
    known: set = set()
    for idx in json.loads(call("GET", mapping_path).decode("utf-8")).values():
        known.update(((idx.get("mappings") or {}).get(type_name) or {}).get("properties") or {})
    result = None
    if refresh.delta:
        with ctx.index_write(refresh.delta, max_docs, max_bytes) as w:
            missing = [f for f in w.fields() if json.loads('"' + f + '"') not in known]
            if missing:
                call("PUT", mapping_path, mapping_additions(missing, ap))
            bulk = f"/{index}/{type_name}/_bulk"
            for q, part in enumerate(w.requests()):
                w.response(q, call("POST", bulk, part))
            for _ in range(retries):
                first, parts = w.retry()
                if not parts:
                    break
                time.sleep(retry_wait_s)
                for k, (_, part) in enumerate(parts):
                    w.response(first + k, call("POST", bulk, part))
            result = w.finish()
        if result.errors:
            shown = result.errors[:5]
            ids = _bulk_ids(refresh.delta, [d for d, _, _ in shown])
            lines = "; ".join(f"{ids[d]!r}: {t or '-'}: {r or '-'}" for d, t, r in shown)
            raise IndexWriteError(f"{len(result.errors)} documents were not written to {index} ({result.n_rejected} still rejected "
                                  f"with 429, {result.n_failed} failed): {lines}", index, result)
    for ids, part in _delete_requests(refresh.deletes, max_docs, max_bytes):
        statuses = bulk_item_statuses(call("POST", f"/{index}/{type_name}/_bulk", part), ids, action="delete")
        bad = [(i, st) for i, (st, _, _) in zip(ids, statuses) if st not in (200, 404)]
        if bad:
            raise IndexWriteError(f"{len(bad)} deletes failed on {index}: " + "; ".join(f"{i!r}: HTTP {st}" for i, st in bad[:5]), index, result)
    call("POST", f"/{index}/_refresh")
    return index, result
