"""cco_item_queries and cco_event_log_user_queries at their edges, each body compared byte for byte (offsets included)
with the host mirror in ur_query and each record read back with json.loads against the structure the inputs were built
with: every code point through the json4s quote (uq_escape on the device, uq_quote in the templates); k_iq_array's
backslash-parity carry, whitespace runs and malformed values at every offset; the 32-candidate steps of uq_list and the
maxQueryEvents slice around 32 and 64; history limits, ties on the limit and 64 query names against history_ref; and
more records than the grid has warps."""
import random

import numpy as np
import pytest
import torch

from universal_recommender_b200 import CcoContext
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_algorithm as ur
from universal_recommender_b200 import ur_query as Q
import query_edges_ref as R

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000_000
MODEL3 = ["purchase", "view", "like"]


@pytest.fixture(scope="module")
def ctx():
    c = CcoContext()
    yield c
    c.close()


def warps() -> int:
    """the warps of one launch at grid_for's cap: sm_count x 8 blocks of 8 warps"""
    return torch.cuda.get_device_properties(0).multi_processor_count * 64


def params(**kw):
    return ur.URAlgorithmParams.from_engine_json(kw)


def item_check(ctx, body, ap, q, items, expect=None):
    """device == mirror; with expect ({id: {name: elements}}, None: a source without members) every record's similar-items
    lists and must_not ids are the expected ones"""
    dev = ctx.item_queries(body, ap, q, items, NOW)
    host = Q.item_queries(body, ap, q, items, NOW)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    if items is None:
        assert dev[2] == host[2]
    if expect is not None:
        p = Q.item_plan(ap, q, NOW)
        skip = _n_clauses(p)
        who = dev[2] if items is None else items
        recs = R.records(dev[0], dev[1])
        assert len(recs) == len(who)
        for it, (_, query) in zip(who, recs):
            pairs, ids = R.clause_lists(query, p.in_must)
            assert pairs[skip:] == R.expected_similar(p.names, expect.get(it), p.max_query_events), it
            assert ids == list(dict.fromkeys(list(p.blacklist_items) + ([it] if p.exclude_self else [])))
    return dev


def _n_clauses(p) -> int:
    """the empty history clauses ahead of the similar items in their section"""
    import json
    return len(json.loads("[" + (p.must_head if p.in_must else p.should_head) + "]"))


def user_check(ctx, data, ap, q, users, chunk=None, pieces=None):
    """device == mirror, for one read (chunk None), a chunked one, or appended pieces; every record's history lists and
    blacklist equal history_ref's"""
    ev = E.read_export(data)
    src = data if pieces is None else [data[a:b] for a, b in zip([0] + pieces, pieces + [len(data)])]
    with ctx.read_events(src, chunk_bytes=chunk, now_ms=NOW, keep_history=True) as log:
        dev = ctx.user_queries(log, ap, q, users, NOW)
    host = Q.user_queries(ev, ap, q, users, NOW)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    if users is None:
        assert dev[2] == host[2]
    p = Q.plan(ap, q or Q.UserQuery(), NOW)
    mine = {}
    for line, (u, n, i, t) in enumerate(ev.events):
        mine.setdefault(u, []).append((n, i, t, line))
    who = dev[2] if users is None else users
    for u, (_, query) in zip(who, R.records(dev[0], dev[1])):
        lists, black = R.history_ref(mine.get(u, []), p.names, p.limits, p.blacklist, p.blacklist_items)
        pairs, ids = R.clause_lists(query, p.in_must)
        assert pairs[:p.n_history] == list(zip(p.names, lists))[:p.n_history], u
        assert ids == black, u
    return dev


# ---- 1. every code point through the quote ------------------------------------------------------------------------------
def test_every_code_point_as_elements_and_ids(ctx):
    body, ids, expect = R.codepoint_index(MODEL3)
    ap = params(eventNames=MODEL3, maxQueryEvents=100)
    dev = item_check(ctx, body, ap, None, None, expect)
    text = dev[0].decode("utf-8", "surrogatepass")
    for s in ids:   # each string re-escaped by uq_escape, as the reference quote writes it
        assert R.json4s_quote_ref(s) in text and Q.json_string(s) == R.json4s_quote_ref(s)
    rng = random.Random(1)
    items = rng.sample(ids, 300) + R.EDGE_STRINGS + ["unknown", ""]
    black = rng.sample(ids, 40) + R.EDGE_STRINGS[:5] + ids[:2]
    item_check(ctx, body, ap, Q.ItemQuery(blacklistItems=black), items, expect)
    item_check(ctx, body, params(eventNames=MODEL3, maxQueryEvents=100, itemBias=-1), Q.ItemQuery(blacklistItems=black, returnSelf=True),
               items, expect)


def test_every_code_point_in_model_names(ctx):
    names = R.names64()
    ap = params(eventNames=names, maxQueryEvents=100)
    docs = [("a", R.source([(names[j], ["x%d" % j, names[j][:3]]) for j in range(0, 64, 3)], 0)),
            ("b", R.source([(names[j], ["y"]) for j in (0, 1, 62, 63)], 1)), ("c", "{}"), ("d", '{"other":[]}')]
    body = R.index_body(docs)
    expect = {"a": {names[j]: ["x%d" % j, names[j][:3]] for j in range(0, 64, 3)}, "b": {names[j]: ["y"] for j in (0, 1, 62, 63)},
              "c": None, "d": {}}
    dev = item_check(ctx, body, ap, None, None, expect)
    text = dev[0].decode("utf-8", "surrogatepass")
    for n in names:   # mq_template's uq_quote
        assert "{" + '"terms":' + "{" + R.json4s_quote_ref(n) + ":[" in text
    item_check(ctx, body, ap, Q.ItemQuery(blacklistItems=["a", "x0"]), ["a", "b", "zz", "a"], expect)


def test_every_code_point_in_user_query_names_and_items(ctx):
    names = R.names64()
    data = R.codepoint_export(names)
    ap = params(eventNames=names, maxQueryEvents=100)
    dev = user_check(ctx, data, ap, None, None)
    assert len(dev[2]) == 7
    text = dev[0].decode("utf-8", "surrogatepass")
    for n in names:   # mq_template's uq_quote
        assert '{"terms":{' + R.json4s_quote_ref(n) + ":[" in text
    for k, s in enumerate(R.codepoint_strings() + R.EDGE_STRINGS):   # the items of the query names' events, through uq_escape
        if k % 3 < 2:
            assert R.json4s_quote_ref(s) in text
    user_check(ctx, data, ap, Q.UserQuery(blacklistItems=R.EDGE_STRINGS + ["e\u0085"]), ["u%d" % k for k in range(7)] + ["nobody"], chunk=65521)


# ---- 2. k_iq_array ------------------------------------------------------------------------------------------------------
def test_array_backslash_runs_whitespace_and_brackets(ctx):
    body, ids, expect = R.array_sweep_index()
    ap = params(eventNames=MODEL3, maxQueryEvents=100)
    item_check(ctx, body, ap, None, None, expect)
    item_check(ctx, body, ap, None, ids[::-3] + ["nope"], expect)


@pytest.mark.parametrize("form", [f for f, _ in R.MALFORMED])
def test_malformed_values_refused_at_every_offset(ctx, form):
    ap = params(eventNames=["purchase", "view"], maxQueryEvents=100)
    for at in (0, 17, 39):
        for pad in (0, 5, 31, 32):
            body = R.malformed_index(form, at, pad)
            with pytest.raises(N.CcoInvalidArgument, match=f'document {at}: its "view" member is not an array of strings'):
                ctx.item_queries(body, ap, None, None, NOW)
            others = ["m%d" % d for d in range(40) if d != at]
            dev = ctx.item_queries(body, ap, None, others, NOW)   # the document is not queried: accepted
            host = Q.item_queries(R.malformed_index('["ok"]', at, pad), ap, None, others, NOW)
            assert dev[0] == host[0] and np.array_equal(dev[1], host[1])


# ---- 3. list and slice boundaries ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("mqe", [1, 2, 3, 31, 32, 33, 34, 63, 64, 65])
def test_list_sizes_around_the_slice(ctx, mqe):
    body, ids, expect = R.list_index()
    item_check(ctx, body, params(eventNames=["purchase", "view"], maxQueryEvents=mqe), None, None, expect)
    item_check(ctx, body, params(eventNames=["view", "purchase"], maxQueryEvents=mqe, itemBias=-1, userBias=-1), Q.ItemQuery(itemBias=0.25),
               ids + ["absent"], expect)
    item_check(ctx, body, params(eventNames=["purchase", "view"], maxQueryEvents=mqe, itemBias=1.5), None, ids[::-1], expect)


def test_blacklist_items_lists_31_to_65(ctx):
    body, ids, expect = R.list_index()
    ap = params(eventNames=["purchase", "view"], maxQueryEvents=40)
    rng = random.Random(2)
    pool = ids + ["unknown", "", "x\u2000"]
    for n in range(31, 66):
        black = [rng.choice(pool) for _ in range(n)]
        item_check(ctx, body, ap, Q.ItemQuery(blacklistItems=black, returnSelf=bool(n % 2)), ids + ["unknown"], expect)


# ---- 4. history limits and ties -----------------------------------------------------------------------------------------
def test_history_limits_and_ties(ctx):
    data, engine, names, users = R.history_export()
    ap = ur.URAlgorithmParams.from_engine_json(engine)
    ev = E.read_export(data)
    black_items = sorted({i for _, n, i, _ in ev.events if n in ("n31", "n1")})
    rng = random.Random(4)
    cut = sorted(rng.sample(range(1, len(data)), 40))
    queries = [None, Q.UserQuery(blacklistItems=(black_items[:20] + ["i0", "nope", "out-u-1-2"] * 5)[:35]),
               Q.UserQuery(eventNames=names[::-1] + [names[2]])]
    for q in queries:
        user_check(ctx, data, ap, q, None)
        user_check(ctx, data, ap, q, users + ["nobody", users[0]])
        user_check(ctx, data, ap, q, users, chunk=4093)
        user_check(ctx, data, ap, q, None, chunk=1 << 16, pieces=cut)


def test_64_query_names(ctx):
    data, engine, names, users = R.names64_export()
    assert len(names) == 64 and len(set(names)) == 63
    ap = ur.URAlgorithmParams.from_engine_json(engine)
    q = Q.UserQuery(eventNames=names)
    dev = user_check(ctx, data, ap, q, None)
    assert len(dev[2]) == len(users)
    user_check(ctx, data, ap, q, users[::-1] + ["nobody"], chunk=8191)
    user_check(ctx, data, ap, Q.UserQuery(eventNames=names[::-1]), users)


# ---- 5. more records than the grid has warps ----------------------------------------------------------------------------
def test_many_documents_per_warp(ctx):
    W = warps()
    body, ids = R.many_index(3 * W + 17)
    assert len(ids) > 3 * W and len(ids) * 3 > 3 * W   # records and (document, name) spans
    ap = params(eventNames=MODEL3, maxQueryEvents=4)
    docs = dict(Q.index_documents(body))
    expect = {i: (src if src else None) for i, src in docs.items()}
    item_check(ctx, body, ap, None, None, expect)
    rng = random.Random(5)
    items = ids[::-1] + rng.choices(ids, k=500) + ["unknown%d" % k for k in range(50)] + ["", ""]
    assert len(items) > 3 * W
    item_check(ctx, body, ap, Q.ItemQuery(blacklistItems=ids[:40:3]), items, expect)


def test_many_users_per_warp(ctx):
    W = warps()
    data = R.many_export(3 * W + 5, 240_000)
    ap = params(indicators=[{"name": "buy", "maxItemsPerUser": 3}, {"name": "view", "maxItemsPerUser": 33}, {"name": "like"}],
                blacklistEvents=["like", "buy"])
    dev = user_check(ctx, data, ap, None, None)
    assert len(dev[2]) > 3 * W
    users = ["u%d" % k for k in random.Random(6).sample(range(3 * W + 5), 3 * W + 5)] + ["nobody", "u0"]
    user_check(ctx, data, ap, Q.UserQuery(blacklistItems=["i1\u2028", "i2\u2028", "i3"]), users)
