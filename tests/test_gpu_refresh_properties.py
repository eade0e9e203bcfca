"""Item properties refreshed in the live index on the H100 (cco_refresh_properties): every output of the device -- the
refreshed body, the delta, the delete lines, the counts and the document numbers -- equal to the host mirror
ur_model.refresh_documents byte for byte; a resident event log extended with property events refreshes a calcAll body
into the body calcAll writes from the extended log; update_index against the Elasticsearch fake of test_refresh_docs."""
import json
import random
import subprocess

import numpy as np
import pytest

import universal_recommender_b200 as ur
from index_pages_data import pages_of
from model_oracle import model_bulk
from test_refresh_docs import (FIELDS, NAMES, RANKS, FakeES, build_abi_check, by_field, docs_of, formatted, random_model,
                               random_props)
from test_event_window import DAY, NOW
from test_events_mirror import iso_ms
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_model as um
from universal_recommender_b200.similarity_analysis import encode_ids

pytestmark = pytest.mark.gpu


def props_of(triples):
    """(item, field, JSON text) triples -> CcoContext's properties argument, fields numbered by first appearance"""
    if not triples:
        return None
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    fidx = {f: k for k, f in enumerate(fields)}
    return (fields, *encode_ids([i for i, _, _ in triples]), [fidx[f] for _, f, _ in triples], *encode_ids([v for _, _, v in triples]))


def check(ctx, body, triples, correlators=NAMES, rankings=RANKS):
    got = ctx.refresh_properties(body, correlators, rankings, properties=props_of(triples))
    want = um.refresh_documents(body, correlators, rankings, [(i, f, um.RawJson(v)) for i, f, v in triples])
    assert got == want
    return got


@pytest.mark.parametrize("seed", range(6))
def test_seeded_models_match_the_mirror(ctx, seed):
    model = random_model(seed)
    p, p2 = by_field(random_props(seed, model[4])), by_field(random_props(seed + 100, model[4]))
    got = check(ctx, formatted(model, p), p2 + [(f"new{seed}", "size", '"S"')])
    assert got.n_changed and got.n_new and got.n_deleted
    same = check(ctx, formatted(model, p), p)   # the fixed point
    assert same.body == formatted(model, p) and same.delta == b"" and same.deletes == b""


def test_handmade_documents_match_the_mirror(ctx):
    body = (b'{"index":{"_id":"a"}}\n{"id":"other","purchase":["x"],"color":"red","purchase":["y"],"popRank":1.0,"popRank":2.0}\n'
            b'{"index":{"_index":"i","_id":"b","_id":"b2"}}\n{"color":"red","id":"b2"}\n'
            b'{"index":{"_id":"c\\u00e9"}}\r\n{ "vi\\"ew" : [ "q" ] , "trendRank":3.0 }\r\n'
            b'{"index":{"_id":"d"}}\n{}\n')
    check(ctx, body, [("a", "color", '"red"'), ("cé", "id", "null"), ("e", "cat\\egory", "[1,{\"k\":\"v\"}]"), ("a", "color", '"blue"')])
    check(ctx, body, [])


def test_an_empty_body_and_no_triples(ctx):
    got = check(ctx, b"", [("a", "color", '"red"'), ("b", "id", "null")])
    assert got.n_new == 2 and got.body == got.delta
    assert check(ctx, b"", []).body == b""
    model = random_model(7)
    old = formatted(model, random_props(7, model[4]))
    gone = check(ctx, old, [])
    assert gone.n_deleted == sum(1 for s in docs_of(old).values() if not any(n in json.loads(s) for n in NAMES + RANKS))


@pytest.mark.parametrize("n", [31, 32, 33, 70])
def test_documents_with_many_members(ctx, n):
    rng = random.Random(n)
    names = NAMES + RANKS + ["o1", "o2", "id", "color"]
    docs = []
    for d in range(5):
        values = ["[]", "1.0", '["x"]', '{"a":[1]}']
        members = [um.json_string(rng.choice(names)) + ":" + rng.choice(values) for _ in range(n + d)]
        docs.append(b'{"index":{"_id":"d%d"}}\n{%s}\n' % (d, ",".join(members).encode()))
    check(ctx, b"".join(docs), [("d1", "color", '"red"'), ("d3", "size", "2"), ("z", "price", "1")])


@pytest.mark.parametrize("page_hits", [0, 7])
def test_bodies_read_back_from_pages(ctx, page_hits):
    model = random_model(11)
    p = by_field(random_props(11, model[4]))
    body = ur.index_from_pages(pages_of(formatted(model, p), page_hits, 3, pretty=page_hits > 0), ctx=ctx)
    check(ctx, body, by_field(random_props(12, model[4])))


def test_a_property_named_like_a_correlator_is_refused(ctx):
    with pytest.raises(N.CcoError, match='"purchase" is named like a correlator'):
        ctx.refresh_properties(b"", NAMES, RANKS, properties=props_of([("a", "purchase", "1")]))


def test_a_hundred_thousand_documents(ctx):
    rng = np.random.default_rng(5)
    n = 100_000
    rows = [f"item{k}" for k in range(n)]
    ind = []
    for _ in NAMES:
        cnt = rng.integers(0, 6, n)
        rp = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        ind.append((rp, rng.integers(0, n, int(rp[-1])).astype(np.int32)))
    fields = ["color", "price", "id"]
    pick = rng.integers(0, n + 5000, 60_000)
    p = sorted([(f"item{k}", int(rng.integers(0, 3)), '"c%d"' % rng.integers(0, 9)) for k in pick], key=lambda t: t[1])
    body = model_bulk(ind, NAMES, rows, [rows, rows], fields, p, [])
    changed = [(i, fields[f], v) for i, f, v in p]
    for k in rng.integers(0, len(changed), 3000):
        changed[k] = (changed[k][0], changed[k][1], '"fresh"')
    got = check(ctx, body, by_field_names(changed + [("brand-new", "price", "1")], fields))
    assert got.n_changed > 1000 and got.n_new == 1


def by_field_names(triples, fields):
    return sorted(triples, key=lambda t: fields.index(t[1]))


AP = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy", "view"], "seed": 1, "rankings": [
    {"name": "popRank", "type": "popular", "eventNames": ["buy", "view"], "duration": "3650 days"}]})


def event(name, etype, eid, t, target=None, props=None) -> bytes:
    r = {"event": name, "entityType": etype, "entityId": eid, "eventTime": iso_ms(t)}
    if target is not None:
        r.update(targetEntityType="item", targetEntityId=target)
    if props is not None:
        r["properties"] = props
    return json.dumps(r).encode() + b"\n"


def test_a_resident_log_extended_with_property_events(ctx):
    rng = random.Random(3)
    items = [f"i{k}" for k in range(40)]
    a = b"".join(event(rng.choice(["buy", "view"]), "user", f"u{rng.randrange(30)}", NOW - rng.randrange(9 * DAY), rng.choice(items))
                 for _ in range(800))
    a += b"".join(event("$set", "item", rng.choice(items), NOW - rng.randrange(9 * DAY), props={f: rng.choice([1, "x", [1, 2]])
                        for f in rng.sample("abcd", rng.randint(0, 3))}) for _ in range(60))
    b = []
    for _ in range(80):
        kind, it = rng.choice(["$set", "$set", "$unset", "$delete"]), rng.choice(items + ["n1", "n2"])
        props = None if kind == "$delete" else {f: rng.choice([2, "y", {"z": 1}]) for f in rng.sample("abce", rng.randint(1, 2))}
        b.append(event(kind, "item", it, NOW - rng.randrange(DAY), props=props))
    with ctx.read_events(a, now_ms=NOW, extendable=True) as log:
        b0 = ur.calc_all_from_events(log, AP, now_ms=NOW, ctx=ctx)
        log.extend(b"".join(b), now_ms=NOW)
        got = ur.refresh_properties_from_events(b0, log, AP, now_ms=NOW, ctx=ctx)
        want = ur.calc_all_from_events(log, AP, now_ms=NOW, ctx=ctx)
        assert docs_of(got.body) == docs_of(want)
        assert got.n_changed + got.n_new + got.n_deleted > 0
        again = ur.refresh_properties_from_events(got.body, log, AP, now_ms=NOW, ctx=ctx)   # the log stays usable
        assert again.body == got.body and again.delta == b"" and again.deletes == b""


def test_refresh_on_device_takes_set_events(ctx):
    body = b'{"index":{"_id":"a"}}\n{"id":"a","buy":["b"],"color":"red","popRank":1.0}\n'
    got = ur.refresh_properties_on_device(body, [("a", {"color": "blue"}), ("c", {})], AP, ctx=ctx)
    assert got.body == (b'{"index":{"_id":"a"}}\n{"id":"a","buy":["b"],"color":"blue","popRank":1.0}\n'
                        b'{"index":{"_id":"c"}}\n{"id":"c"}\n')


def test_update_index_end_to_end_with_429_rounds(ctx):
    model = random_model(21, n_rows=40)
    p = by_field(random_props(21, model[4], 120))
    body = formatted(model, p)
    es = FakeES({"urindex_7": {i: s.decode("utf-8", "surrogatepass") for i, s in docs_of(body).items()}})
    r = ctx.refresh_properties(body, NAMES, RANKS, properties=props_of(by_field(random_props(22, model[4], 120))))
    es.reject = set(list(docs_of(r.delta))[::3])
    ap = ur.URAlgorithmParams(eventNames=NAMES, indexName="urindex", typeName="items",
                              rankings=[um.RankingParams(n, m, None, None, None, "1 day") for n, m in zip(RANKS, ["popular", "trending"])])
    index, result = ur.update_index(r, ap, es, max_docs=5, max_bytes=1 << 12, retry_wait_s=0, ctx=ctx)
    assert index == "urindex_7" and result.n_rejected == 0 and not es.reject
    # what write_index of the refreshed full body writes: every document of the body, and no other
    assert {i: s.encode("utf-8", "surrogatepass") for i, s in es.docs["urindex_7"].items()} == docs_of(r.body)
    assert ("PUT", "/urindex_7/_mapping/items") not in es.log or set(es.props["urindex_7"]) >= set(FIELDS) - {"id"}


def test_c_program_refreshes_on_the_device(tmp_path):
    out = subprocess.run([build_abi_check(tmp_path), "run"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout == "ok\n", out.stdout + out.stderr
