"""cco_item_queries against the host mirror (ur_query.item_queries over the same index body): byte-identical bodies on the
handmade index for every golden template, on indexes the device wrote from seeded random exports (before and after a
re-rank, with property-only documents), on a hostile hand-built body and on an empty one; the error cases."""
import ctypes as C
import json
import random

import numpy as np
import pytest

import universal_recommender_b200 as ur
from universal_recommender_b200 import CcoContext
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_query as Q
from conftest import load_golden
from user_query_data import handmade_params, random_export

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000_000


@pytest.fixture(scope="module")
def ctx():
    c = CcoContext()
    yield c
    c.close()


def check(ctx, body, ap, q, items):
    dev = ctx.item_queries(body, ap, q, items, NOW)
    host = Q.item_queries(body, ap, q, items, NOW)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    if items is None:
        assert dev[2] == host[2]
    return dev


def test_handmade_every_template(ctx):
    fx = load_golden("item_queries_handmade.json")
    body = fx["index"].encode()
    items = fx["items"] + ["Iphone 4", "", "Surface", "xyz"]
    for tpl in fx["queries"]:
        q = Q.ItemQuery.from_json(tpl)
        check(ctx, body, handmade_params(), q, items)
        check(ctx, body, handmade_params(), q, None)
    out, off = check(ctx, body, handmade_params(), None, ["Iphone 4"])
    assert out == b"{}\n" + fx["iphone4_default"].encode() + b"\n"


@pytest.mark.parametrize("over", [dict(userBias=-1), dict(itemBias=-1), dict(itemBias=2.5, returnSelf=True), dict(recsModel="collabFiltering"),
                                  dict(indicators=None, eventNames=["purchase", "view"], maxQueryEvents=2),
                                  dict(indicators=None, eventNames=["view", "purchase", "category-pref"], maxQueryEvents=1)])
def test_handmade_params(ctx, over):
    fx = load_golden("item_queries_handmade.json")
    q = Q.ItemQuery(blacklistItems=["Galaxy", "x", "Nexus", "x"], itemBias=0.5)
    check(ctx, fx["index"].encode(), handmade_params(**over), q, fx["items"] + ["Nexus", "Nexus"])
    check(ctx, fx["index"].encode(), handmade_params(**over), None, None)


def with_properties(export: bytes, seed: int) -> bytes:
    """$set lines for some traded items and for items with no event (property-only documents)"""
    rng = random.Random(seed)
    lines = [json.dumps({"event": "$set", "entityType": "item", "entityId": i, "properties": {"colour": [rng.choice("rgb")]},
                         "eventTime": Q.iso_utc(1_600_000_000_000 + k)}, ensure_ascii=False)
             for k, i in enumerate(["i1", "i2", "prop-only", "p\u2028\"o", "i" + chr(0x1F600)])]
    return export + ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_indexes_written_on_the_device(ctx, seed):
    export = with_properties(random_export(seed), seed)
    ap = ur.URAlgorithmParams.from_engine_json({"indicators": [{"name": "buy", "maxItemsPerUser": 5}, {"name": "view", "maxItemsPerUser": 3},
                                                               {"name": "like"}], "maxQueryEvents": 40})
    index = ur.calc_all_from_events(export, ap, now_ms=NOW, ctx=ctx)
    reranked = ur.calc_pop_from_events(index, export, ap, now_ms=NOW + 1000, ctx=ctx)
    small = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy", "view", "like"], "maxQueryEvents": 3, "itemBias": 1.5})
    docs = Q.index_documents(index)
    ids = [i for i, _ in docs]
    items = ids[::3] + ["absent", ids[0], "", "prop-only"] + ids[:5]
    q = Q.ItemQuery(blacklistItems=ids[:6:2] + ["nope", ids[0]], userBias=2)
    for body in (index, reranked):
        check(ctx, body, ap, q, items)
        check(ctx, body, ap, None, None)
        check(ctx, body, small, Q.ItemQuery(returnSelf=True, eventNames=["view"]), None)


def hostile_body() -> bytes:
    ids = ['q"uote', "back\\slash", "ctl\x01\x1f\b\f\n\r\t", "c1\u0085", "ls\u2028ps\u2029", "emoji\U0001f600", "plain"]
    out = []
    for k, i in enumerate(ids):
        out.append(json.dumps({"index": {"_index": "urindex", "_id": i}}, ensure_ascii=bool(k % 2)))
        out.append(json.dumps({"purchase": ids[k:] + ["\u00e9"], "id": i, "view": [x + "!" for x in ids[:k]]}, ensure_ascii=bool(k % 3)))
    out += ['{ "index" : {\r\t "_id" : "esc\\u00e9\\/x\\ud83d\\ude00" , "_type":"items"} }',
            '{\t"view" : [ "a" ,\r"b\\"c" ] , "popRank":2.0, "purchase":[ ] }',
            '{"index":{"_id":"lone\\ud800"}}', '{"category-pref":["s\\udc00", "\\u20ac\\u0085"],"purchase":["x"],"purchase":["y"]}',
            '{"index":{"_id":""}}', '{}',
            '{"index":{"_id":"no-fields"}}', '{"id":"no-fields","defaultRank":1.5}']
    return ("\n".join(out) + "\n").encode("utf-8", "surrogatepass")


def test_hostile_body(ctx):
    body = hostile_body()
    docs = Q.index_documents(body)
    ids = [i for i, _ in docs]
    assert "esc\u00e9/x\U0001f600" in ids and "lone\ud800" in ids
    ap = handmade_params(indicators=None, eventNames=["purchase", "view", "category-pref"], maxQueryEvents=3)
    items = ids + ids[::-1] + ["unknown", "", "lone\ud800", "esc\u00e9/x\ud83d\ude00"]
    for q in (None, Q.ItemQuery(blacklistItems=ids[:3] + ["plain"]), Q.ItemQuery(returnSelf=True, itemBias=7)):
        check(ctx, body, ap, q, items)
        check(ctx, body, ap, q, None)
    check(ctx, body, handmade_params(itemBias=-2, userBias=-1), None, items)


def test_empty_body(ctx):
    ap = handmade_params()
    body, off, items = check(ctx, b"", ap, None, None)
    assert body == b"" and list(off) == [0] and items == []
    check(ctx, b"", ap, Q.ItemQuery(blacklistItems=["a"]), ["a", "b", ""])
    body, off = ctx.item_queries(b"", ap, None, [], NOW)
    assert body == b"" and list(off) == [0]


def raw_call(ctx, body, q, items=None):
    L = N.lib()
    out, ln, off, n = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
    if items is None:
        rc = L.cco_item_queries(ctx._h, body, len(body), C.byref(q), 0, None, None, C.byref(out), C.byref(ln), C.byref(off), C.byref(n), None)
    else:
        io, ib = items
        rc = L.cco_item_queries(ctx._h, body, len(body), C.byref(q), len(io) - 1, io.ctypes.data_as(C.POINTER(C.c_int64)), C.cast(ib, C.c_void_p),
                                C.byref(out), C.byref(ln), C.byref(off), C.byref(n), None)
    if rc == N.OK:
        L.cco_host_free(ctx._h, out)
        L.cco_host_free(ctx._h, off)
    return rc, L.cco_last_error().decode()


def test_errors(ctx):
    nm = (C.c_char_p * 2)(b"purchase", b"view")
    ok = np.array([0, 1], dtype=np.int64)
    bad = np.array([0, 4, 2], dtype=np.int64)
    blob = C.create_string_buffer(b"abcd")

    def q(**kw):
        d = dict(n_names=2, names=nm, max_query_events=3, similar_in_must=0, similar_boost=None, exclude_self=1, head=b'{"from":0,"size":1',
                 should_head=b"", should=b"{}", must_head=b"", must=b"", must_not=b"", sort=b"[]", header=b"{}", n_blacklist_items=0,
                 blacklist_item_offsets=ok.ctypes.data_as(C.POINTER(C.c_int64)), blacklist_item_bytes=None)
        d.update(kw)
        return N.ItemQueryT(**d)
    good = b'{"index":{"_id":"a"}}\n{"purchase":["x"]}\n{"index":{"_id":"b"}}\n{"purchase":"x"}\n'
    assert raw_call(ctx, good, q(), (ok, blob))[0] == N.OK   # b, whose member is bad, is not queried
    rc, msg = raw_call(ctx, good, q())
    assert rc == N.E_INVALID_ARG and 'document 1: its "purchase" member is not an array of strings' in msg
    for src in (b'["x",]', b'[,"x"]', b'["x" "y"]', b'[1]', b'null', b'{"a":["x"]}', b'[["x"]]'):
        body = b'{"index":{"_id":"a"}}\n{"view":' + src + b'}\n'
        rc, msg = raw_call(ctx, body, q())
        assert rc == N.E_INVALID_ARG and '"view" member' in msg, src
    rc, msg = raw_call(ctx, good + b'{"index":{"_id":"a"}}\n{}\n', q(), (ok, blob))
    assert rc == N.E_INVALID_ARG and "document 2: its _id is the _id of document 0" in msg
    for body in (b'{"index":{"_id":"a"}}\n{}', b'{"index":{"_id":"a"}}\n', b'{"create":{"_id":"a"}}\n{}\n', b'{"index":{"_id":1}}\n{}\n',
                 b'{"index":{"_id":"a"}}\n[]\n', b'{"index":{"_id":"a"}}\n{"x":"\\q"}\n'):
        rc, msg = raw_call(ctx, body, q())
        assert rc == N.E_INVALID_ARG, body
        with pytest.raises(N.CcoInvalidArgument) as e:
            ctx.rerank_model(body)
        assert msg in str(e.value)   # the messages of cco_rerank_model
    assert raw_call(ctx, good, q(), (bad, blob))[0] == N.E_INVALID_ARG
    assert raw_call(ctx, good, q(n_blacklist_items=2, blacklist_item_offsets=bad.ctypes.data_as(C.POINTER(C.c_int64)),
                                 blacklist_item_bytes=C.cast(blob, C.c_void_p)), (ok, blob))[0] == N.E_INVALID_ARG
    assert raw_call(ctx, good, q(n_names=0), (ok, blob))[0] == N.E_INVALID_ARG
    assert raw_call(ctx, good, q(n_names=65), (ok, blob))[0] == N.E_INVALID_ARG
    assert raw_call(ctx, good, q(names=(C.c_char_p * 2)(b"purchase", b"")), (ok, blob))[0] == N.E_INVALID_ARG
    assert raw_call(ctx, good, q(max_query_events=0), (ok, blob))[0] == N.E_INVALID_ARG
    assert raw_call(ctx, good, q(sort=None), (ok, blob))[0] == N.E_INVALID_ARG
    with pytest.raises(ValueError):
        Q.item_queries(good, handmade_params(), None, None, NOW)


def test_package_entry(ctx):
    fx = load_golden("item_queries_handmade.json")
    body, off, items = ur.item_queries(fx["index"].encode(), handmade_params(), None, None, NOW, ctx=ctx)
    host = Q.item_queries(fx["index"].encode(), handmade_params(), None, None, NOW)
    assert body == host[0] and items == host[2]
