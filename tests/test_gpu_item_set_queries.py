"""cco_item_set_queries against the host mirror (ur_query.item_set_queries over the same sets): byte-identical bodies and
offsets on every golden template, on seeded random batches of hostile ids, on sets around a warp's width and one of 10^5
elements, on repeats a warp or two apart, on zero and all-empty batches, on more sets than one launch has warps; the error
cases."""
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
from user_query_data import ODD, handmade_params

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000_000
OVERS = [dict(userBias=-1), dict(itemBias=-1), dict(itemBias=2.5, returnSelf=True), dict(recsModel="collabFiltering"),
         dict(indicators=None, eventNames=["purchase", "view"], maxQueryEvents=2),
         dict(indicators=None, eventNames=["view", "purchase", "category-pref"], maxQueryEvents=1)]   # test_gpu_item_queries.py's


@pytest.fixture(scope="module")
def ctx():
    c = CcoContext()
    yield c
    c.close()


def sets_params(**over):
    return ur.URAlgorithmParams.from_engine_json({**load_golden("item_set_queries_handmade.json")["params"], **over})


def arrow(sets):
    """the Arrow list<large_string> buffers of a batch"""
    enc = [x.encode("utf-8", "surrogatepass") for s in sets for x in s]
    so = np.zeros(len(sets) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in sets], out=so[1:])
    eo = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in enc], out=eo[1:])
    return so, eo, np.frombuffer(b"".join(enc), dtype=np.uint8)


def check(ctx, sets, ap, q=None, header="{}", buffers=False):
    dev = ctx.item_set_queries(arrow(sets) if buffers else sets, ap, q, NOW, header)
    host = Q.item_set_queries(sets, ap, q, NOW, header)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    return dev


def test_handmade_every_template(ctx):
    fx = load_golden("item_set_queries_handmade.json")
    sets = fx["sets"] + [[], ["iPhone 6", "iPhone 6", "AirPods"]]
    for ap in (sets_params(), handmade_params()):
        for tpl in fx["queries"]:
            check(ctx, sets, ap, Q.ItemSetQuery.from_json(tpl))
            check(ctx, sets, ap, Q.ItemSetQuery.from_json(tpl), buffers=True)
    body, off = check(ctx, fx["sets"], sets_params())
    assert body[off[-2]:off[-1]] == b"{}\n" + fx["last_set_default"].encode() + b"\n"


@pytest.mark.parametrize("over", OVERS)
def test_handmade_params_and_header(ctx, over):
    fx = load_golden("item_set_queries_handmade.json")
    q = Q.ItemSetQuery(blacklistItems=["AirPods", "x", "iPhone 6", "x"], itemSetBias=0.5)
    sets = fx["sets"] + [["x", "AirPods", "y", "x"], []]
    for header in ("{}", '{"index":"ur-item-sets-index","type":"items"}'):
        check(ctx, sets, handmade_params(**over), q, header)
        check(ctx, sets, handmade_params(**over), None, header, buffers=True)


def long_id(rng):
    """an id of exactly 1 500 UTF-8 bytes, escape classes first"""
    x = "L"
    while len(x.encode("utf-8")) < 1400:
        x += rng.choice(ODD)
    return x + "x" * (1500 - len(x.encode("utf-8")))


SIZES = [0, 1, 31, 32, 33, 64, 65]


def random_batch(seed, n_sets=300):
    """sets of every size in SIZES and random ones, ids drawn from a small pool of hostile ids (so sets repeat elements and
    share them with the blacklist)"""
    rng = random.Random(seed)
    pool = ["", long_id(rng), long_id(rng)] + ["".join(rng.choice(ODD) for _ in range(rng.randrange(4))) + str(k) for k in range(150)]
    sizes = SIZES + [rng.choice([0, 1, 2, 5, 17, 40, 70, 130]) for _ in range(n_sets - len(SIZES))]
    rng.shuffle(sizes)
    return [[rng.choice(pool) for _ in range(n)] for n in sizes], pool


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_hostile_batches(ctx, seed):
    sets, pool = random_batch(seed)
    lens = {len(s) for s in sets}
    assert all(n in lens for n in SIZES), "a set size of the list does not occur"
    used = {x for s in sets for x in s}
    assert "" in used and sum(len(x.encode("utf-8")) == 1500 for x in used) == 2
    assert any(len(set(s)) < len(s) for s in sets)
    rng = random.Random(seed)
    black = [rng.choice(pool) for _ in range(40)] + ["not-in-any-set"]
    for q in (None, Q.ItemSetQuery(blacklistItems=black, itemSetBias=1.05, userBias=2), Q.ItemSetQuery(itemSetBias=0, blacklistItems=black[:3]),
              Q.ItemSetQuery(itemSetBias=-1)):
        body, off = check(ctx, sets, handmade_params(), q)
        check(ctx, sets, sets_params(indicators=None, eventNames=["c \"t" + chr(0x1F600)]), q, buffers=True)
    for s in (0, 7, len(sets) - 1):
        h, text, _ = body[off[s]:off[s + 1]].decode("utf-8", "surrogatepass").split("\n")
        json.loads(text)


def test_one_set_of_1e5_elements_among_short_ones(ctx):
    rng = random.Random(5)
    big = [f"big{rng.randrange(60_000)}{rng.choice(ODD)}" for _ in range(100_000)]
    sets = [["a"], [], big, ["b", "a"], big[:3]]
    body, off = check(ctx, sets, handmade_params(), Q.ItemSetQuery(blacklistItems=big[:10] + ["a"]))
    b = json.loads(body[off[2]:off[3]].decode("utf-8", "surrogatepass").split("\n")[1])["query"]["bool"]
    assert b["should"][3]["terms"]["purchase"] == big
    check(ctx, sets, sets_params(), None, buffers=True)


@pytest.mark.parametrize("gap", [1, 32, 64])
def test_repeats_a_warp_apart(ctx, gap):
    s = [f"e{k}" for k in range(gap)] * 3 + ["e0"]
    sets = [s, s[1:], ["r"] * (gap + 1), [f"x{k}" for k in range(gap)] + ["x0"] + [f"x{k}" for k in range(gap)]]
    body, off = check(ctx, sets, sets_params())
    b = json.loads(body[off[0]:off[1]].decode().split("\n")[1])["query"]["bool"]
    assert b["must_not"][0]["ids"]["values"] == [f"e{k}" for k in range(gap)]
    check(ctx, sets, sets_params(), Q.ItemSetQuery(blacklistItems=["e1", "r", "x5"]))


def test_zero_sets_and_all_empty_sets(ctx):
    body, off = check(ctx, [], sets_params())
    assert body == b"" and list(off) == [0]
    check(ctx, [], sets_params(), buffers=True)
    check(ctx, [[]] * 100, sets_params())
    check(ctx, [[]] * 100, handmade_params(), Q.ItemSetQuery(blacklistItems=["a", "b", "a"]), buffers=True)


def test_more_sets_than_one_launch_has_warps(ctx):
    import torch
    warps = torch.cuda.get_device_properties(0).multi_processor_count * 64   # grid_for's cap: 8 blocks per SM of 8 warps
    n = 3 * warps + 17
    assert n > 3 * warps
    rng = random.Random(9)
    sets = [[f"i{rng.randrange(500)}" for _ in range(rng.randrange(4))] for _ in range(n)]
    check(ctx, sets, handmade_params(), Q.ItemSetQuery(blacklistItems=["i1", "i2"]), buffers=True)


def test_package_entry(ctx):
    fx = load_golden("item_set_queries_handmade.json")
    body, off = ur.item_set_queries(fx["sets"], sets_params(), None, NOW, ctx=ctx)
    host = Q.item_set_queries(fx["sets"], sets_params(), None, NOW)
    assert body == host[0] and np.array_equal(off, host[1])
    with pytest.raises(ValueError):
        ctx.item_set_queries([["a"]], ur.URAlgorithmParams.from_engine_json({"eventNames": []}), None, NOW)


def raw_call(ctx, q, so, eo, eb, n_elements=None):
    L = N.lib()
    out, ln, off, n = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
    p64 = C.POINTER(C.c_int64)
    rc = L.cco_item_set_queries(ctx._h, C.byref(q), len(so) - 1, so.ctypes.data_as(p64), len(eo) - 1 if n_elements is None else n_elements,
                                eo.ctypes.data_as(p64), C.cast(eb, C.c_void_p), C.byref(out), C.byref(ln), C.byref(off), C.byref(n))
    if rc == N.OK:
        L.cco_host_free(ctx._h, out)
        L.cco_host_free(ctx._h, off)
    return rc, L.cco_last_error().decode()


def test_errors(ctx):
    ok1 = np.array([0, 1], dtype=np.int64)
    blob = C.create_string_buffer(b"abcdefgh")
    so, eo = np.array([0, 1, 3], dtype=np.int64), np.array([0, 2, 4, 8], dtype=np.int64)

    def q(**kw):
        d = dict(name=b"purchase", with_set=1, boost=None, head=b'{"from":0,"size":1', should_head=b"", should_tail=b"{}", must=b"",
                 must_not=b"", sort=b"[]", header=b"{}", n_blacklist_items=1, blacklist_item_offsets=ok1.ctypes.data_as(C.POINTER(C.c_int64)),
                 blacklist_item_bytes=C.cast(blob, C.c_void_p))
        d.update(kw)
        return N.ItemSetQueryT(**d)
    assert raw_call(ctx, q(), so, eo, blob)[0] == N.OK
    # non-monotone set offsets (a middle offset past the last), decided on the device
    rc, msg = raw_call(ctx, q(), np.array([0, 9, 3], dtype=np.int64), eo, blob)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    rc, msg = raw_call(ctx, q(), np.array([0, 2, 1, 3], dtype=np.int64), eo, blob)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    # element offsets that decrease, one of them past the end of the bytes
    rc, msg = raw_call(ctx, q(), so, np.array([0, 1 << 40, 4, 8], dtype=np.int64), blob)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    rc, msg = raw_call(ctx, q(), so, np.array([0, 5, 4, 8], dtype=np.int64), blob)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    # blacklist item offsets that decrease
    bad = np.array([0, 6, 2], dtype=np.int64)
    rc, msg = raw_call(ctx, q(n_blacklist_items=2, blacklist_item_offsets=bad.ctypes.data_as(C.POINTER(C.c_int64))), so, eo, blob)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    # the last set offset beyond the element count, a negative first one, first after last
    assert raw_call(ctx, q(), np.array([0, 1, 4], dtype=np.int64), eo, blob)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, q(), so, eo, blob, n_elements=2)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, q(), np.array([-1, 1, 3], dtype=np.int64), eo, blob)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, q(), np.array([3, 1, 2], dtype=np.int64), eo, blob)[0] == N.E_INVALID_ARG
    # fragments and the name
    for f in ("head", "should_head", "should_tail", "must", "must_not", "sort", "header"):
        rc, msg = raw_call(ctx, q(**{f: None}), so, eo, blob)
        assert rc == N.E_INVALID_ARG and "null fragment" in msg, f
    assert raw_call(ctx, q(name=None), so, eo, blob)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, q(name=b""), so, eo, blob)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, q(name=None, with_set=0), so, eo, blob)[0] == N.OK
    assert raw_call(ctx, q(with_set=2), so, eo, blob)[0] == N.E_INVALID_ARG
    # a later good call is unaffected
    assert raw_call(ctx, q(), so, eo, blob)[0] == N.OK
