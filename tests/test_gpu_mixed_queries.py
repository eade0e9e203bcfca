"""cco_mixed_queries against the host mirror (ur_query.mixed_queries over the same export, index and rows): byte-identical
bodies and offsets on every golden template for all eight member combinations, on seeded exports and the indexes
calc_all_from_events writes from them, on hostile ids in every column, on every source's list around a warp's width, on
one id repeated in all four sources at lanes 0, 31 and 32, on validity bitmaps, zero rows and more rows than one launch
has warps; rows with one member against the three single device builders; the error cases.  Records are also decoded
and their lists compared with a restatement built from tests/query_edges_ref.py."""
import ctypes as C
import json
import random

import numpy as np
import pytest

import universal_recommender_b200 as ur
from universal_recommender_b200 import CcoContext
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_query as Q
from conftest import load_golden
from query_edges_ref import event_line, expected_similar, export, history_ref, index_body, source
from user_query_data import ODD, handmade_export, handmade_params, random_export

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000_000
COMBOS = [(u, i, s) for u in (0, 1) for i in (0, 1) for s in (0, 1)]


@pytest.fixture(scope="module")
def ctx():
    c = CcoContext()
    yield c
    c.close()


@pytest.fixture(scope="module")
def hand(ctx):
    """(log, host events, index) of the handmade data"""
    log = ctx.read_events(handmade_export(), keep_history=True)
    yield log, E.read_export(handmade_export()), load_golden("item_queries_handmade.json")["index"].encode()
    log.free()


def arrow_strings(col):
    """a column of str / None -> the Arrow large_string buffers with a validity bitmap (None when every row has one)"""
    enc = [b"" if x is None else x.encode("utf-8", "surrogatepass") for x in col]
    off = np.zeros(len(enc) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in enc], out=off[1:])
    valid = None if all(x is not None for x in col) else np.packbits(np.array([x is not None for x in col]), bitorder="little")
    return off, b"".join(enc), valid


def arrow_sets(col):
    flat = [x for s in col if s is not None for x in s]
    so = np.zeros(len(col) + 1, dtype=np.int64)
    np.cumsum([0 if s is None else len(s) for s in col], out=so[1:])
    eo, eb, _ = arrow_strings(flat)
    valid = None if all(s is not None for s in col) else np.packbits(np.array([s is not None for s in col]), bitorder="little")
    return so, eo, eb, valid


def check(ctx, log, ev, index, users, items, sets, ap, q=None, header="{}", buffers=False):
    args = (users, items, sets)
    if buffers:
        args = (None if users is None else arrow_strings(users), None if items is None else arrow_strings(items),
                None if sets is None else arrow_sets(sets))
    dev = ctx.mixed_queries(log, index, ap, q, *args, now_ms=NOW, header=header)
    host = Q.mixed_queries(ev, index, ap, q, users, items, sets, NOW, header)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    return dev


def combo_rows(users, items, sets, n):
    """n rows cycling through the eight member combinations"""
    out = ([], [], [])
    for r in range(n):
        hu, hi, hs = COMBOS[r % 8]
        out[0].append(users[r % len(users)] if hu else None)
        out[1].append(items[r % len(items)] if hi else None)
        out[2].append(sets[r % len(sets)] if hs else None)
    return out


def test_handmade_every_template_every_combination(ctx, hand):
    log, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    users, items, sets = combo_rows(fx["users"], fx["items"], [["Iphone 6", "Soap"], [], ["Galaxy", "Iphone 4", "Galaxy"]], 24)
    for k, ap in enumerate((handmade_params(), handmade_params(userBias=-1, itemBias=-1, recsModel="collabFiltering"))):
        for t, tpl in enumerate(fx["queries"]):
            q = Q.MixedQuery.from_json(tpl)
            check(ctx, log, ev, index, users, items, sets, ap, q, buffers=(t + k) % 2 == 1)
            rs = [tuple(r) for r in fx["rows"]]
            check(ctx, log, ev, index, [r[0] for r in rs], [r[1] for r in rs], [r[2] for r in rs], ap, q)
    body, off = ctx.mixed_queries(log, index, handmade_params(), None, ["u1"], ["Iphone 4"], None, now_ms=NOW)
    assert body == b"{}\n" + fx["u1_iphone4_default"].encode() + b"\n"


def test_single_member_rows_equal_the_device_builders(ctx, hand):
    log, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    users, items, sets = fx["users"], fx["items"], [["Iphone 6", "Soap", "Iphone 6"], [], ["x"], ["AirPods"], ["Nexus"], ["Galaxy"]]
    for ap in (handmade_params(), handmade_params(userBias=-1, itemBias=-1)):
        for tpl in fx["queries"]:
            q = Q.MixedQuery.from_json(tpl)
            assert ctx.mixed_queries(log, None, ap, q, users, now_ms=NOW)[0] == ctx.user_queries(log, ap, q, users, NOW)[0]
            assert ctx.mixed_queries(None, index, ap, q, items=items, now_ms=NOW)[0] == ctx.item_queries(index, ap, q, items, NOW)[0]
            assert ctx.mixed_queries(None, None, ap, q, item_sets=sets, now_ms=NOW)[0] == ctx.item_set_queries(sets, ap, q, NOW)[0]
            n = len(users)
            none = ctx.mixed_queries(log, index, ap, q, [None] * n, [None] * n, [None] * n, now_ms=NOW)
            assert none[0] == ctx.user_queries(log, ap, q, ["no such user"] * n, NOW)[0]
            mixed = ctx.mixed_queries(log, index, ap, q, [users[0], None, None], [None, items[0], None], [None, None, sets[0]], now_ms=NOW)
            single = (ctx.user_queries(log, ap, q, users[:1], NOW)[0] + ctx.item_queries(index, ap, q, items[:1], NOW)[0]
                      + ctx.item_set_queries(sets[:1], ap, q, NOW)[0])
            assert mixed[0] == single


def restate(ev_events, docs, p, users, items, sets):
    """each row's (should terms lists, excluded ids) from history_ref and expected_similar, not from the mirror"""
    by_user: dict = {}
    for line, (u, name, item, t) in enumerate(ev_events):
        by_user.setdefault(u, []).append((name, item, t, line))
    out = []
    for u, it, s in zip(users, items, sets):
        hist, black = history_ref(by_user.get(u, []) if u is not None else [], p.user.names, p.user.limits or [0] * len(p.user.names),
                                  p.user.blacklist, p.user.blacklist_items)
        lists = list(zip(p.user.names[:p.user.n_history], hist[:p.user.n_history]))
        if it is not None:
            lists += expected_similar(p.item.names, docs.get(it), p.item.max_query_events)
        if s is not None and p.with_set:
            lists.append((p.set_name, list(s)))
        ex = list(black) + ([it] if it is not None and p.item.exclude_self else []) + list(s or [])
        out.append((lists, list(dict.fromkeys(ex))))
    return out


def structure(body, off, expect):
    for r, (lists, excluded) in enumerate(expect):
        q = json.loads(body[off[r]:off[r + 1]].decode("utf-8", "surrogatepass").split("\n")[1])["query"]["bool"]
        terms = [c["terms"] for c in q["should"] if "terms" in c]
        got = [next((k, v) for k, v in t.items() if k != "boost") for t in terms]
        assert got == lists, r
        assert q["must_not"][0]["ids"]["values"] == excluded, r


def docs_of(index):
    return {i: (src if src else None) for i, src in Q.index_documents(index)}


@pytest.mark.parametrize("seed", [1, 2])
def test_seeded_exports_and_device_written_indexes(ctx, seed):
    exp = random_export(seed)
    ap = ur.URAlgorithmParams.from_engine_json({"indicators": [{"name": "buy", "maxItemsPerUser": 5}, {"name": "view", "maxItemsPerUser": 3},
                                                               {"name": "like"}], "maxQueryEvents": 40,
                                                "blacklistEvents": ["buy", "like"], "recsModel": "collabFiltering"})
    index = ur.calc_all_from_events(exp, ap, now_ms=NOW, ctx=ctx)
    ev = E.read_export(exp)
    log = ctx.read_events(exp, keep_history=True)
    try:
        rng = random.Random(seed)
        all_users = list(dict.fromkeys(u for u, _, _, _ in ev.events))
        ids = [i for i, _ in Q.index_documents(index)]
        users = [rng.choice(all_users + ["nobody"]) for _ in range(200)]
        items = [rng.choice(ids + ["absent", ""]) for _ in range(200)]
        sets = [[rng.choice(ids + ["s"]) for _ in range(rng.randrange(1, 21))] for _ in range(200)]
        users, items, sets = [[x if rng.random() < 0.6 else None for x in col] for col in (users, items, sets)]
        for q in (None, Q.MixedQuery(blacklistItems=ids[:5] + ["nope", ids[0]], itemSetBias=2, userBias=3),
                  Q.MixedQuery(returnSelf=True, eventNames=["view", "buy"], itemSetBias=0)):
            body, off = check(ctx, log, ev, index, users, items, sets, ap, q)
            structure(body, off, restate(ev.events, docs_of(index), Q.mixed_plan(ap, q, NOW), users, items, sets))
            check(ctx, log, ev, index, users, items, sets, ap, q, buffers=True)
    finally:
        log.free()


def long_id(rng):
    x = "L"
    while len(x.encode("utf-8")) < 1400:
        x += rng.choice(ODD)
    return x + "x" * (1500 - len(x.encode("utf-8")))


def test_hostile_ids_in_every_column(ctx):
    rng = random.Random(4)
    pool = ["", long_id(rng), long_id(rng), "e\u0085", "q\"\\", "t\t\n", "\U0001f600x", " "] + [
        "".join(rng.choice(ODD) for _ in range(3)) + str(k) for k in range(20)]
    named = pool[1:]   # events need non-empty ids
    lines = [event_line(named[k % 10], ["buy", "view"][k % 2], named[(k * 7) % len(named)], 1_600_000_000_000 + k * 1000, k) for k in range(300)]
    exp = export(lines)
    docs = [(pool[k], source([("buy", [pool[(k + j) % len(pool)] for j in range(k % 5)]), ("view", [pool[(k * 3) % len(pool)]])], k))
            for k in range(len(pool))]
    index = index_body(docs)
    ap = ur.URAlgorithmParams.from_engine_json({"indicators": [{"name": "buy"}, {"name": "view"}], "recsModel": "collabFiltering"})
    ev = E.read_export(exp)
    log = ctx.read_events(exp, keep_history=True)
    try:
        n = 64
        users_c = [rng.choice(pool) for _ in range(n)]
        items_c = [rng.choice(pool + ["absent"]) for _ in range(n)]
        sets_c = [[rng.choice(pool) for _ in range(rng.randrange(6))] for _ in range(n)]
        users_c, items_c, sets_c = combo_rows(users_c, items_c, sets_c, n)
        items_c[2], items_c[3], users_c[4], users_c[5], sets_c[1] = "", pool[1], pool[2], "", ["", pool[1], "\U0001f600x"]
        q = Q.MixedQuery(blacklistItems=pool[:6] + [pool[0]], itemSetBias=1.05)
        body, off = check(ctx, log, ev, index, users_c, items_c, sets_c, ap, q)
        structure(body, off, restate(ev.events, docs_of(index), Q.mixed_plan(ap, q, NOW), users_c, items_c, sets_c))
        check(ctx, log, ev, index, users_c, items_c, sets_c, ap, None, buffers=True)
    finally:
        log.free()


SIZES = [0, 1, 31, 32, 33, 64, 65]


def sized_data():
    """user hN has N distinct buy events (N items in its history and in its blacklist), document dN has N elements under
    each model name; the same id "dup" is at position P of user pP's history / blacklist, of document dP's lists"""
    base = 1_600_000_000_000
    lines, docs = [], []
    for n in SIZES:
        for j in range(n):   # newest first is j = 0: the history list is oldest first, the blacklist newest first
            lines.append(event_line("h%d" % n, "buy", "h%d-%d" % (n, j), base - j * 1000, j))
        docs.append(("d%d" % n, source([("buy", ["d%d-%d" % (n, j) for j in range(n)]), ("view", ["v%d" % j for j in range(n)])], n)))
    for p in (0, 31, 32):
        for j in range(40):
            lines.append(event_line("p%d" % p, "buy", "dup" if j == p else "p%d-%d" % (p, j), base - j * 1000, j))
        docs.append(("dp%d" % p, source([("buy", ["dup" if j == p else "x%d" % j for j in range(40)])], p)))
    docs.append(("dup", source([("buy", ["dup"])])))
    return export(lines), index_body(docs)


def test_every_source_around_a_warp(ctx):
    exp, index = sized_data()
    ap = ur.URAlgorithmParams.from_engine_json({"indicators": [{"name": "buy"}, {"name": "view"}], "recsModel": "collabFiltering",
                                                "maxQueryEvents": 1000})
    ev = E.read_export(exp)
    log = ctx.read_events(exp, keep_history=True)
    seen = {"history": set(), "similar": set(), "set": set(), "black": set()}
    try:
        users = ["h%d" % n for n in SIZES]
        items = ["d%d" % n for n in SIZES]
        sets = [["s%d" % j for j in range(n)] for n in SIZES]
        for nb in SIZES:
            q = Q.MixedQuery(blacklistItems=["b%d" % j for j in range(nb)])
            for rows in (COMBOS, [(1, 1, 1)]):
                us = [users[k % 7] if c[0] else None for k, c in enumerate(rows * 7)]
                its = [items[(k // 2) % 7] if c[1] else None for k, c in enumerate(rows * 7)]
                ss = [sets[(k // 3) % 7] if c[2] else None for k, c in enumerate(rows * 7)]
                body, off = check(ctx, log, ev, index, us, its, ss, ap, q)
                structure(body, off, restate(ev.events, docs_of(index), Q.mixed_plan(ap, q, NOW), us, its, ss))
                for r in range(len(us)):
                    b = json.loads(body[off[r]:off[r + 1]].decode().split("\n")[1])["query"]["bool"]
                    t = [c["terms"] for c in b["should"] if "terms" in c]
                    seen["history"].add(len(t[0]["buy"]))
                    if its[r] is not None:
                        seen["similar"].add(len(t[2]["buy"]))
                    if ss[r] is not None:
                        seen["set"].add(len(t[-1]["buy"]))
            seen["black"].add(nb)
        for k, v in seen.items():
            assert all(n in v for n in SIZES), (k, sorted(v))
        # one id in all four sources at lanes 0, 31 and 32
        for p in (0, 31, 32):
            filler = ["f%d" % j for j in range(40)]
            black = filler[:p] + ["dup"] + filler[p:]
            st = ["g%d" % j for j in range(p)] + ["dup"] + ["g%d" % j for j in range(40)]
            q = Q.MixedQuery(blacklistItems=black)
            us, its, ss = ["p%d" % p, None, "p%d" % p, None], ["dup", "dup", "dp%d" % p, None], [st, st, None, st]
            body, off = check(ctx, log, ev, index, us, its, ss, ap, q)
            structure(body, off, restate(ev.events, docs_of(index), Q.mixed_plan(ap, q, NOW), us, its, ss))
            ex = json.loads(body[off[0]:off[1]].decode().split("\n")[1])["query"]["bool"]["must_not"][0]["ids"]["values"]
            assert ex.count("dup") == 1 and ex.index("dup") == p
    finally:
        log.free()


def test_validity_bitmaps(ctx, hand):
    log, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    n = 70
    absent = {7, 8, 9, 63, 64, 65}
    rng = random.Random(3)
    users = [None if r in absent else rng.choice(fx["users"]) for r in range(n)]
    items = [None if r in absent else rng.choice(fx["items"]) for r in range(n)]
    sets = [None if r in absent else [rng.choice(fx["items"]) for _ in range(r % 4)] for r in range(n)]
    for cols in ((users, items, sets), (users, None, None), (None, items, None), (None, None, sets), (users, items, None)):
        check(ctx, log, ev, index, *cols, handmade_params(), None, buffers=True)
    full = [rng.choice(fx["users"]) for _ in range(n)]
    check(ctx, log, ev, index, full, [x or "Nexus" for x in items], [s or [] for s in sets], handmade_params(), None, buffers=True)
    # bytes under an absent row are never read as an id: the bitmap alone decides
    off, blob, valid = arrow_strings(["u1", "u1", "Iphone 4"])
    valid = np.array([0b101], dtype=np.uint8)
    body, o = ctx.mixed_queries(log, index, handmade_params(), None, (off, blob, valid), (off, blob, np.array([0b010], dtype=np.uint8)),
                                None, now_ms=NOW)
    host = Q.mixed_queries(ev, index, handmade_params(), None, ["u1", None, "Iphone 4"], [None, "u1", None], None, NOW)
    assert body == host[0] and np.array_equal(o, host[1])


def test_zero_rows(ctx, hand):
    log, ev, index = hand
    for cols in (([], [], []), (None, None, None), ([], None, None)):
        body, off = check(ctx, log, ev, index, *cols, handmade_params())
        assert body == b"" and list(off) == [0]
    body, off = ctx.mixed_queries(None, None, handmade_params(), None, now_ms=NOW)
    assert body == b"" and list(off) == [0]


def test_more_rows_than_one_launch_has_warps(ctx, hand):
    import torch
    log, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    warps = torch.cuda.get_device_properties(0).multi_processor_count * 64   # grid_for's cap: 8 blocks per SM of 8 warps
    n = 3 * warps + 17
    rng = random.Random(9)
    users, items, sets = combo_rows(fx["users"], fx["items"], [[rng.choice(fx["items"]) for _ in range(k % 5)] for k in range(50)], n)
    check(ctx, log, ev, index, users, items, sets, handmade_params(), Q.MixedQuery(blacklistItems=["Nexus", "Soap"]), buffers=True)


def test_package_entry(ctx, hand):
    _, ev, index = hand
    fx = load_golden("mixed_queries_handmade.json")
    body, off = ur.mixed_queries_from_events(handmade_export(), index, handmade_params(), None, ["u1", None], ["Iphone 4", "Nexus"],
                                             [None, ["Soap"]], now_ms=NOW, ctx=ctx)
    host = Q.mixed_queries(ev, index, handmade_params(), None, ["u1", None], ["Iphone 4", "Nexus"], [None, ["Soap"]], NOW)
    assert body == host[0] and np.array_equal(off, host[1])
    assert body[off[0]:off[1]] == b"{}\n" + fx["u1_iphone4_default"].encode() + b"\n"
    body, _ = ur.mixed_queries_from_events(None, None, handmade_params(), None, item_sets=[["a"]], now_ms=NOW, ctx=ctx)
    assert body == Q.mixed_queries(None, None, handmade_params(), None, None, None, [["a"]], NOW)[0]


# ---- errors ------------------------------------------------------------------------------------------------------------
def raw_call(ctx, log, body, q, n, users=None, items=None, sets=None, n_elements=None):
    L = N.lib()
    out, ln, off, nn = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
    p64 = C.POINTER(C.c_int64)
    ptr = lambda a: None if a is None else a.ctypes.data_as(p64)
    u = users or (None, None, None)
    i = items or (None, None, None)
    s = sets or (None, None, None, None)
    rc = L.cco_mixed_queries(ctx._h, log, body, 0 if body is None else len(body), C.byref(q), n, ptr(u[0]), u[1], u[2], ptr(i[0]), i[1], i[2],
                             ptr(s[0]), (len(s[1]) - 1 if s[1] is not None else 0) if n_elements is None else n_elements, ptr(s[1]), s[2], s[3],
                             C.byref(out), C.byref(ln), C.byref(off), C.byref(nn))
    if rc == N.OK:
        L.cco_host_free(ctx._h, out)
        L.cco_host_free(ctx._h, off)
    return rc, L.cco_last_error().decode()


def test_errors(ctx, hand):
    log, _, index = hand
    keep = []

    def names(*xs):
        a = (C.c_char_p * max(len(xs), 1))(*xs)
        keep.append(a)
        return a
    lim = np.array([100, 100], dtype=np.int32)
    no = np.zeros(1, dtype=np.int64)

    def q(**kw):
        d = dict(n_names=1, n_history_names=1, names=names(b"purchase"), limits=lim.ctypes.data_as(C.POINTER(C.c_int32)), n_blacklist_names=1,
                 history_in_must=0, blacklist_names=names(b"purchase"), history_boost=None, n_model_names=1, model_names=names(b"purchase"),
                 max_query_events=100, similar_in_must=0, similar_boost=None, exclude_self=1, set_name=b"purchase", with_set=1, set_boost=None,
                 head=b'{"from":0,"size":4', boosted=b"", should_tail=b"{}", must=b"", must_not=b"", sort=b"[]", header=b"{}",
                 n_blacklist_items=0, blacklist_item_offsets=no.ctypes.data_as(C.POINTER(C.c_int64)), blacklist_item_bytes=None)
        d.update(kw)
        return N.MixedQueryT(**d)
    blob = C.create_string_buffer(b"u1Iphone 4abcdefgh")
    addr = C.cast(blob, C.c_void_p).value
    uo = np.array([0, 2, 2], dtype=np.int64)
    io = np.array([2, 10, 10], dtype=np.int64)
    users, items = (uo, addr, None), (io, addr, None)
    so, eo = np.array([0, 1, 2], dtype=np.int64), np.array([10, 12, 14], dtype=np.int64)
    sets = (so, eo, addr, None)
    lh = log._h
    assert raw_call(ctx, lh, index, q(), 2, users, items, sets)[0] == N.OK
    assert raw_call(ctx, None, None, q(), 2, None, None, sets)[0] == N.OK           # no user, no item: neither log nor body
    assert raw_call(ctx, None, b"", q(), 2, None, items, sets)[0] == N.OK           # an empty body: every item unknown
    # a row with a user but no log, or a log without history; a row with an item but no body
    rc, msg = raw_call(ctx, None, index, q(), 2, users, items)
    assert rc == N.E_INVALID_ARG and "needs a log" in msg
    plain = ctx.read_events(handmade_export())
    try:
        rc, msg = raw_call(ctx, plain._h, index, q(), 2, users)
        assert rc == N.E_INVALID_ARG and "without history retention" in msg
        assert raw_call(ctx, plain._h, index, q(), 2, None, items)[0] == N.OK   # no user row: the log is not read
    finally:
        plain.free()
    rc, msg = raw_call(ctx, lh, None, q(), 2, users, items)
    assert rc == N.E_INVALID_ARG and "need an index body" in msg
    # validity bitmaps decide: no row has a user or an item
    zero = C.create_string_buffer(b"\x00")
    zaddr = C.cast(zero, C.c_void_p).value
    assert raw_call(ctx, None, None, q(), 2, (uo, addr, zaddr), (io, addr, zaddr))[0] == N.OK
    # a log of another context
    other = CcoContext()
    try:
        olog = other.read_events(handmade_export(), keep_history=True)
        try:
            rc, msg = raw_call(ctx, olog._h, index, q(), 2, users)
            assert rc == N.E_INVALID_ARG and "another context" in msg
        finally:
            olog.free()
    finally:
        other.close()
    # decreasing offsets in each column, decided on the device
    for bad in ((np.array([0, 2, 1], dtype=np.int64), addr, None),):
        rc, msg = raw_call(ctx, lh, index, q(), 2, bad, items, sets)
        assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
        rc, msg = raw_call(ctx, lh, index, q(), 2, users, (np.array([2, 1 << 40, 10], dtype=np.int64), addr, None), sets)
        assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    rc, msg = raw_call(ctx, lh, index, q(), 2, users, items, (np.array([0, 3, 2], dtype=np.int64), eo, addr, None), n_elements=2)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    rc, msg = raw_call(ctx, lh, index, q(), 2, users, items, (so, np.array([10, 9, 14], dtype=np.int64), addr, None))
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    bl = np.array([0, 6, 2], dtype=np.int64)
    rc, msg = raw_call(ctx, lh, index, q(n_blacklist_items=2, blacklist_item_offsets=bl.ctypes.data_as(C.POINTER(C.c_int64)),
                                         blacklist_item_bytes=addr), 2, users, items, sets)
    assert rc == N.E_INVALID_ARG and "decreasing offsets" in msg
    # set offsets outside [0, n_elements]
    assert raw_call(ctx, lh, index, q(), 2, users, items, sets, n_elements=1)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, lh, index, q(), 2, users, items, (np.array([-1, 1, 2], dtype=np.int64), eo, addr, None))[0] == N.E_INVALID_ARG
    # the template
    for f in ("head", "boosted", "should_tail", "must", "must_not", "sort", "header"):
        rc, msg = raw_call(ctx, lh, index, q(**{f: None}), 2, users, items, sets)
        assert rc == N.E_INVALID_ARG and "null fragment" in msg, f
    assert raw_call(ctx, lh, index, q(set_name=None), 2, users, items, sets)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, lh, index, q(set_name=None, with_set=0), 2, users, items, sets)[0] == N.OK
    assert raw_call(ctx, lh, index, q(with_set=2), 2, users, items, sets)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, lh, index, q(n_names=65), 2, users)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, lh, index, q(n_history_names=2), 2, users)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, lh, index, q(limits=None), 2, users)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, None, index, q(limits=None), 2, None, items)[0] == N.OK   # no user column: no limits needed
    rc, msg = raw_call(ctx, lh, index, q(n_model_names=0), 2, users, items)
    assert rc == N.E_INVALID_ARG and "model event names" in msg
    assert raw_call(ctx, lh, index, q(max_query_events=0), 2, users, items)[0] == N.E_INVALID_ARG
    assert raw_call(ctx, lh, index, q(exclude_self=2), 2, users, items)[0] == N.E_INVALID_ARG
    # the body, with cco_item_queries' messages
    rc, msg = raw_call(ctx, lh, index[:-1], q(), 2, users, items)
    assert rc == N.E_INVALID_ARG and "does not end in a newline" in msg
    dup = b'{"index":{"_id":"a"}}\n{}\n{"index":{"_id":"a"}}\n{}\n'
    rc, msg = raw_call(ctx, lh, dup, q(), 2, users, items)
    assert rc == N.E_INVALID_ARG and "its _id is the _id of document 0" in msg
    bad_doc = b'{"index":{"_id":"Iphone 4"}}\n{"purchase":"x"}\n'
    rc, msg = raw_call(ctx, lh, bad_doc, q(), 2, users, items)
    assert rc == N.E_INVALID_ARG and 'document 0: its "purchase" member is not an array of strings' in msg
    assert raw_call(ctx, lh, bad_doc, q(), 2, users, None, sets)[0] == N.OK   # an unqueried document is not checked
    # group contexts
    group = CcoContext(devices=[0])
    try:
        assert raw_call(group, None, None, q(), 2, None, None, sets)[0] == N.E_UNSUPPORTED
    finally:
        group.close()
    # a later good call is unaffected
    assert raw_call(ctx, lh, index, q(), 2, users, items, sets)[0] == N.OK
