"""cco_event_log_user_queries against the host mirror (ur_query.user_queries over events.read_export): byte-identical
bodies on the handmade data for every golden template, seeded random exports with hostile ids, streamed and windowed reads;
the error cases; a log read without history retention is unchanged and refuses the call."""
import numpy as np
import pytest

from universal_recommender_b200 import CcoContext, EventWindow
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import events as E
from universal_recommender_b200 import ur_algorithm as ur
from universal_recommender_b200 import ur_query as Q
from user_query_data import golden, handmade_export, handmade_params, random_export

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000_000


@pytest.fixture(scope="module")
def ctx():
    c = CcoContext()
    yield c
    c.close()


def check(ctx, data, ap, q, users, chunk=None, window=None, now=NOW):
    ev = E.read_export(data, window, now)
    with ctx.read_events(data, chunk_bytes=chunk, window=window, now_ms=now, keep_history=True) as log:
        dev = ctx.user_queries(log, ap, q, users, now)
    host = Q.user_queries(ev, ap, q, users, now)
    assert dev[0] == host[0]
    assert np.array_equal(dev[1], host[1])
    if users is None:
        assert dev[2] == host[2]
    return dev


def test_handmade_every_template(ctx):
    g = golden()
    data = handmade_export()
    for tpl in g["queries"]:
        q = Q.UserQuery.from_json(tpl)
        check(ctx, data, handmade_params(), q, g["users"] + ["u1"])
        check(ctx, data, handmade_params(), q, None)
    body, off = check(ctx, data, handmade_params(), None, ["u1"])
    assert body == b"{}\n" + g["u1_default"].encode() + b"\n"


@pytest.mark.parametrize("over", [dict(userBias=-1), dict(blacklistEvents=[]), dict(blacklistEvents=["view", "category-pref"]),
                                  dict(recsModel="collabFiltering"), dict(indicators=None, eventNames=["purchase", "view"], maxQueryEvents=2)])
def test_handmade_params(ctx, over):
    check(ctx, handmade_export(), handmade_params(**over), Q.UserQuery(blacklistItems=["Galaxy", "x", "x"]), golden()["users"])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_exports(ctx, seed):
    data = random_export(seed)
    ap = ur.URAlgorithmParams.from_engine_json({"indicators": [{"name": "buy", "maxItemsPerUser": 5}, {"name": "view", "maxItemsPerUser": 3},
                                                               {"name": "like"}], "blacklistEvents": ["like", "other", "buy"]})
    ev = E.read_export(data)
    some = list(dict.fromkeys(u for u, *_ in ev.events))[:20]
    users = some + ["absent", some[0], "\"", ""] + some[:3]
    items = list(dict.fromkeys(i for _, _, i, _ in ev.events))[:10]
    q = Q.UserQuery(userBias=1.5, blacklistItems=items[::2] + ["nope", items[0]])
    check(ctx, data, ap, q, users)
    check(ctx, data, ap, q, None)
    check(ctx, data, ap, q, users, chunk=4096)
    check(ctx, data, ap, Q.UserQuery(eventNames=["view", "view", "buy"]), None, chunk=1 << 20)


def test_windowed_reads(ctx):
    data = random_export(7) + random_export(7)   # every event twice: removeDuplicates collapses them
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": ["buy", "view", "like"]})
    w = EventWindow("20 seconds", True)
    now = 1_600_000_000_000 + 40_000
    check(ctx, data, ap, None, None, window=w, now=now)
    check(ctx, data, ap, None, None, chunk=8192, window=w, now=now)


def test_log_without_history_is_unchanged_and_refused(ctx):
    data = handmade_export()
    with ctx.read_events(data) as a, ctx.read_events(data, keep_history=True) as b:
        assert a.info() == b.info()
        ia, ib = [ctx.ingest_event_log(x, ["purchase", "view"], 0) for x in (a, b)]
        try:
            assert ia[1] == ib[1] and ia[2] == ib[2]
            for t in range(2):
                assert all(np.array_equal(x, y) for x, y in zip(ctx.dataset_matrix(ia[0], t), ctx.dataset_matrix(ib[0], t)))
        finally:
            ctx.free_dataset(ia[0])
            ctx.free_dataset(ib[0])
        with pytest.raises(N.CcoInvalidArgument, match="history"):
            ctx.user_queries(a, handmade_params(), None, ["u1"], NOW)


def test_errors_before_any_kernel(ctx):
    import ctypes as C
    L = N.lib()
    with ctx.read_events(handmade_export(), keep_history=True) as log:
        nm = (C.c_char_p * 1)(b"purchase")
        lim = (C.c_int32 * 1)(5)
        bad = np.array([0, 4, 2], dtype=np.int64)   # decreasing offsets
        ok = np.array([0, 1], dtype=np.int64)
        frag = [b'{"from":0,"size":1', b"{}", b"", b"", b"[]", b"{}"]
        def q(**kw):
            d = dict(n_names=1, n_history_names=1, names=nm, limits=lim, n_blacklist_names=0, history_in_must=0, blacklist_names=None,
                     boost=None, head=frag[0], should=frag[1], must=frag[2], must_not=frag[3], sort=frag[4], header=frag[5],
                     n_blacklist_items=0, blacklist_item_offsets=ok.ctypes.data_as(C.POINTER(C.c_int64)), blacklist_item_bytes=None)
            d.update(kw)
            return N.UserQueryT(**d)
        out, ln, off, n = C.c_void_p(), C.c_int64(), C.c_void_p(), C.c_int64()
        call = lambda qt, nu=0, uo=None, ub=None: L.cco_event_log_user_queries(ctx._h, log._h, C.byref(qt), nu, uo, ub, C.byref(out), C.byref(ln),
                                                                               C.byref(off), C.byref(n), None)
        blob = C.create_string_buffer(b"abcd")
        assert call(q(n_blacklist_items=2, blacklist_item_offsets=bad.ctypes.data_as(C.POINTER(C.c_int64)), blacklist_item_bytes=C.cast(blob, C.c_void_p))) == N.E_INVALID_ARG
        assert call(q(), 2, bad.ctypes.data_as(C.POINTER(C.c_int64)), C.cast(blob, C.c_void_p)) == N.E_INVALID_ARG
        assert call(q(n_history_names=2)) == N.E_INVALID_ARG
        assert call(q(should=b"")) == N.E_INVALID_ARG
        assert call(q(limits=(C.c_int32 * 1)(-1))) == N.E_INVALID_ARG
        assert call(q(names=(C.c_char_p * 1)(b""))) == N.E_INVALID_ARG
        assert call(q(), 1, ok.ctypes.data_as(C.POINTER(C.c_int64)), C.cast(blob, C.c_void_p)) == N.OK
        L.cco_host_free(ctx._h, out)
        L.cco_host_free(ctx._h, off)


def test_from_events_entry(ctx):
    body, off, users = ur.user_queries_from_events(handmade_export(), handmade_params(), None, None, NOW, ctx=ctx)
    host = Q.user_queries(E.read_export(handmade_export()), handmade_params(), None, None, NOW)
    assert body == host[0] and users == host[2]
