"""cco_index_pages on the H100 against the ur_model.index_from_pages mirror, byte for byte: every CPU case, the compaction's
lane and word edges (whitespace and backslash runs, escaped quotes and brackets inside strings, at every offset of a warp
step and a 64-byte word, sources of 0 .. 65 bytes inside), a page of 10^5 hits, every error code and message with the
errors a later call reports, and calcPop and the item queries fed from pages of a seeded export's index."""
import random

import pytest

import index_pages_data as D
import test_index_pages as C
import universal_recommender_b200 as ur
from test_gpu_event_stream import AP, NOW
from test_gpu_events import random_export
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_model as um

pytestmark = pytest.mark.gpu


def device(ctx, pages):
    """-> (body, n_docs, total, [(n_hits, scroll_id)] per page)"""
    with ctx.index_pages() as r:
        per = [r.append(p) for p in pages]
        body = r.finish()
        return body, r.n_docs, r.total, per


def expect_mirror(ctx, pages):
    body, n, total, per = device(ctx, pages)
    assert (body, n, total) == um.index_from_pages(pages)
    assert per == [um.index_page(p, k)[1:3] for k, p in enumerate(pages)]
    return body


CPU_PAGES = [
    b'{"_scroll_id":"DnF1ZXJ5\\u0041","took":2,"timed_out":false,"_shards":{"total":1,"successful":1,"skipped":0,"failed":0},'
    b'"hits":{"total":2,"max_score":1.0,"hits":[{"_index":"urindex","_type":"items","_id":"a","_score":1.0,'
    b'"_source":{"id":"a","purchase":["b","c"]}},{"_index":"urindex","_type":"items","_id":"b","_score":1.0,"_source":{"id":"b"}}]}}',
    b'{"took":1}', b'{"hits":{"hits":null}}',
    b'{"hits":{"hits":[{"sort":[3,"x]"],"_score":null,"_source":{"id":"i"},"fields":{"a":[{"b":"}"}]},'
    b'"_routing":"r","_id":"i","_index":"u"}]},"took":1}',
    b'{"hits":{"hits":[{"_id":"x","_source":{"id":"x","n":1.0E7,"n":-0,"m":12345678901234567890,"s":"\\u00e9\\u0041\\/\\ud83d\\ude00","e":[],"o":{}}}]}}',
    b'{\n  "hits" : {\n    "hits" : [ {\n      "_id" : "a b",\n      "_source" : {\n        "id" : "a b",\n'
    b'        "t" : " x\\t y \\" { ",\n        "l" : [ 1 , 2 ]\r\n      }\n    } ]\n  }\n}\n',
    '{"hits":{"hits":[{"_id":"q\\"\\\\\\/\\u0001\\u00e9\\ud83d\\ude00\\ud800","_source":{}}]}}'.encode(),
    b'{"hits":{"hits":[{"_id":"a","_source":{"k":1},"_source":{"k":2}}]},"hits":{"hits":[{"_id":"b","_source":{}}]},'
    b'"_scroll_id":"one","_scroll_id":"two","timed_out":false,"timed_out":true}',
] + [('{"hits":{"total":%s,"hits":[]}}' % t).encode() for t in
     ('{"value":3,"relation":"eq"}', '{"value":10000,"relation":"gte"}', '{"relation":"eq","value":7}', '{"value":3}', "null", "1.5")]


@pytest.mark.parametrize("k", range(len(CPU_PAGES)))
def test_hand_written_pages(ctx, k):
    expect_mirror(ctx, [CPU_PAGES[k]])
    expect_mirror(ctx, [CPU_PAGES[k], CPU_PAGES[0], b'{"hits":{"hits":[]}}'])


def test_empty_index(ctx):
    assert device(ctx, []) == (b"", 0, -1, [])
    assert expect_mirror(ctx, [b'{"hits":{"total":0,"hits":[]}}']) == b""


@pytest.mark.parametrize("page_hits,pretty,es7", C.LAYOUTS)
def test_round_trip_of_the_handmade_model(ctx, orc, page_hits, pretty, es7):
    for k, (_, body) in enumerate(D.handmade_bodies(orc)):
        assert expect_mirror(ctx, D.pages_of(body, page_hits, seed=k, pretty=pretty, es7=es7)) == body


@pytest.mark.parametrize("page_hits,pretty,es7", C.LAYOUTS)
def test_round_trip_of_edge_ids(ctx, page_hits, pretty, es7):
    body = D.edge_body(random.Random(5))
    assert expect_mirror(ctx, D.pages_of(body, page_hits, seed=page_hits, pretty=pretty, es7=es7)) == body


# ---- lane and word edges -------------------------------------------------------------------------------------------------
INSIDE = [0, 1, 31, 32, 33, 64, 65]


def edge_source(rng, inside: int) -> bytes:
    """a _source whose compact form holds `inside` bytes between its braces, with whitespace outside strings"""
    if inside < 6:
        return b"{" + b" " * rng.randrange(40) + b"7" * inside + b"\n" * rng.randrange(3) + b"}"
    s = b'"k' + b"\\\\" * rng.randrange(0, 3)
    s = s[:inside - 4]
    pad = inside - len(s) - 4
    return b"{ " + s + b'"' + b" " * rng.randrange(33) + b":" + b"\t" * rng.randrange(33) + b'"' + b"v" * pad + b'" }'


def run_source(rng) -> bytes:
    """whitespace runs outside strings and backslash runs, escaped quotes and brackets inside them, of random lengths"""
    parts = []
    for k in range(rng.randrange(1, 8)):
        ws = bytes(rng.choice(b" \t\n\r") for _ in range(rng.randrange(0, 70)))
        inner = rng.choice([b"\\\\" * rng.randrange(0, 40), b'\\"' * rng.randrange(0, 20), b"{[\\\"]}" * rng.randrange(0, 12),
                            b" " * rng.randrange(0, 70), b"\\u00e9\\/" * rng.randrange(0, 9)])
        parts.append(ws + b'"m' + str(k).encode() + b'"' + ws + b":" + ws + b'"' + inner + b'"' + ws)
    return b"{" + b",".join(parts) + b"}"


@pytest.mark.parametrize("seed", range(6))
def test_lane_and_word_edges(ctx, seed):
    rng = random.Random(seed)
    hits = []
    for k in range(400):
        src = edge_source(rng, INSIDE[k % len(INSIDE)]) if k % 2 else run_source(rng)
        pad = "p" * rng.randrange(130)   # moves the _source across every offset of a word and a warp step
        hits.append('{"_index":"%s","_id":"d%d","_source":%s}' % (pad, k, src.decode()))
    pages = [("{\"hits\":{\"hits\":[" + ",".join(hits[a:a + 97]) + "]}}").encode() for a in range(0, len(hits), 97)]
    body = expect_mirror(ctx, pages)
    inside = {len(s) - 2 for _, s in D.docs_of(body)}
    assert set(INSIDE) <= inside


def test_one_page_of_1e5_hits(ctx):
    rng = random.Random(3)
    hits = ['{"_id":"i%d","_score":null,"_source":{"id":"i%d","v":[%s]}}' % (k, k, ",".join('"x"' for _ in range(rng.randrange(4))))
            for k in range(100_000)]
    page = ('{"_scroll_id":"s","hits":{"total":{"value":100000,"relation":"eq"},"hits":[' + ",".join(hits) + "]}}").encode()
    body, n, total, per = device(ctx, [page, b'{"hits":{"hits":[]}}'])
    assert (n, total, per) == (100_000, 100_000, [(100_000, "s"), (0, None)])
    assert body == um.index_from_pages([page])[0]


# ---- errors -------------------------------------------------------------------------------------------------------------
GOOD = b'{"hits":{"hits":[{"_id":"z","_source":{}}]}}'
ERRORS = [p for p in (m.args[1] for m in C.test_errors.pytestmark if m.name == "parametrize")][0]


@pytest.mark.parametrize("page,msg", ERRORS)
def test_each_error(ctx, page, msg):
    with ctx.index_pages() as r:
        r.append(GOOD)
        if ", hit " in msg:   # a document error: the page's hits are counted, the next call reports it
            r.append(page)
            with pytest.raises(N.CcoInvalidArgument) as e:
                r.append(GOOD)
        else:
            with pytest.raises(N.CcoInvalidArgument) as e:
                r.append(page)
        assert msg in str(e.value)
        with pytest.raises(N.CcoInvalidArgument) as again:   # every later call fails with the same message
            r.finish()
        assert str(again.value) == str(e.value)
        with pytest.raises(N.CcoInvalidArgument):
            r.append(GOOD)


def test_document_error_of_the_last_page_comes_from_finish(ctx):
    with ctx.index_pages() as r:
        assert r.append(C.hits_page('{"_id":"a"}')) == (1, None)
        with pytest.raises(N.CcoInvalidArgument, match="page 0, hit 0: the hit has no _source"):
            r.finish()


def test_scroll_ended_early(ctx):
    p = b'{"hits":{"total":3,"hits":[{"_id":"a","_source":{}}]}}'
    with pytest.raises(ValueError, match="scroll ended early"):
        ur.index_from_pages([p], ctx=ctx)


# ---- end to end --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pretty", [False, True])
def test_calc_pop_and_item_queries_from_pages(ctx, pretty, tmp_path):
    data = random_export(11)
    body = ur.calc_all_from_events(data, AP, 0, now_ms=NOW, ctx=ctx)
    pages = D.pages_of(body, 7, seed=2, pretty=pretty)
    paths = []
    for k, p in enumerate(pages):
        paths.append(str(tmp_path / f"page-{k:03d}.json"))
        open(paths[-1], "wb").write(p)
    got = ur.index_from_pages(paths, ctx=ctx)
    assert got == D.compact(body) and got != body   # the export spells some property values with spaces
    assert ur.index_from_pages(iter(pages), ctx=ctx) == got
    assert ur.index_from_pages(D.pages_of(got, 5, seed=3, pretty=pretty), ctx=ctx) == got   # a compact index comes back as it is
    pop = ur.calc_pop_from_events(got, data, AP, now_ms=NOW, ctx=ctx)
    assert D.compact(pop) == D.compact(ur.calc_pop_from_events(body, data, AP, now_ms=NOW, ctx=ctx))
    want_q = ur.item_queries(body, AP, now_ms=NOW, ctx=ctx)
    got_q = ur.item_queries(got, AP, now_ms=NOW, ctx=ctx)
    assert got_q[0] == want_q[0] and list(got_q[1]) == list(want_q[1])
