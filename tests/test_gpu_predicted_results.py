"""cco_search_results on the H100 against the ur_predict mirror, byte for byte on the text and on every column: the
reference's served PredictedResult lines, the structural index's edges (backslash runs across words and chunks, brackets
and quotes inside strings, pretty printing), hit counts around a warp, many records and hits, rankings and per-record
withRanks, streams split at uneven points, and every documented error."""
import math
import random

import numpy as np
import pytest

import search_results_data as D
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_predict as P

pytestmark = pytest.mark.gpu
NAMES = ["popRank", "trendRank", "hotRank", "uniqueRank", "défaut\"Rank"]


def expect_equal(res, preds):
    """device results == mirror predictions on every column and the text"""
    assert len(res) == len(preds)
    assert res.records() == [p.text() for p in preds]
    K = len(res.ranking_names)
    off = [0]
    ids, scores, ranks = [], [], []
    for p in preds:
        off.append(off[-1] + len(p.items))
        ids += [i for i, _ in p.items]
        scores += p.scores
        ranks += [[r.get(n, math.nan) for n in res.ranking_names] for r in p.ranks]
    assert res.hit_offsets.tolist() == off
    assert res.status.tolist() == [p.status for p in preds]
    assert res.total.tolist() == [p.total for p in preds]
    assert res.ids == ids
    assert np.array_equal(res.scores.view(np.uint64), np.array(scores, np.float64).view(np.uint64))
    want = np.array(ranks, np.float64).reshape(len(ids), K)
    assert np.array_equal(np.isnan(res.ranks), np.isnan(want))
    assert np.array_equal(np.nan_to_num(res.ranks).view(np.uint64), np.nan_to_num(want).view(np.uint64))


def test_golden_lines_byte_for_byte(ctx):
    g = D.golden_elements()
    res = ctx.search_results(D.body([e for _, e in g]), [], counts=[len(g)])
    assert res.records() == [x["text"] for x, _ in g]
    assert res.n_exact > 0   # the 16- and 17-digit rank-test scores


@pytest.mark.parametrize("pretty", [False, True])
@pytest.mark.parametrize("k", [0, 1, 3, 5])
def test_random_bodies_equal_the_mirror(ctx, pretty, k):
    names = NAMES[:k]
    els = D.random_elements(100 + k, 400, names)
    rng = random.Random(k)
    flags = [rng.random() < 0.5 for _ in els]
    b = D.body(els, pretty)
    expect_equal(ctx.search_results(b, names, with_ranks=flags), P.predictions(b, names, flags))
    expect_equal(ctx.search_results(b, names, with_ranks=True), P.predictions(b, names, True))


def test_pretty_and_compact_agree(ctx):
    els = D.random_elements(7, 300, NAMES[:2])
    a = ctx.search_results(D.body(els), NAMES[:2], with_ranks=True)
    b = ctx.search_results(D.body(els, True), NAMES[:2], with_ranks=True)
    assert a.records() == b.records() and a.ids == b.ids and a.total.tolist() == b.total.tolist()


def test_hit_counts_around_a_warp(ctx):
    rng = random.Random(3)
    counts = [0, 1, 31, 32, 33, 64, 65, 10 ** 4]
    els = [D.random_element(rng, ["popRank"], n_hits=n, errors=False) for n in counts]
    b = D.body(els)
    preds = P.predictions(b, ["popRank"], True)
    res = ctx.search_results(b, ["popRank"], with_ranks=True)
    expect_equal(res, preds)
    assert set(np.diff(res.hit_offsets).tolist()) == set(counts), "a hit count did not occur"


def test_empty_responses_array(ctx):
    res = ctx.search_results(b'{"responses":[]}', [], counts=[0])
    assert len(res) == 0 and res.records() == [] and res.hit_offsets.tolist() == [0]


def test_backslash_runs_at_every_offset(ctx):
    """ids ending in runs of 0..70 backslashes, shifted so the run ends at every offset mod 64 and across chunks"""
    els = []
    for run in range(71):
        for shift in range(0, 64, 7):
            iid = "p" * shift + "\\" * run
            els.append('{"hits":{"hits":[{"_id":' + '"' + iid.replace("\\", "\\\\") + '"' + ',"_score":1.5,"_source":{"s":"' + "\\\\" * (run % 5) + '\\""}}]}}')
    b = D.body(els)
    expect_equal(ctx.search_results(b, []), P.predictions(b, [], False))
    pad = b'{"pad":"' + b"\\\\" * 1100 + b'","responses":[' + b",".join(e.encode() for e in els) + b"]}"
    expect_equal(ctx.search_results(pad, []), P.predictions(pad, [], False))


def test_many_records_and_hits(ctx):
    names = NAMES[:2]
    els = D.random_elements(11, 40000, names)
    b = D.body(els)
    expect_equal(ctx.search_results(b, names, with_ranks=True), P.predictions(b, names, True))


def test_stream_split_points_do_not_matter(ctx):
    names = NAMES[:3]
    els = D.random_elements(21, 3000, names)
    rng = random.Random(5)
    cuts = sorted(rng.sample(range(1, len(els)), 40))
    parts = [els[a:b] for a, b in zip([0] + cuts, cuts + [len(els)])]
    flags = [rng.random() < 0.5 for _ in els]
    bodies = (D.body(p, pretty_print=i % 3 == 0) for i, p in enumerate(parts))
    res = ctx.search_results(bodies, names, with_ranks=flags, counts=[len(p) for p in parts])
    expect_equal(res, P.predictions(D.body(els), names, flags))


ERRORS = [
    (b'{"responses":[{"hits":{"hits":[]}}', N.E_INVALID_ARG, "byte"),
    (b'{"responses":[{"hits":{"hits":[]}]]}', N.E_INVALID_ARG, "byte"),
    (b'{"responses":[{"hits":{"hits":"x"}}]}', N.E_INVALID_ARG, "record 0: hits.hits is not an array"),
    (b'{"responses":[{}, 5]}', N.E_INVALID_ARG, "not an object"),
    (b'{"took":1}', N.E_INVALID_ARG, "responses"),
    (b'[1]', N.E_INVALID_ARG, "responses"),
    (b'{"responses":[{"hits":{"hits":[{"_score":1}]}}]}', N.E_INVALID_ARG, "record 0 hit 0: the hit has no string _id"),
    (b'{"responses":[{"hits":{"hits":[{"_id":1,"_score":1}]}}]}', N.E_INVALID_ARG, "no string _id"),
    (b'{"responses":[{"hits":{"hits":[{"_id":"a","_id":"b","_score":1}]}}]}', N.E_INVALID_ARG, "repeated"),
    (b'{"responses":[{},{"hits":{"hits":[{"_id":"a"},{"_id":"b","_score":null}]}}]}', N.E_INVALID_ARG, "record 1 hit 0: _score"),
    (b'{"responses":[{"hits":{"hits":[{"_id":"a","_score":"1"}]}}]}', N.E_INVALID_ARG, "_score"),
    (b'{"responses":[{"hits":{"hits":[{"_id":"a","_score":1,"_source":{"popRank":"x"}}]}}]}', N.E_INVALID_ARG, "rank"),
    (b'{"responses":[{"hits":{"hits":[{"_id":"a","_score":1e999}]}}]}', N.E_INVALID_ARG, "range"),
    (b'{"responses":[{"hits":{"hits":[{"_id":"a\\x","_score":1}]}}]}', N.E_INVALID_ARG, "escape"),
    (b'{"responses":[{"status":"ok"}]}', N.E_INVALID_ARG, "status"),
    (b'{"responses":[{"hits":{"hits":[{"_id":"a","_score":01}]}}]}', N.E_INVALID_ARG, ""),
    (b'{"responses":[{"hits":{"hits":[]}}]} x', N.E_INVALID_ARG, "byte"),
]


@pytest.mark.parametrize("body,code,text", ERRORS)
def test_errors(ctx, body, code, text):
    with pytest.raises(N.CcoError) as e:
        ctx.search_results(body, ["popRank"], with_ranks=True)
    assert e.value.status == code and text in str(e.value), str(e.value)
    with pytest.raises(ValueError):
        P.predictions(body, ["popRank"], True)


def test_count_mismatch(ctx):
    with pytest.raises(N.CcoInvalidArgument, match="2 response elements for 3 records"):
        ctx.search_results(b'{"responses":[{},{}]}', [], counts=[3])


def test_repeated_names_are_one(ctx):
    b = D.body(D.random_elements(9, 50, ["popRank"]))
    a = ctx.search_results(b, ["popRank", "popRank"], with_ranks=True)
    assert a.ranks.shape[1] == 1
    expect_equal(a, P.predictions(b, ["popRank"], True))


def test_served_lines_through_the_public_api(ctx):
    """the golden elements streamed in bodies of 7 through ur.predictions_from_responses: the served lines, one per line"""
    import universal_recommender_b200 as ur
    g = D.golden_elements()
    parts = [g[i:i + 7] for i in range(0, len(g), 7)]
    res = ur.predictions_from_responses([D.body([e for _, e in p]) for p in parts], [], counts=[len(p) for p in parts], ctx=ctx)
    assert res.text().decode().splitlines() == [x["text"] for x, _ in g]


def test_unsupported(ctx):
    """a body claiming 2^31 records, and a group context, are CCO_E_UNSUPPORTED"""
    import ctypes as C
    L = N.lib()
    prm = N.SearchResultsParamsT(0, None, N.SR_TEXT)
    h = C.c_void_p()
    N.check(L.cco_search_results_begin(ctx._h, C.byref(prm), C.byref(h)))
    try:
        assert L.cco_search_results_append(h, b'{"responses":[]}', 16, 1 << 31, None, None, None) == N.E_UNSUPPORTED
        assert b"2^31" in L.cco_last_error()
    finally:
        L.cco_search_results_free(h)
    import universal_recommender_b200 as ur
    g = ur.CcoContext(devices=[0])
    try:
        with pytest.raises(N.CcoError) as e:
            g.search_results(b'{"responses":[]}', [])
        assert e.value.status == N.E_UNSUPPORTED
    finally:
        g.close()


@pytest.mark.parametrize("edge", range(len(D.ID_EDGES)))
def test_id_edges_on_hits_0_31_32(ctx, edge):
    """each id edge on hits 0, 31 and 32 of one record, and on records 0, 31 and 32"""
    iid = D.ID_EDGES[edge]
    def hit(i):
        return '{"_id":' + (D.json.dumps(iid) if i in (0, 31, 32) else '"x%d"' % i) + ',"_score":1.25}'
    el = '{"hits":{"hits":[' + ",".join(hit(i) for i in range(40)) + "]}}"
    small = '{"hits":{"hits":[' + hit(0) + "]}}"
    els = [el if r in (0, 31, 32) else small.replace(D.json.dumps(iid), '"y"') for r in range(40)]
    b = D.body(els)
    expect_equal(ctx.search_results(b, []), P.predictions(b, [], False))


LINES = [
    '{"user":"u1"}',
    '  { "user" : "u\\u00e9\\\"1" , "num" : -0 , "from":12345678901234567890, "bias": 1.50, "e": 1E2 , "withRanks" : true }  ',
    '{"item":"\\ud83d\\ude00 \u00e9 \\u0085","withRanks":false,"fields":[{"name":"c","values":["a","b"],"bias":-1.0e-3}]}',
    '{"itemSet":["a","b"],"withRanks":null,"x":[[],{},[1,[2.5e-7,{"y":null}]]],"x":0.10000000000000001}',
    '{"user":"u2","userBias":3.14159265358979323,"itemBias":1e-400,"t":true,"f":false}',
]


def test_batchpredict_lines_equal_the_mirror(ctx):
    rng = random.Random(4)
    names = NAMES[:2]
    lines = [rng.choice(LINES) for _ in range(300)]
    els = D.random_elements(31, 300, names)
    parts = [(0, 120), (120, 121), (121, 300)]
    bodies = [D.body(els[a:b], pretty_print=a == 120) for a, b in parts]
    qf = ("\n".join(lines) + "\n").encode()
    res = ctx.search_results(bodies, names, counts=[b - a for a, b in parts], query_lines=qf)
    want = P.batchpredict_lines(qf, bodies, names)
    assert res.records() == want
    assert res.text().decode().splitlines() == want
    flags = [P.line_with_ranks(x) for x in lines]
    res = ctx.search_results(bodies, names, counts=[b - a for a, b in parts], query_lines=qf)
    expect_equal_columns = P.predictions(D.body(els), names, flags)
    assert res.ids == [i for p in expect_equal_columns for i, _ in p.items]
    assert np.array_equal(np.isnan(res.ranks), np.isnan(np.array([[r.get(n, math.nan) for n in names] for p in expect_equal_columns
                                                                   for r in p.ranks]).reshape(-1, len(names))))


@pytest.mark.parametrize("line,text", [
    ('{"withRanks":"yes"}', "withRanks is not true"),
    ('{"withRanks":true,"withRanks":false}', "repeats withRanks"),
    ('{"user":"u1"', "not one JSON object"),
    ('["user"]', "not one JSON object"),
    ('', "not one JSON object"),
    ('{"user":"u1"} {}', "not one JSON object"),
    ('{"a":01}', "not one JSON object"),
    ('{"a":"\\x"}', "not one JSON object"),
    ('{"a":1e400}', "out of the range"),
])
def test_batchpredict_line_errors(ctx, line, text):
    b = D.body(['{"hits":{"hits":[]}}', '{"hits":{"hits":[]}}'])
    qf = ('{"user":"ok"}\n' + line + "\n").encode()
    with pytest.raises(N.CcoInvalidArgument) as e:
        ctx.search_results(b, [], query_lines=qf)
    assert "record 1" in str(e.value) and text in str(e.value), str(e.value)
    with pytest.raises(ValueError):
        P.batchpredict_lines(qf, [b], [])


def test_batchpredict_output_end_to_end(ctx, tmp_path):
    """queries_from_file's body for the handmade query file -> responses synthesised from the handmade index, one per
    record, streamed in bodies of 5 -> ur.batchpredict_output, equal to the mirror"""
    import universal_recommender_b200 as ur
    from conftest import load_golden
    from user_query_data import handmade_export, handmade_params
    fx = load_golden("query_file_handmade.json")
    index = load_golden("item_queries_handmade.json")["index"].encode()
    ap = handmade_params()
    qbody, off = ur.queries_from_file(fx["file"].encode(), handmade_export(), index, ap, now_ms=fx["now_ms"], ctx=ctx)
    n = len(off) - 1
    src = D.index_sources()
    ids = list(src)
    rng = random.Random(8)
    els = []
    for r in range(n):
        picked = rng.sample(ids, rng.randint(0, 4))
        hits = ['{"_index":"urindex","_id":' + D.json.dumps(i) + ',"_score":' + str(round(rng.random() * 3, 7)) + ',"_source":' + src[i] + "}"
                for i in picked]
        els.append('{"took":2,"hits":{"total":{"value":%d,"relation":"eq"},"hits":[%s]},"status":200}' % (len(hits), ",".join(hits)))
    parts = [els[i:i + 5] for i in range(0, n, 5)]
    bodies = [D.body(p) for p in parts]
    names = P.ranking_names(ap)
    out = tmp_path / "predictions.json"
    assert ur.batchpredict_output(fx["file"].encode(), bodies, ap, out=str(out), counts=[len(p) for p in parts], ctx=ctx) is None
    want = P.batchpredict_lines(fx["file"].encode(), bodies, names)
    assert out.read_bytes().decode().splitlines() == want and len(want) == n
