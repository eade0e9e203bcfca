"""cco_rerank_model on the H100 (calcPop, recsModel "backfill"): every body byte for byte against tests/rerank_oracle.py and,
parsed, against the host mirror ur_model.rerank_documents."""
import json

import numpy as np
import pytest

import rerank_oracle as rr
import universal_recommender_b200 as ur
from conftest import load_golden
from test_gpu_format_model import _hostile, device_args
from test_model_docs import CONFIGS, MODEL_FIXTURES, docs_of, model_inputs
from test_rerank_docs import fixture_rankings
from universal_recommender_b200 import ur_model as um

pytestmark = pytest.mark.gpu


def rerank_both(ctx, body, triples, rankings):
    """device body == restatement body, and its documents == the mirror's; mirror triples (item, field, value) and
    um.Rankings"""
    fields = list(dict.fromkeys(f for _, f, _ in triples))
    jt = [(i, f, um.property_json(v)) for i, f, v in triples]
    rk = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings]
    props, ranks = device_args(fields, jt, rk)
    got = ctx.rerank_model(body, props if triples else None, ranks)
    want = rr.rerank_bulk(body, fields, [(i, fields.index(f), t) for i, f, t in jt], rk)
    assert got == want
    assert docs_of(got) == um.rerank_documents(rr.old_documents(body), triples, rankings)
    return got


def device_model(ctx, fx, config):
    prepared, triples, fields, rankings = model_inputs(fx, config)
    mats = [(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
    names = [n for n, _ in prepared]
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    jt = [(i, f, um.property_json(v)) for i, f, v in triples]
    props, ranks = device_args(fields, jt, [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings])
    _, h = ctx.train_csr(mats, [(500, 50, None)] * len(mats), 1, keep=True)
    try:
        body = ctx.format_model(h, names, rows, cols, props, ranks)
    finally:
        ctx.free_result(h)
    return body, triples, rankings


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_fixed_point_and_refresh_on_the_reference_data(ctx, name, config):
    fx = load_golden(name)
    body, triples, rankings = device_model(ctx, fx, config)
    assert rerank_both(ctx, body, triples, rankings) == body
    later = fixture_rankings(fx, config, fx["now_ms"] + 3 * 86_400_000)
    changed = [(i, f, "changed" if k % 3 == 0 else v) for k, (i, f, v) in enumerate(triples)] + [("brand-new", "category", ["x"])]
    again = rerank_both(ctx, body, changed, later)
    assert docs_of(again)[-1]["id"] == "brand-new"


@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_calc_pop_on_device(ctx, name):
    fx = load_golden(name)
    config = "rank/rank-engine.json"
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": fx["event_names"], "indicators": fx["indicators"], "seed": 1,
                                                "rankings": fx["rankings"][config]})
    events = [tuple(e) for e in fx["events"]]
    sets = [(s[0], s[1]) for s in fx["set_events"]]
    body = ur.calc_all_on_device(events, sets, ap, fx["min_events_per_user"], now_ms=fx["now_ms"], ctx=ctx)
    assert ur.calc_pop_on_device(body, events, sets, ap, now_ms=fx["now_ms"], ctx=ctx) == body
    later = fx["now_ms"] + 86_400_000
    sets2 = sets[::2] + [(sets[0][0], {"extra": "yes"})]
    got = ur.calc_pop_on_device(body, events, sets2, ap, now_ms=later, ctx=ctx)
    triples = [(i, f, um.extract_jvalue(f, v)) for i, f, v in um.aggregate_properties(sets2)]
    assert got == rerank_both(ctx, body, triples, fixture_rankings(fx, config, later))
    ap.recsModel = "backfill"
    with pytest.raises(ValueError):
        ur.calc_all_on_device(events, sets, ap, fx["min_events_per_user"], now_ms=fx["now_ms"], ctx=ctx)


def test_hostile_ids_on_a_synth_model(ctx):
    import synth
    rng = np.random.default_rng(11)
    w = synth.make("small")
    ids = _hostile(rng, w.n_items, "i")
    _, h = ctx.train_csr(w.mats, w.params, 3, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR, keep=True)
    try:
        body = ctx.format_es_bulk(h, [f"ev{t}" for t in range(w.n_types)], ids, [ids] * w.n_types)
    finally:
        ctx.free_result(h)
    others = _hostile(rng, 50, "o")
    pool = ids[:200] + others
    items = [pool[int(x)] for x in rng.integers(0, len(pool), 3000)]
    times = [int(t) for t in rng.integers(0, 100, 3000)]
    triples = [(pool[int(rng.integers(0, len(pool)))], f, v) for f, v in [("ev0", 1), ('q"uote', "x\\y"), ("id", 2)] * 40]
    rankings = [um.Ranking("popRank", "popular", 0, 100, [(items, times)]), um.Ranking("trendRank", "trending", 0, 100, [(items, times)]),
                um.Ranking("uniqueRank", "random", 0, 100, [(items[:100], times[:100])])]
    got = rerank_both(ctx, body, triples, rankings)
    assert len(docs_of(got)) > w.n_items


FOREIGN = [
    # whitespace and \r\n
    b' { "index" : { "_index" : "m" , "_id" : "a" } } \r\n\t{ "x" : [ 1 , 2 ] ,\r "y" : { "z" : null } }\r\n',
    # _ids written with escapes: \u00e9, a surrogate pair, \/
    b'{"index":{"_id":"caf\\u00e9"}}\n{"n":1}\n{"index":{"_id":"\\ud83d\\ude00"}}\n{"n":2}\n{"index":{"_id":"a\\/b"}}\n{"n":3}\n',
    # a member that clashes with the popRank ranking, written with an escape
    b'{"index":{"_id":"p"}}\n{"pop\\u0052ank":99.0,"keep":true}\n{"index":{"_id":"q"}}\n{"popRank":5.0}\n',
    # } ] and \" inside string values
    b'{"index":{"_id":"s"}}\n{"t":"}]\\"{[","u":["]","}"],"v":"\\\\"}\n',
    # {} sources
    b'{"index":{"_id":"e1"}}\n{}\n{"index":{"_id":"e2"}}\n{ }\n',
]


def test_foreign_valid_bodies(ctx):
    rankings = [um.Ranking("popRank", "popular", 0, 100, [(["p", "a", "caf\u00e9", "\U0001f600", "a/b", "s", "new"], [1, 2, 3, 4, 5, 6, 7])])]
    triples = [("a", "x", "fresh x"), ("e1", "color", "red"), ("p", "keep", False), ("new2", "color", "blue")]
    for body in FOREIGN:
        rerank_both(ctx, body, triples, rankings)
    # long documents: members past 4 KB and a 1 MB value
    big = b'{"index":{"_id":"big"}}\n{' + b",".join(b'"k%d":"%s"' % (k, b"v" * (k % 97)) for k in range(200)) + b'}\n'
    huge = b'{"index":{"_id":"huge"}}\n{"a":1,"blob":"' + b"\\\"x" * 350_000 + b'","b":[' + b"1," * 1000 + b'2]}\n'
    got = rerank_both(ctx, big + huge, triples, rankings)
    assert len(got) > 1_050_000
    # an empty body: the new items' documents alone
    empty = rerank_both(ctx, b"", triples, rankings)
    assert [d["id"] for d in docs_of(empty)] == ["a", "e1", "p", "new2", "caf\u00e9", "\U0001f600", "a/b", "s", "new"]


def test_malformed_bodies_are_rejected_and_the_context_keeps_working(ctx):
    ok = b'{"index":{"_id":"a"}}\n{"x":1}\n'
    bad = [
        b'{"index":{"_id":"a"}}\n',                              # odd number of lines
        b'{"index":{"_id":"a"}}\n{"x":1}',                       # no final newline
        ok + b'{"index":{"_id":"b"}}\n{"x":[1}\n',               # unbalanced brackets
        ok + b'{"index":{"_id":"b"}}\n{"x":{"y":1}\n',
        ok + b'{"index":{"_id":"b"}}\n{"x":1}}\n',
        ok + b'{"index":{"_id":"b"}}\n{"x":"abc}\n',             # unterminated string
        ok + b'{"index":{"_id":"b"}}\n{"x":"a\\qb"}\n',          # bad escapes
        ok + b'{"index":{"_id":"b"}}\n{"x":"\\u12g4"}\n',
        ok + b'{"index":{"_id":"b"}}\n{"x":"a\tb"}\n',           # a raw control byte in a string
        ok + b'{"create":{"_id":"b"}}\n{"x":1}\n',               # action not index
        ok + b'{"index":{"_id":"b"},"delete":{}}\n{"x":1}\n',
        ok + b'{"index":{"_index":"m"}}\n{"x":1}\n',             # no _id
        ok + b'{"index":{"_id":7}}\n{"x":1}\n',                  # _id not a string
        ok + b'{"index":"b"}\n{"x":1}\n',
        ok + b'{"index":{"_id":"b"}}\n["x",1]\n',                # source not an object
        ok + b'{"index":{"_id":"b"}}\n"x"\n',
        ok + b'{"index":{"_id":"b"}}\n\n',
        ok + b'{"index":{"_id":"b"}}\n{"x":}\n',                 # an empty value
        ok + b'{"index":{"_id":"b"}}\n{"x":1,}\n',
        ok + b'{"index":{"_id":"a"}}\n{"x":2}\n',                # an _id in two documents
        ok + b'{"index":{"_id":"\\u0061"}}\n{"x":2}\n',
    ]
    ranks = [("popRank", "popular", 0, 10, [(*ur.encode_ids(["a"]), np.array([1], np.int64))])]
    for body in bad:
        with pytest.raises(ur.CcoInvalidArgument) as e:
            ctx.rerank_model(body, None, ranks)
        with pytest.raises(ValueError):
            rr.parse_body(body)
        if body.startswith(ok) and body != ok:
            assert "document 1" in str(e.value), (body, str(e.value))
    assert ctx.rerank_model(ok, None, ranks) == b'{"index":{"_id":"a"}}\n{"id":"a","x":1,"popRank":1.0}\n'
    assert json.loads(ctx.rerank_model(ok, None, ranks).split(b"\n")[1]) == {"id": "a", "x": 1, "popRank": 1.0}
