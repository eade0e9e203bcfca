"""cco_format_model on the H100: the complete model index byte for byte against the restatement tests/model_oracle.py."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

import universal_recommender_b200 as ur
from conftest import ROOT, load_golden
from test_model_docs import CONFIGS, MODEL_FIXTURES, docs_of, model_inputs
from universal_recommender_b200 import ur_model as um

pytestmark = pytest.mark.gpu


def device_args(fields, triples, rankings):
    """mirror values -> format_model's properties / rankings arguments"""
    fidx = {f: k for k, f in enumerate(fields)}
    props = (list(fields), *ur.encode_ids([i for i, _, _ in triples]), [fidx[f] for _, f, _ in triples],
             *ur.encode_ids([t for _, _, t in triples]))
    ranks = [(r[0], r[1], r[2], r[3], [(*ur.encode_ids(items), np.asarray(times, np.int64)) for items, times in r[4]]) for r in rankings]
    return props, ranks


def format_both(ctx, mats, params, names, rows, cols, fields, triples, rankings, seed=1):
    """(device body, restatement body) for JSON-text triples [(item, field name, text)] and rankings
    [(name, mode, start, end, [(items, times)])]"""
    import model_oracle as mo
    res, h = ctx.train_csr(mats, params, seed, keep=True)
    try:
        props, ranks = device_args(fields, triples, rankings)
        got = ctx.format_model(h, names, rows, cols, props if triples else None, ranks)
    finally:
        ctx.free_result(h)
    want = mo.model_bulk([(r[3], r[4]) for r in res], names, rows, cols, list(fields),
                         [(i, list(fields).index(f), t) for i, f, t in triples], rankings)
    return got, want


def fixture_case(name, config):
    fx = load_golden(name)
    prepared, triples, fields, rankings = model_inputs(fx, config)
    mats = [(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
    names = [n for n, _ in prepared]
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    jt = [(i, f, um.property_json(v)) for i, f, v in triples]
    rk = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings]
    return fx, mats, names, rows, cols, fields, jt, rk


@pytest.mark.parametrize("config", CONFIGS)
@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_format_model_on_the_reference_data(ctx, name, config):
    fx, mats, names, rows, cols, fields, jt, rk = fixture_case(name, config)
    got, want = format_both(ctx, mats, [(500, 50, None)] * len(mats), names, rows, cols, fields, jt, rk)
    assert got == want
    assert len(docs_of(got)) >= len(rows)


@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_calc_all_on_device_is_the_whole_train_half(ctx, name):
    fx, mats, names, rows, cols, fields, jt, rk = fixture_case(name, "rank/rank-engine.json")
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": fx["event_names"], "indicators": fx["indicators"], "seed": 1,
                                                "rankings": fx["rankings"]["rank/rank-engine.json"]})
    events = [tuple(e) for e in fx["events"]]
    sets = [(s[0], s[1]) for s in fx["set_events"]]
    body = ur.calc_all_on_device(events, sets, ap, fx["min_events_per_user"], now_ms=fx["now_ms"], ctx=ctx)
    got, want = format_both(ctx, mats, [(500, 50, None)] * len(mats), names, rows, cols, fields, jt, rk)
    assert body == want == got
    ap.recsModel = "collabFiltering"
    res, h = ctx.train_csr(mats, [(500, 50, None)] * len(mats), 1, keep=True)
    try:
        es = ctx.format_es_bulk(h, names, rows, cols)
    finally:
        ctx.free_result(h)
    assert ur.calc_all_on_device(events, sets, ap, fx["min_events_per_user"], now_ms=fx["now_ms"], ctx=ctx) == es
    ap.recsModel = "backfill"
    with pytest.raises(ValueError):
        ur.calc_all_on_device(events, sets, ap, fx["min_events_per_user"], now_ms=fx["now_ms"], ctx=ctx)


def test_no_properties_no_rankings_is_the_es_bulk_body(ctx):
    import synth
    cases = [fixture_case(n, CONFIGS[0])[1:5] for n in MODEL_FIXTURES]
    w = synth.make("small")
    ids = [f"item-{j}" for j in range(w.n_items)]
    cases.append((w.mats, [f"ev{t}" for t in range(w.n_types)], ids, [ids] * w.n_types))
    for mats, names, rows, cols in cases:
        params = w.params if mats is w.mats else [(500, 50, None)] * len(mats)
        _, h = ctx.train_csr(mats, params, 3, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR, keep=True)
        try:
            es = ctx.format_es_bulk(h, names, rows, cols)
            assert ctx.format_model(h, names, rows, cols) == es
            assert ctx.format_model(h, names, rows, cols, (["f"], [0], [], [], [0], []), []) == es
        finally:
            ctx.free_result(h)


def _hostile(rng, n, salt):
    alphabet = ['"', "\\", "\t", "\n", "\x00", "\x01", "é", "☃", "\U0001f600", "a", " "]
    out = ["".join(alphabet[int(x)] for x in rng.integers(0, len(alphabet), int(rng.integers(0, 6)))) + f"{salt}{i}" for i in range(n)]
    out[0] = ""
    return out


def test_hostile_ids_on_property_and_ranking_items(ctx):
    rng = np.random.default_rng(5)
    rows = _hostile(rng, 40, "r")
    mats = [(3, 40, np.array([0, 1, 2, 3], np.int64), np.array([0, 1, 2], np.int32))]
    others = _hostile(rng, 30, "o")
    pool = rows[:20] + others
    fields = ['c"at', "id", "popRank", "n\\x"]
    triples = [(pool[int(rng.integers(0, len(pool)))], fields[int(rng.integers(0, 4))], t)
               for t in ['["a","b"]', "3", '"\\u0000x"', "true", "1.5E-4", "{\"k\":[1]}"] * 8]
    items = [pool[int(x)] for x in rng.integers(0, len(pool), 400)] + ["only-out-of-window"]
    times = list(rng.integers(0, 90, 400)) + [95]
    rankings = [("popRank", "popular", 0, 90, [(items[:200], times[:200]), (items[200:], times[200:])]),
                ("trendRank", "trending", 0, 90, [(items, times)]), ("c\"at", "hot", 0, 90, [(items, times)]),
                ("popRank", "hot", 30, 60, [(items, times)])]
    got, want = format_both(ctx, mats, [(500, 50, None)], ["buy"], rows, [rows], fields, triples, rankings)
    assert got == want
    assert b"only-out-of-window" not in got and len(docs_of(got)) > 40


@pytest.mark.parametrize("mode", ["popular", "trending", "hot"])
def test_million_event_ranking_stream(ctx, mode):
    rng = np.random.default_rng(9)
    n_items, n_ev = 20_000, 1_100_000
    ids = [f"sku-{j}" for j in range(n_items)]
    rows = ids[:5000]
    mats = [(2, 5000, np.array([0, 1, 2], np.int64), np.array([0, 1], np.int32))]
    pick = (rng.zipf(1.3, n_ev) - 1) % n_items
    items = [ids[int(j)] for j in pick]
    start, end = 1_600_000_000_000, 1_600_000_000_000 + 9 * 86_400_000 + 2
    times = rng.integers(start - 86_400_000, end + 86_400_000, n_ev)
    got, want = format_both(ctx, mats, [(500, 50, None)], ["buy"], rows, [rows], [], [],
                            [("rank", mode, start, end, [(items, times)])])
    assert got == want


def test_empty_bucket_rules_give_no_rank(ctx):
    mats = [(1, 2, np.array([0, 1], np.int64), np.array([0], np.int32))]
    rows = ["a", "b"]
    rk = [("t", "trending", 0, 90, [(["a", "c"], [50, 60])]), ("h", "hot", 0, 90, [(["a", "a", "d"], [5, 70, 80])])]
    got, want = format_both(ctx, mats, [(500, 50, None)], ["buy"], rows, [rows], [], [], rk)
    assert got == want and b'"t"' not in got and b'"h"' not in got and len(docs_of(got)) == 2


def test_malformed_inputs_are_rejected_and_the_context_keeps_working(ctx):
    mats = [(1, 2, np.array([0, 1], np.int64), np.array([0], np.int32))]
    rows = ["a", "b"]
    _, h = ctx.train_csr(mats, [(500, 50, None)], 1, keep=True)
    off, b = ur.encode_ids(["a", "x"])
    vo, vb = ur.encode_ids(["1", "2"])
    bad_off = np.array([0, 2, 1], np.int64)
    try:
        for props, ranks in [((["f"], bad_off, b, [0, 0], vo, vb), None),                        # item offsets decrease
                             ((["f"], off, b, [0, 0], bad_off, vb), None),                       # value offsets decrease
                             ((["f"], off, b, [0, 1], vo, vb), None),                            # field index out of range
                             ((["f"], off, b, [0, -1], vo, vb), None),
                             ((["f"], off, b, [0, 0], np.array([0, 1, 1], np.int64), vb), None),  # empty value
                             ((["f", "f"], off, b, [0, 1], vo, vb), None),                       # repeated field name
                             ((["f"], np.array([-1, 0, 1], np.int64), b, [0, 0], vo, vb), None),  # negative offset
                             (None, [("r", "popular", 10, 5, [(off, b, [1, 2])])]),               # end before start
                             (None, [("r", "weekly", 0, 5, [(off, b, [1, 2])])]),                 # bad mode
                             (None, [("r", "popular", 0, 5, [(bad_off, b, [1, 2])])])]:
            with pytest.raises(ur.CcoInvalidArgument):
                ctx.format_model(h, ["buy"], rows, [rows], props, ranks)
        with pytest.raises(ur.CcoError) as e:
            ctx.format_model(h, ["buy"], rows, [rows], None, [("r", "popular", 0, 5, [(off, b, [1, 2])])] * 9)
        assert e.value.status == -6
        ok = ctx.format_model(h, ["buy"], rows, [rows], (["f"], off, b, [0, 0], vo, vb), [("r", "popular", 0, 5, [(off, b, [1, 2])])])
        assert docs_of(ok) == [{"id": "a", "buy": [], "f": 1, "r": 1.0}, {"id": "b", "buy": []}, {"id": "x", "f": 2, "r": 1.0}]
    finally:
        ctx.free_result(h)
    assert len(ctx.train_csr(mats, [(500, 50, None)], 1)) == 1


# ---- two GPUs: each rank formats its row slice; rank 0 adds the items without a row --------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _slice_worker(rank, world, port, ret):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import universal_recommender_b200 as ur_
        from universal_recommender_b200 import distributed as D
        _, mats, names, rows, cols, fields, jt, rk = fixture_case("model_handmade.json", "rank/rank-engine.json")
        props, ranks = device_args(fields, jt, rk)
        ctx = D.context_from_env(dist)
        _, h = ctx.train_csr(mats, [(500, 50, None)] * len(mats), 1, keep=True)
        ret[rank] = ctx.format_model(h, names, rows, cols, props, ranks)
        ctx.free_result(h)
        if rank == 0:
            single = ur_.CcoContext(device=0)
            _, h = single.train_csr(mats, [(500, 50, None)] * len(mats), 1, keep=True)
            ret["single"] = single.format_model(h, names, rows, cols, props, ranks)
            single.free_result(h)
            single.close()
        ctx.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_slices_together_are_the_single_gpu_body():
    import torch.multiprocessing as mp
    ret = mp.Manager().dict()
    mp.spawn(_slice_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    pairs = lambda body: sorted(zip(body.split(b"\n")[0:-1:2], body.split(b"\n")[1::2]))
    assert pairs(ret[0] + ret[1]) == pairs(ret["single"])
