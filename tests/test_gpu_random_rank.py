"""Random rankings (uniqueRank) in cco_format_model on the H100, byte for byte against the restatement
tests/random_rank_oracle.py: the rank engine's own entry through calc_all_on_device, a million hostile ids, repeatability,
name clashes and row slices."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
import torch

import universal_recommender_b200 as ur
from conftest import ROOT, load_golden
from test_gpu_format_model import _free_port, device_args
from test_model_docs import MODEL_FIXTURES, docs_of, model_inputs
from test_random_rank import with_random
from universal_recommender_b200 import _native as N
from universal_recommender_b200 import ur_model as um

pytestmark = pytest.mark.gpu

RANK_ENGINE = "rank/rank-engine.json"
RANK_VALUE = re.compile(rb',"uniqueRank":([-0-9.E]+)\}')   # an escaped id never holds an unescaped quote


def format_both(ctx, mats, params, names, rows, cols, fields, triples, rankings, seed=1):
    """(device body, restatement body) for JSON-text triples [(item, field name, text)] and rankings
    [(name, mode, start, end, [(items, times)])], random ones included"""
    import random_rank_oracle as ro
    res, h = ctx.train_csr(mats, params, seed, keep=True)
    try:
        props, ranks = device_args(fields, triples, rankings)
        got = ctx.format_model(h, names, rows, cols, props if triples else None, ranks)
    finally:
        ctx.free_result(h)
    want = ro.model_bulk([(r[3], r[4]) for r in res], names, rows, cols, list(fields),
                         [(i, list(fields).index(f), t) for i, f, t in triples], rankings)
    return got, want


def random_fixture_case(name):
    fx = with_random(load_golden(name))
    prepared, triples, fields, rankings = model_inputs(fx, RANK_ENGINE)
    mats = [(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in prepared]
    names = [n for n, _ in prepared]
    rows = prepared[0][1].column_ids.inverse
    cols = [d.column_ids.inverse for _, d in prepared]
    jt = [(i, f, um.property_json(v)) for i, f, v in triples]
    rk = [(r.field, r.mode, r.start_ms, r.end_ms, r.streams) for r in rankings]
    return fx, mats, names, rows, cols, fields, jt, rk


@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_calc_all_on_device_runs_the_rank_engine_with_its_random_entry(ctx, name):
    fx, mats, names, rows, cols, fields, jt, rk = random_fixture_case(name)
    assert [r[1] for r in rk] == ["popular", "random"]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": fx["event_names"], "indicators": fx["indicators"], "seed": 1,
                                                "rankings": fx["rankings"][RANK_ENGINE]})
    events = [tuple(e) for e in fx["events"]]
    sets = [(s[0], s[1]) for s in fx["set_events"]]
    body = ur.calc_all_on_device(events, sets, ap, fx["min_events_per_user"], now_ms=fx["now_ms"], ctx=ctx)
    got, want = format_both(ctx, mats, [(500, 50, None)] * len(mats), names, rows, cols, fields, jt, rk)
    assert body == want == got
    ranked = [d for d in docs_of(body) if "uniqueRank" in d]
    assert len(ranked) >= len({s[0] for s in sets}) and all(0 <= d["uniqueRank"] < 1 for d in ranked)


def _hostile_distinct(rng, n):
    alphabet = ['"', "\\", "\t", "\n", "\x00", "\x01", "\x1f", "é", "☃", "\U0001f600", "a", " "]
    lens = rng.integers(0, 6, n).tolist()
    chars = rng.integers(0, len(alphabet), (n, 5)).tolist()
    out = ["".join(alphabet[c] for c in chars[j][:lens[j]]) + f"h{j}" for j in range(n)]   # the suffix keeps them distinct
    out[0] = ""
    return out


def test_million_distinct_hostile_ids(ctx):
    rng = np.random.default_rng(21)
    n = 1_050_000
    ids = _hostile_distinct(rng, n)
    rows = ids[:5000]
    mats = [(2, 5000, np.array([0, 1, 2], np.int64), np.array([0, 1], np.int32))]
    start, end = 1_600_000_000_000, 1_600_000_000_000 + 30 * 86_400_000
    order = rng.permutation(n)
    items = [ids[int(j)] for j in order] + [ids[int(j)] for j in rng.integers(0, n, 50_000)]
    times = rng.integers(start - 86_400_000, end + 86_400_000, len(items))   # about 6 % outside the window
    times[0], times[1] = start, end                                           # the edges: in, and out unless seen again
    half = len(items) // 2
    streams = [(items[:half], times[:half]), (items[half:], times[half:])]
    fields = ["color"]
    triples = [(ids[int(j)], "color", '"c%d"' % k) for k, j in enumerate(rng.integers(0, n, 3000))]
    got, want = format_both(ctx, mats, [(500, 50, None)], ["buy"], rows, [rows], fields, triples,
                            [("uniqueRank", "random", start, end, streams)])
    assert got == want
    values = RANK_VALUE.findall(got)
    sci = sum(1 for v in values if b"E" in v)
    assert len(values) > 900_000 and 0 < sci < len(values)   # ~1 in 1000 below 10^-3: E notation
    assert all(v.startswith(b"0.") or b"E-" in v for v in values)


def _small_case(rng, n=20_000):
    ids = [f"sku-{j}" for j in range(n)]
    rows = ids[:300]
    mats = [(3, 300, np.array([0, 1, 2, 3], np.int64), np.array([0, 1, 2], np.int32))]
    start, end = 1_600_000_000_000, 1_600_000_000_000 + 7 * 86_400_000
    items = [ids[int(j)] for j in rng.integers(0, n, 60_000)]
    times = rng.integers(start + 1000, end - 1000, len(items))   # inside the window and inside the window moved by 1 ms
    return ids, rows, mats, start, end, [(items, times)]


def test_same_inputs_same_body_and_the_window_moves_the_values(ctx):
    ids, rows, mats, start, end, streams = _small_case(np.random.default_rng(4))
    triples = [(ids[j], "f", "1") for j in (5, 18_000, 19_999)]
    got, want = format_both(ctx, mats, [(500, 50, None)], ["buy"], rows, [rows], ["f"], triples,
                            [("uniqueRank", "random", start, end, streams)])
    assert got == want
    props, ranks = device_args(["f"], triples, [("uniqueRank", "random", start, end, streams)])
    moved = [("uniqueRank", "random", start, end + 1, ranks[0][4])]
    _, h = ctx.train_csr(mats, [(500, 50, None)], 1, keep=True)
    try:
        again = ctx.format_model(h, ["buy"], rows, [rows], props, ranks)
        later = ctx.format_model(h, ["buy"], rows, [rows], props, moved)
    finally:
        ctx.free_result(h)
    other = ur.CcoContext(device=0)
    try:
        _, h2 = other.train_csr(mats, [(500, 50, None)], 1, keep=True)
        elsewhere = other.format_model(h2, ["buy"], rows, [rows], props, ranks)
        other.free_result(h2)
    finally:
        other.close()
    assert again == got == elsewhere
    a, b = docs_of(got), docs_of(later)
    assert [d["id"] for d in a] == [d["id"] for d in b]
    changed = sum(x.get("uniqueRank") != y.get("uniqueRank") for x, y in zip(a, b))
    assert changed > 0.99 * sum("uniqueRank" in x for x in a)


def test_name_clashes_follow_the_precedence(ctx):
    ids, rows, mats, start, end, streams = _small_case(np.random.default_rng(8), 2000)
    fields = ["color", "id"]
    triples = [(ids[j], fields[j % 2], '"p%d"' % j) for j in range(0, 2000, 7)]
    rk = [("uniqueRank", "popular", start, end, streams),       # an earlier ranking of the same name: the random one wins
          ("color", "random", start, end, streams),             # named like a property: the rank wins
          ("buy", "random", start, end, streams),               # named like the indicator: the rank wins
          ("uniqueRank", "random", start, end + 5, streams),
          ("id", "random", start, end, streams)]                # named "id": the document's id wins
    got, want = format_both(ctx, mats, [(500, 50, None)], ["buy"], rows, [rows], fields, triples, rk)
    assert got == want
    docs = docs_of(got)
    assert all(d["id"] == i for d, i in zip(docs, rows))
    ranked = [d for d in docs if "uniqueRank" in d]
    assert ranked and all(0 <= d["uniqueRank"] < 1 and 0 <= d["color"] < 1 and 0 <= d["buy"] < 1 for d in ranked)
    assert not any(isinstance(d.get("color"), str) or isinstance(d.get("buy"), list) for d in ranked)


def test_pop_model_refuses_random(ctx):
    score, present = np.zeros(1), np.zeros(1, np.uint8)
    st = ctx._L.cco_pop_model(ctx._h, 3, 0, None, None, 1, 0, 10, score.ctypes.data_as(C.POINTER(C.c_double)),
                              present.ctypes.data_as(C.POINTER(C.c_ubyte)))
    assert st == N.E_INVALID_ARG   # it works on item indices; a random rank is keyed by id string


# ---- two GPUs: each rank formats its row slice with the same random values; rank 0 adds the items without a row -------
def _slice_worker(rank, world, port, ret):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import universal_recommender_b200 as ur_
        from universal_recommender_b200 import distributed as D
        _, mats, names, rows, cols, fields, jt, rk = random_fixture_case("model_handmade.json")
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
    assert b'"uniqueRank":' in ret[0] + ret[1]
