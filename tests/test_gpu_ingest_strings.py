"""cco_ingest_strings (SURVEY.md 8f-1 on string ids): the dictionaries (content and order), row_ptr and col_idx equal what
preparator.prepare builds on the host; a model trained from the resident dataset equals the host path's, as indicators and
as an Elasticsearch bulk body; truncated hashes (forced collisions) give the same dictionaries; malformed offsets are
rejected and leave the context usable."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

import universal_recommender_b200 as ur
from conftest import ROOT, load_golden, prepared_from_fixture
from universal_recommender_b200 import preparator

pytestmark = pytest.mark.gpu


def assert_same_prepared(got, want):
    assert [n for n, _ in got] == [n for n, _ in want]
    for (_, g), (_, w) in zip(got, want):
        assert list(g.row_ids.inverse) == list(w.row_ids.inverse)
        assert list(g.column_ids.inverse) == list(w.column_ids.inverse)
        assert (g.n_rows, g.n_cols) == (w.n_rows, w.n_cols)
        assert np.array_equal(g.row_ptr, w.row_ptr) and np.array_equal(g.col_idx, w.col_idx)
        assert g.row_ids is got[0][1].row_ids   # one user dictionary object, as prepare shares it


def check(ctx, actions, min_ev):
    want = preparator.prepare(actions, min_ev)
    got = ur.prepare_on_device(actions, min_ev, ctx=ctx)
    assert_same_prepared(got, want)
    return got


def zipf_actions(seed, n_types=3, n_events=150_000, n_users=20_000, n_items=3_000):
    rng = np.random.default_rng(seed)
    out = []
    for t in range(n_types):
        u = (rng.zipf(1.3, n_events) - 1) % n_users
        i = (rng.zipf(1.2, n_events) - 1) % n_items
        items = [f"i{x}" if x % 7 else f"é{x}·項目" for x in i.tolist()]   # some multi-byte UTF-8 ids
        out.append((f"ev{t}", list(zip([f"u{x}" for x in u.tolist()], items))))
    return out


@pytest.mark.parametrize("min_ev", [None, 0, 3])
def test_random_zipf_events_match_the_host_preparator(ctx, min_ev):
    got = check(ctx, zipf_actions(11), min_ev)
    if min_ev == 3:
        assert 0 < got[0][1].n_rows < 20_000


EDGE_IDS = ["", "é", "日本語", "\"quoted\"", "back\\slash", "\x00\x01ctl\x1f\x7f", "x" * 1500, "y" * 1029 + "é",
            "u1", "u10", "u100", "u1\x00", "same"]


def test_edge_ids(ctx):
    rng = np.random.default_rng(3)
    ids = EDGE_IDS
    actions = []
    for t in range(3):
        u = rng.integers(0, len(ids), 4000)
        i = rng.integers(0, len(ids), 4000)
        actions.append((f"e{t}", [(ids[a], ids[b]) for a, b in zip(u.tolist(), i.tolist())]))
    actions[1][1].append(("same", "same"))   # one string as both a user and an item id
    for min_ev in (None, 2, 300):
        check(ctx, actions, min_ev)


def test_edge_streams(ctx):
    # secondary events of unknown users are dropped
    check(ctx, [("buy", [("a", "x"), ("b", "y")]), ("view", [("c", "x"), ("a", "z"), ("d", "w"), ("b", "x")])], None)
    # the first event of item X belongs to a dropped user: X comes after Y in the item dictionary
    got = check(ctx, [("buy", [("a", "X"), ("b", "Y"), ("b", "X"), ("c", "Z"), ("c", "Z")]), ("view", [("a", "V"), ("c", "W")])], 2)
    assert list(got[0][1].column_ids.inverse) == ["Y", "X", "Z"]
    # a type with zero events, at either position
    check(ctx, [("buy", [("a", "x"), ("b", "y")]), ("view", [])], None)
    check(ctx, [("buy", []), ("view", [("a", "x")])], None)
    # every user filtered out
    got = check(ctx, [("buy", [("a", "x"), ("b", "y"), ("a", "y")]), ("view", [("a", "x")])], 5)
    assert got[0][1].n_rows == 0
    # a stream that is all duplicates
    got = check(ctx, [("buy", [("u", "i")] * 1000), ("view", [("u", "j")] * 500)], None)
    assert got[0][1].nnz == 1 and got[1][1].nnz == 1


@pytest.mark.parametrize("hash_bits", [0, 1, 4])
def test_forced_hash_collisions_give_the_same_ids(ctx, hash_bits):
    rng = np.random.default_rng(hash_bits)
    pool = EDGE_IDS + [f"k{j}" for j in range(300)]
    col = [pool[j] for j in rng.integers(0, len(pool), 3000).tolist()]
    off, data = ur.encode_ids(col)
    first = {}
    want = np.array([first.setdefault(x, len(first)) for x in col], dtype=np.int32)
    assert np.array_equal(ctx.debug_string_ids(off, data, 64), want)
    assert np.array_equal(ctx.debug_string_ids(off, data, hash_bits), want)


def test_malformed_offsets_are_rejected_and_the_context_still_trains(ctx):
    off, data = ur.encode_ids(["a", "bb", "ccc", "d"])
    good = (off, data, off.copy(), data)
    dec = off.copy()
    dec[2] = dec[1] - 1                     # decreasing
    neg = off.copy() - 5                    # below 0
    inv = off.copy()
    inv[0] = inv[-1] + 1                    # offsets[0] > offsets[n]
    mid = off.copy()
    mid[1], mid[2] = -3, 2                  # a negative offset inside, first and last fine
    for bad in (dec, neg, inv, mid):
        for cols in ((bad, data, off, data), (off, data, bad, data)):
            with pytest.raises(ur.CcoInvalidArgument):
                ctx.ingest_strings([good, cols])
            with pytest.raises(ur.CcoInvalidArgument):
                ctx.ingest_strings([cols])
        with pytest.raises(ur.CcoInvalidArgument):
            ctx.debug_string_ids(bad, data)
    ds, users, items = ctx.ingest_strings([good, good])
    assert users == ["a", "bb", "ccc", "d"] and items == [users, users]
    res = ctx.train_dataset(ds, [(500, 10, None)] * 2, seed=1)
    assert len(res) == 2
    ctx.free_dataset(ds)


def _fixture_actions(fx):
    actions = [(n, [(u, i) for (u, e, i) in fx["events"] if e == n]) for n in fx["event_names"]]
    return [(n, p) for n, p in actions if p]


@pytest.mark.parametrize("name", ["handmade.json", "item_sets.json", "movielens_sample.json"])
def test_golden_fixtures_train_and_format_like_the_host_path(ctx, name):
    fx = load_golden(name)
    want = prepared_from_fixture(fx)
    actions = _fixture_actions(fx)
    got = ur.prepare_on_device(actions, fx.get("min_events_per_user"), ctx=ctx)
    assert_same_prepared(got, want)
    params = fx["params"]
    mk = lambda prep: [ur.DownsamplableCrossOccurrenceDataset(d, *p) for (_, d), p in zip(prep, params)]
    for g, w in zip(ur.SimilarityAnalysis.crossOccurrenceDownsampled(mk(got), 1, ctx=ctx),
                    ur.SimilarityAnalysis.crossOccurrenceDownsampled(mk(want), 1, ctx=ctx)):
        assert np.array_equal(g.row_ptr, w.row_ptr) and np.array_equal(g.col_idx, w.col_idx)
        assert np.array_equal(g.values, w.values) and list(g.column_ids.inverse) == list(w.column_ids.inverse)
    # strings -> resident dataset -> model -> bulk body, against the host path's body
    names = [n for n, _ in want]
    mats = [(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in want]
    _, h = ctx.train_csr(mats, params, 1, keep=True)
    try:
        host_body = ctx.format_es_bulk(h, names, want[0][1].column_ids.inverse, [d.column_ids.inverse for _, d in want])
    finally:
        ctx.free_result(h)
    cols = [(*ur.encode_ids([u for u, _ in p]), *ur.encode_ids([i for _, i in p])) for _, p in actions]
    ds, users, items = ctx.ingest_strings(cols, fx.get("min_events_per_user"))
    try:
        _, h = ctx.train_dataset(ds, params, 1, keep=True)
        try:
            body = ctx.format_es_bulk(h, names, items[0], items)
        finally:
            ctx.free_result(h)
    finally:
        ctx.free_dataset(ds)
    assert body == host_body


def _tokenise_like_the_dictionaries(actions):
    """integer events whose cco_ingest dictionaries (ascending raw id) coincide with the string dictionaries (first
    appearance): users numbered by first primary appearance, items by first appearance among the surviving events"""
    u0 = [u for u, _ in actions[0][1]]
    users = {}
    for u in u0:
        users.setdefault(u, len(users))
    n_primary = len(users)
    events = []
    for _, pairs in actions:
        items = {}
        for u, i in pairs:
            if u in users and users[u] < n_primary:
                items.setdefault(i, len(items))
        for u, i in pairs:
            users.setdefault(u, len(users))
            items.setdefault(i, len(items))
        ui = np.array([users[u] for u, _ in pairs], dtype=np.int64)
        ii = np.array([items[i] for _, i in pairs], dtype=np.int32)
        events.append((ui, ii, len(items)))
    return events, len(users)


def test_string_ingest_trains_like_integer_ingest(ctx):
    actions = zipf_actions(5, n_types=2, n_events=60_000, n_users=6_000, n_items=900)
    cols = [(*ur.encode_ids([u for u, _ in p]), *ur.encode_ids([i for _, i in p])) for _, p in actions]
    ds_s, users, items = ctx.ingest_strings(cols, 0)
    events, n_users_raw = _tokenise_like_the_dictionaries(actions)
    ds_i, _, _ = ctx.ingest(events, n_users_raw, 0)
    params = [(500, 20, None)] * 2
    try:
        for t in range(2):
            a, b = ctx.dataset_matrix(ds_s, t), ctx.dataset_matrix(ds_i, t)
            assert a[:2] == b[:2] and np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
        got_s = ctx.train_dataset(ds_s, params, seed=4, flags=ur.FLAG_ASSUME_CANONICAL)
        got_i = ctx.train_dataset(ds_i, params, seed=4, flags=ur.FLAG_ASSUME_CANONICAL)
    finally:
        ctx.free_dataset(ds_s)
        ctx.free_dataset(ds_i)
    host = preparator.prepare(actions, 0)
    for t, (s, i) in enumerate(zip(got_s, got_i)):
        assert all(np.array_equal(x, y) for x, y in zip(s[3:], i[3:]))
        # as strings: each primary item's ordered correlators through the string dictionaries == the host dictionaries'
        rp, ci = s[3], s[4]
        as_str = {items[0][r]: [items[t][c] for c in ci[rp[r]:rp[r + 1]]] for r in range(len(rp) - 1)}
        host_cols, host_rows = host[t][1].column_ids.inverse, host[0][1].column_ids.inverse
        assert as_str == {host_rows[r]: [host_cols[c] for c in ci[rp[r]:rp[r + 1]]] for r in range(len(rp) - 1)}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import universal_recommender_b200 as ur_
        from universal_recommender_b200 import distributed as D
        ctx = D.context_from_env(dist)
        actions = zipf_actions(8, n_types=2, n_events=40_000, n_users=5_000, n_items=700)
        cols = [(*ur_.encode_ids([u for u, _ in p]), *ur_.encode_ids([i for _, i in p])) for _, p in actions]
        ds, _, _ = ctx.ingest_strings(cols, 0)
        params = [(500, 20, None)] * 2
        merged = D.gather_indicators(dist, ctx.train_dataset(ds, params, seed=42))
        ctx.free_dataset(ds)
        host = preparator.prepare(actions, 0)
        single = ur_.CcoContext(device=rank).train_csr([(d.n_rows, d.n_cols, d.row_ptr, d.col_idx) for _, d in host], params, seed=42)
        ok = True
        for (n_rows, n_cols, rp, ci, ll, cn), r in zip(merged, single):
            ok &= np.array_equal(rp, r[3]) and np.array_equal(ci, r[4]) and np.array_equal(cn, r[6])
        ctx.close()
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_string_ingest_trains_the_same_model():
    import torch.multiprocessing as mp
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    assert dict(ret) == {0: True, 1: True}
