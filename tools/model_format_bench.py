"""Cost of writing the complete model index (cco_format_model) against the correlators-only body (cco_format_es_bulk).

A resident train of a synth.py config (C3, C4, ...) gives the indicator model; on top of it:
  - 2 property fields per primary item ("category": a JSON array, "available": a JSON boolean),
  - a popular ranking over the primary event stream and a trending ranking over every event type, 30 days of synthetic
    event times, item ids "i<j>" in pinned arrays.
Prints one JSON line:
  - es_bulk_ms_median / model_ms_median: wall time of each call (each ends in a stream synchronise), median of --steps
  - es_bulk_bytes / model_bytes: body sizes; model_h2d_bytes: what cco_format_model copies host -> device beyond es_bulk
  - host_mirror: ur_model.model_documents on a sample (the first --sample events of each stream, all properties), its rate
  - parity_ok: json.loads of every document of format_model on that sample == model_documents
  - gpu name and power limit, read in the same run
  - with --random: model_random_ms_median / model_random_bytes, the same call with a third ranking, uniqueRank (random) over
    every event stream, timed after the call without it; the parity sample then holds the random ranking too
  - with --rerank: cco_rerank_model (calcPop) on the body format_model wrote, with the same properties and rankings,
    alternated step by step with format_model on the same inputs: rerank_ms_median / format_alt_ms_median, the body MB in
    and out, the H2D bytes of the call, and rerank_fixed_point (the rerank of the body equals the body)
usage: python tools/model_format_bench.py --config C3 --steps 5 --warmup 1 --sample 200000 [--random] [--rerank]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from ingest_strings_bench import decimal_ids, events_for_type, gpu_info  # noqa: E402
from universal_recommender_b200 import ur_model as um  # noqa: E402

END_MS = 1_700_000_000_000
WINDOW_MS = 30 * 86_400_000


def docs_of(body: bytes):
    lines = body.decode("utf-8").split("\n")
    return [json.loads(lines[i + 1]) for i in range(0, len(lines) - 1, 2)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=200_000, help="events per stream for the host mirror and the parity check")
    ap.add_argument("--random", action="store_true", help="also time format_model with a random (uniqueRank) ranking added")
    ap.add_argument("--rerank", action="store_true", help="also time rerank_model on the model body, alternated with format_model")
    a = ap.parse_args()
    cfg = synth.CONFIGS[a.config]
    n_types, n_users, n_items = cfg["n_types"], cfg["n_users"], cfg["n_items"]
    per_type = cfg["n_events"] // n_types
    ctx = ur.CcoContext(device=0)

    w = synth.make(a.config, ctx=ctx, keep_dataset=True)
    params = [(500, 50, None)] * n_types
    res, h = ctx.train_dataset(w.dataset, params, seed=42, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR, keep=True)
    names = [f"e{t}" for t in range(n_types)]
    ids = [f"i{j}" for j in range(n_items)]
    cols = [ids] * n_types

    # properties: 2 fields per item
    j = np.repeat(np.arange(n_items), 2)
    triples_items = [ids[int(x)] for x in j]
    values = [f'["c{x % 50}"]' if k % 2 == 0 else ("true" if x % 3 else "false") for k, x in enumerate(j.tolist())]
    fields = ["category", "available"]
    props = (fields, *ur.encode_ids(triples_items), np.tile(np.arange(2, dtype=np.int32), n_items), *ur.encode_ids(values))

    # rankings: the event streams of the config as string ids with synthetic times in the last 30 days
    utab = synth.user_tables(n_users)
    streams = []
    rng = np.random.default_rng(7)
    for t in range(n_types):
        _, items = events_for_type(n_users, n_items, per_type, t, (utab, synth.item_tables(n_items, t)), os.cpu_count() or 1)
        off, data = decimal_ids(ctx, b"i", items)
        tm = ctx.host_array(per_type, np.int64)
        tm[:] = END_MS - rng.integers(1, WINDOW_MS + 1, per_type)
        streams.append((off, data, tm))
        del items
    rankings = [("popRank", "popular", END_MS - WINDOW_MS, END_MS, streams[:1]),
                ("trendRank", "trending", END_MS - WINDOW_MS, END_MS, streams)]
    random_ranking = ("uniqueRank", "random", END_MS - WINDOW_MS, END_MS, streams)
    model_h2d = int(sum(o.nbytes + (o[-1] - o[0]) + tm.nbytes for o, _, tm in streams) + sum(o.nbytes + (o[-1] - o[0]) for o, _, _ in streams[:1])
                    + props[1].nbytes + len(props[2]) + props[3].nbytes + props[4].nbytes + len(props[5]))

    def timed(fn):
        out, ts = None, []
        for step in range(a.warmup + a.steps):
            t0 = time.perf_counter()
            out = fn()
            dt = (time.perf_counter() - t0) * 1e3
            if step >= a.warmup:
                ts.append(dt)
        return out, ts

    es, es_ms = timed(lambda: ctx.format_es_bulk(h, names, ids, cols))
    body, model_ms = timed(lambda: ctx.format_model(h, names, ids, cols, props, rankings))
    extra = {}
    if a.random:
        body_r, random_ms = timed(lambda: ctx.format_model(h, names, ids, cols, props, rankings + [random_ranking]))
        extra = {"model_random_ms_median": round(float(np.median(random_ms)), 2), "model_random_ms_all": [round(x, 2) for x in random_ms],
                 "model_random_bytes": len(body_r)}
        del body_r
    if a.rerank:
        fmt_ms, rr_ms, out = [], [], None
        for step in range(a.warmup + a.steps):
            t0 = time.perf_counter()
            ctx.format_model(h, names, ids, cols, props, rankings)
            t1 = time.perf_counter()
            out = ctx.rerank_model(body, props, rankings)
            t2 = time.perf_counter()
            if step >= a.warmup:
                fmt_ms.append((t1 - t0) * 1e3)
                rr_ms.append((t2 - t1) * 1e3)
        extra.update({"rerank_ms_median": round(float(np.median(rr_ms)), 2), "rerank_ms_all": [round(x, 2) for x in rr_ms],
                      "format_alt_ms_median": round(float(np.median(fmt_ms)), 2), "format_alt_ms_all": [round(x, 2) for x in fmt_ms],
                      "rerank_mb_in": round(len(body) / 1e6, 2), "rerank_mb_out": round(len(out) / 1e6, 2),
                      "rerank_h2d_bytes": int(len(body) + model_h2d),
                      "rerank_fixed_point": out == body})
        del out

    # host mirror and parity on a sample of every stream
    S = min(a.sample, per_type)
    sample_streams = []
    for off, data, tm in streams:
        sample_streams.append((ur.decode_ids(off[:S + 1], bytes(data[:off[S]])), tm[:S].tolist()))
    sample_rankings = [um.Ranking("popRank", "popular", END_MS - WINDOW_MS, END_MS, sample_streams[:1]),
                       um.Ranking("trendRank", "trending", END_MS - WINDOW_MS, END_MS, sample_streams)]
    if a.random:
        sample_rankings.append(um.Ranking("uniqueRank", "random", END_MS - WINDOW_MS, END_MS, sample_streams))
    per_row = [(n, [[ids[c] for c in r[4][r[3][q]:r[3][q + 1]]] for q in range(len(r[3]) - 1)]) for n, r in zip(names, res)]
    triples = [(i, fields[k % 2], json.loads(v)) for k, (i, v) in enumerate(zip(triples_items, values))]
    t0 = time.perf_counter()
    want = um.model_documents(ids, per_row, triples, sample_rankings)
    host_s = time.perf_counter() - t0
    got = ctx.format_model(h, names, ids, cols, props,
                           [(r.field, r.mode, r.start_ms, r.end_ms, [(*ur.encode_ids(s[0]), np.asarray(s[1], np.int64)) for s in r.streams])
                            for r in sample_rankings])
    parity = docs_of(got) == want
    ctx.free_result(h)
    ctx.free_dataset(w.dataset)

    name, plimit = gpu_info()
    print(json.dumps({
        "tool": "model_format_bench", "config": a.config, "gpu": name, "power_limit_w": plimit,
        "items": n_items, "property_triples": 2 * n_items, "ranking_events": per_type * (n_types + 1),
        "es_bulk_ms_median": round(float(np.median(es_ms)), 2), "es_bulk_ms_all": [round(x, 2) for x in es_ms],
        "model_ms_median": round(float(np.median(model_ms)), 2), "model_ms_all": [round(x, 2) for x in model_ms],
        "es_bulk_bytes": len(es), "model_bytes": len(body), "model_documents": body.count(b"\n") // 2, "model_h2d_bytes": model_h2d,
        **extra,
        "host_mirror": {"ranking_events": S * (n_types + 1), "documents": len(want), "s": round(host_s, 3), "threads": 1},
        "parity_ok": bool(parity),
    }), flush=True)
    ctx.close()
    if not parity:
        sys.exit(1)


if __name__ == "__main__":
    main()
