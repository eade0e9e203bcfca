"""Cost of refreshing item properties in place (cco_refresh_properties) against rewriting the whole index.

The model body is the one tools/model_format_bench.py builds: a resident train of a synth.py config, 2 property fields per
item ("category", "available"), a popular and a trending ranking over synthetic event times.  Then, for each fraction of
the items (--fractions), those items get fresh properties: "available" flipped, and "category" unset for every other one.
Per fraction, alternated step by step on the same inputs:
  - refresh_ms: CcoContext.refresh_properties(body, event names, ranking names, fresh properties)
  - rerank_ms:  CcoContext.rerank_model(body, fresh properties, rankings)          (calcPop's rewrite of every document)
  - format_ms:  CcoContext.format_model(model, ..., fresh properties, rankings)    (calcAll's write of every document)
Each call ends in a stream synchronise; medians of --steps after --warmup.  Also: the delta and delete bytes and counts,
fixed_point (a refresh with the properties that made the body returns it with an empty delta) and the GPU's name and
power limit, read in the same run.  One JSON line.
usage: python tools/refresh_properties_bench.py --config C3 --steps 5 --warmup 1 --fractions 0.001,0.01,0.1
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

END_MS = 1_700_000_000_000
WINDOW_MS = 30 * 86_400_000


def properties(ids, values_of):
    """(fields, ...) of CcoContext.format_model from {item index: [(field index, JSON text)]}"""
    items, field, vals = [], [], []
    for j, fv in values_of.items():
        for f, v in fv:
            items.append(ids[j])
            field.append(f)
            vals.append(v)
    return (["category", "available"], *ur.encode_ids(items), np.asarray(field, np.int32), *ur.encode_ids(vals))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--fractions", default="0.001,0.01,0.1")
    a = ap.parse_args()
    cfg = synth.CONFIGS[a.config]
    n_types, n_users, n_items = cfg["n_types"], cfg["n_users"], cfg["n_items"]
    per_type = cfg["n_events"] // n_types
    ctx = ur.CcoContext(device=0)
    w = synth.make(a.config, ctx=ctx, keep_dataset=True)
    _, h = ctx.train_dataset(w.dataset, [(500, 50, None)] * n_types, seed=42, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR, keep=True)
    names = [f"e{t}" for t in range(n_types)]
    ids = [f"i{j}" for j in range(n_items)]
    cols = [ids] * n_types
    base = {j: [(0, f'["c{j % 50}"]'), (1, "true" if j % 3 else "false")] for j in range(n_items)}
    props = properties(ids, base)
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
    rank_names = [r[0] for r in rankings]
    body = ctx.format_model(h, names, ids, cols, props, rankings)
    same = ctx.refresh_properties(body, names, rank_names, properties=props)
    out = {"config": a.config, "n_docs": body.count(b"\n") // 2, "body_mb": round(len(body) / 1e6, 2), "n_triples": int(len(props[3])),
           "fixed_point": same.body == body and same.delta == b"" and same.deletes == b"", "fractions": {}}
    for frac in [float(x) for x in a.fractions.split(",")]:
        picked = rng.choice(n_items, max(1, int(frac * n_items)), replace=False)
        fresh = dict(base)
        for k, j in enumerate(picked.tolist()):
            avail = (1, "false" if j % 3 else "true")
            fresh[j] = [avail] if k % 2 else [base[j][0], avail]
        p2 = properties(ids, fresh)
        ts = {"refresh": [], "rerank": [], "format": []}
        r = None
        for step in range(a.warmup + a.steps):
            t0 = time.perf_counter()
            r = ctx.refresh_properties(body, names, rank_names, properties=p2)
            t1 = time.perf_counter()
            ctx.rerank_model(body, p2, rankings)
            t2 = time.perf_counter()
            ctx.format_model(h, names, ids, cols, p2, rankings)
            t3 = time.perf_counter()
            if step >= a.warmup:
                ts["refresh"].append((t1 - t0) * 1e3)
                ts["rerank"].append((t2 - t1) * 1e3)
                ts["format"].append((t3 - t2) * 1e3)
        out["fractions"][str(frac)] = {
            "items_changed": int(len(picked)), "n_changed": r.n_changed, "n_new": r.n_new, "n_deleted": r.n_deleted,
            "delta_bytes": len(r.delta), "delete_bytes": len(r.deletes),
            **{f"{k}_ms_median": round(float(np.median(v)), 2) for k, v in ts.items()},
            **{f"{k}_ms_all": [round(x, 2) for x in v] for k, v in ts.items()}}
    ctx.free_result(h)
    ctx.free_dataset(w.dataset)
    name, plimit = gpu_info()
    out.update(gpu=name, power_limit=plimit)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
