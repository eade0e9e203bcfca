"""Cost of building item-set ("shopping cart") queries on the device (CcoContext.item_set_queries, cco_item_set_queries) for a
seeded batch of sets over a synth.py config's item space: --sets sets (default: the config's user count) of 1 to --max-set
item ids each, drawn with the config's item popularity (so a set may repeat an id), passed as Arrow list<large_string>
buffers.  Prints one JSON line:
  - item_set_queries_ms: the median of --steps calls after --warmup, each bracketed by a device synchronise
  - n_sets, n_elements, body_bytes, body_gb_per_s (body bytes per second of the median call)
  - parity_ok: the device records equal ur_query.item_set_queries (the host mirror) on --sample sets spread over the batch
  - gpu name and power limit, read in the same run
usage: python tools/item_set_queries_bench.py --config C3 --steps 5 --warmup 1 [--sets N] [--max-set 20] [--sample 20000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from events_bench import END_MS, _digits, timed  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from universal_recommender_b200 import ur_query as Q  # noqa: E402

ID_WIDTH = 10   # "i" + 9 digits, the item ids of tools/events_bench.py's exports


def build_sets(n_items: int, n_sets: int, max_set: int, seed: int = 11):
    """-> (set_offsets, elem_offsets, elem_bytes): n_sets sets of 1..max_set ids, fixed-width ids"""
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, max_set + 1, n_sets)
    so = np.zeros(n_sets + 1, dtype=np.int64)
    np.cumsum(sizes, out=so[1:])
    n = int(so[-1])
    icdf, iperm = synth.item_tables(n_items, 0)
    items = iperm[np.minimum(np.searchsorted(icdf, rng.random(n), side="right"), n_items - 1)].astype(np.int64)
    eb = np.empty((n, ID_WIDTH), dtype=np.uint8)
    eb[:, 0] = ord("i")
    eb[:, 1:] = _digits(items, ID_WIDTH - 1)
    return so, np.arange(n + 1, dtype=np.int64) * ID_WIDTH, eb.reshape(-1)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C2")
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sets", type=int, default=None)
    p.add_argument("--max-set", type=int, default=20)
    p.add_argument("--sample", type=int, default=20_000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("item_set_queries_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    n_sets = a.sets if a.sets is not None else cfg["n_users"]
    so, eo, eb = build_sets(cfg["n_items"], n_sets, a.max_set)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "availableDateName": "available", "expireDateName": "expires"})
    query = Q.ItemSetQuery(blacklistItems=["i000000000", "i000000001", "i000000002"])
    ctx = ur.CcoContext(device=0)
    out = {}

    def run():
        out["r"] = ctx.item_set_queries((so, eo, eb), ap, query, END_MS)
    ms = timed(run, a.steps, a.warmup)
    body, off = out["r"]

    # parity: a sample of sets spread over the batch, through the device and the mirror
    step = max(n_sets // max(a.sample, 1), 1)
    idx = list(range(0, n_sets, step))[:a.sample] + ([n_sets - 1] if n_sets else [])
    blob = eb.tobytes()
    sample = [[blob[eo[e]:eo[e + 1]].decode() for e in range(so[s], so[s + 1])] for s in idx]
    dev = ctx.item_set_queries(sample, ap, query, END_MS)
    host = Q.item_set_queries(sample, ap, query, END_MS)
    parity = dev[0] == host[0] and np.array_equal(dev[1], host[1])
    # and the same records inside the whole batch's body
    parity = parity and all(body[off[s]:off[s + 1]] == host[0][host[1][k]:host[1][k + 1]] for k, s in enumerate(idx))
    name, plimit = gpu_info()
    print(json.dumps({
        "config": a.config, "n_sets": n_sets, "n_elements": int(so[-1]), "max_set": a.max_set, "item_set_queries_ms": round(ms, 3),
        "body_bytes": len(body), "body_gb_per_s": round(len(body) / (ms * 1e-3) / 1e9, 2), "bytes_per_record": round(len(body) / max(n_sets, 1), 1),
        "parity_sets": len(idx), "parity_ok": bool(parity), "gpu": name, "power_limit_w": plimit}))
    ctx.close()


if __name__ == "__main__":
    main()
