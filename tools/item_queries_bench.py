"""Cost of building every item's query on the device (CcoContext.item_queries, cco_item_queries) over the model index that
calc_all_from_events writes for the export of tools/events_bench.py (a synth.py config as fixed-width JSON lines).  Prints one
JSON line:
  - calc_all_ms: one calc_all_from_events of the export (the index the queries read; informational, one run)
  - item_queries_ms: the median of --steps calls for every document after --warmup, each bracketed by a device synchronise
  - n_documents, index_bytes, n_records, body_bytes
  - parity_ok: the device records equal ur_query.item_queries (the host mirror): every document when the index has at most
    --sample documents, else a sample of --sample documents spread over the index plus unknown ids
  - gpu name and power limit, read in the same run
usage: python tools/item_queries_bench.py --config C2 --steps 5 --warmup 1 [--fraction 1.0] [--sample 20000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from events_bench import END_MS, build_export, timed  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from universal_recommender_b200 import ur_query as Q  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C2")
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--fraction", type=float, default=1.0)
    p.add_argument("--sample", type=int, default=20_000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("item_queries_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    buf, n_lines = build_export(ctx, cfg, a.fraction)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "availableDateName": "available", "expireDateName": "expires"})
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    index = ur.calc_all_from_events(buf, ap, now_ms=END_MS, ctx=ctx, flags=0)
    torch.cuda.synchronize()
    calc_ms = (time.perf_counter() - t0) * 1e3
    ctx.host_free(buf)
    out = {}

    def run():
        out["r"] = ctx.item_queries(index, ap, None, None, END_MS)
    iq_ms = timed(run, a.steps, a.warmup)
    body, off, items = out["r"]

    # parity: every document, or a spread sample of them and unknown ids
    if len(items) <= a.sample:
        dev = ctx.item_queries(index, ap, None, None, END_MS)
        host = Q.item_queries(index, ap, None, None, END_MS)
        parity, n_parity = dev[0] == host[0] and dev[2] == host[2], len(items)
    else:
        step = max(len(items) // a.sample, 1)
        who = items[::step][:a.sample] + ["unknown-1", "", items[0], "i000000000x"]
        dev = ctx.item_queries(index, ap, None, who, END_MS)
        host = Q.item_queries(index, ap, None, who, END_MS)
        parity, n_parity = dev[0] == host[0] and (dev[1] == host[1]).all(), len(who)
    name, plimit = gpu_info()
    print(json.dumps({
        "config": a.config, "fraction": a.fraction, "n_lines": n_lines, "calc_all_ms": round(calc_ms, 1),
        "n_documents": len(items), "index_bytes": len(index), "item_queries_ms": round(iq_ms, 3), "n_records": len(off) - 1,
        "body_bytes": len(body), "bytes_per_record": round(len(body) / max(len(off) - 1, 1), 1), "parity_records": n_parity,
        "parity_ok": bool(parity), "gpu": name, "power_limit_w": plimit}))
    ctx.close()


if __name__ == "__main__":
    main()
