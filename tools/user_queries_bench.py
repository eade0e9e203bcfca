"""Cost of building every user's query on the device (CcoContext.user_queries, cco_event_log_user_queries) over the export
of tools/events_bench.py (a synth.py config as fixed-width JSON lines).  Prints one JSON line:
  - read_ms / read_history_ms: cco_event_log_read without and with history retention, alternated, medians of --steps
  - user_queries_ms: the median of --steps calls for every user after --warmup, each bracketed by a device synchronise
  - n_records, body_bytes
  - parity_ok: the device records of a sample of users equal ur_query.user_queries (the host mirror) on a sample export
  - gpu name and power limit, read in the same run
usage: python tools/user_queries_bench.py --config C2 --steps 5 --warmup 1 [--fraction 0.25] [--sample 100000]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from events_bench import END_MS, EV, build_export, timed  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from universal_recommender_b200 import events as E  # noqa: E402
from universal_recommender_b200 import ur_query as Q  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C2")
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--fraction", type=float, default=1.0)
    p.add_argument("--sample", type=int, default=100_000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("user_queries_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    buf, n_lines = build_export(ctx, cfg, a.fraction)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "availableDateName": "available", "expireDateName": "expires"})

    t_plain, t_hist = [], []
    for k in range(a.steps + a.warmup):   # alternated
        for keep, acc in ((False, t_plain), (True, t_hist)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.read_events(buf, keep_history=keep).free()
            torch.cuda.synchronize()
            if k >= a.warmup:
                acc.append((time.perf_counter() - t0) * 1e3)
    log = ctx.read_events(buf, keep_history=True)
    out = {}

    def run():
        out["r"] = ctx.user_queries(log, ap, None, None, END_MS)
    uq_ms = timed(run, a.steps, a.warmup)
    body, off, users = out["r"]
    log.free()

    # parity on a sample export: the first --sample event lines of each type
    n_ev = n_lines - cfg["n_items"]
    per, L = n_ev // cfg["n_types"], len(EV)
    k = min(a.sample // cfg["n_types"], per)
    mv = memoryview(buf)
    sample = b"".join(bytes(mv[t * per * L:(t * per + k) * L]) for t in range(cfg["n_types"]))
    with ctx.read_events(sample, keep_history=True) as slog:
        dev = ctx.user_queries(slog, ap, None, None, END_MS)
    host = Q.user_queries(E.read_export(sample), ap, None, None, END_MS)
    name, plimit = gpu_info()
    print(json.dumps({
        "config": a.config, "fraction": a.fraction, "export_bytes": len(buf), "n_lines": n_lines,
        "read_ms": round(statistics.median(t_plain), 3), "read_history_ms": round(statistics.median(t_hist), 3),
        "user_queries_ms": round(uq_ms, 3), "n_records": len(users), "body_bytes": len(body),
        "bytes_per_record": round(len(body) / max(len(users), 1), 1), "parity_users": len(host[2]),
        "parity_ok": dev[0] == host[0] and dev[2] == host[2], "gpu": name, "power_limit_w": plimit}))
    ctx.host_free(buf)
    ctx.close()


if __name__ == "__main__":
    main()
