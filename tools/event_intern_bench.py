"""Cost of a retrain cycle from a resident, extendable event log with interned ids (read_events(intern_ids=True)) against
the same log without them, stage by stage.

The export is event_extend_bench.py's (export_days): eventTimes uniform over the 31 days before END_MS, days 0-29 are A,
day 30 is B.  Each round, for an interned and a plain extendable log in turn (alternated, one warm-up round first):
  read     read_events of A with a 30-day window at now = END_MS - 1 day, to a finished log (the interned read's extra
           cost is the first-read overhead of interning);
  extend   EventLog.extend(B) at now = END_MS;
  ingest   ingest_event_log of the model's event names (the key path on the interned log, the string path on the other);
  train    train_dataset of that dataset;
  format   format_model with the log's properties and rankings (format_model_log);
  cycle    extend + ingest + train + format.
The two logs' bodies must be equal in every round.  Prints one JSON line: per mode the median of each stage, the
resident bytes and, for the interned log, intern_stats (user and item keys); the plain log's calc_all_from_events time
(the call a retrain made before interning existed); the GPU's name and power limit, read in the same run.
usage: python tools/event_intern_bench.py --config C2 --steps 5
       python tools/event_intern_bench.py --config C3 --steps 3
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
from universal_recommender_b200 import ur_algorithm as ua  # noqa: E402
from event_extend_bench import DAY, export_days  # noqa: E402
from events_bench import END_MS  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402

STAGES = ("read", "extend", "ingest", "train", "format", "cycle")


def cycle(ctx, torch, A, B, window, chunk, intern, ap, names, mepu):
    """one timed read + extend + retrain -> (ms per stage, body, log)"""
    ms = {}

    def timed(stage, f):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = f()
        torch.cuda.synchronize()
        ms[stage] = (time.perf_counter() - t0) * 1e3
        return r

    log = timed("read", lambda: ctx.read_events(A, chunk_bytes=chunk, window=window, now_ms=END_MS - DAY, extendable=True,
                                                 intern_ids=intern))
    timed("extend", lambda: log.extend(B, window=window, now_ms=END_MS))
    seed, flags = ua._seed_and_flags(ap, 0)
    ds, _, items = timed("ingest", lambda: ctx.ingest_event_log(log, names, mepu))
    try:
        _, h = timed("train", lambda: ctx.train_dataset(ds, ua._indicator_params(ap, names), seed, flags, keep=True))
        try:
            body = timed("format", lambda: ctx.format_model(h, names, items[0], items, rankings=ua._log_rankings(ap, END_MS), log=log))
        finally:
            ctx.free_result(h)
    finally:
        ctx.free_dataset(ds)
    ms["cycle"] = ms["extend"] + ms["ingest"] + ms["train"] + ms["format"]
    return ms, body, log


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, default=256 << 20)
    ap_.add_argument("--steps", type=int, default=3)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_intern_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": names, "duration": 30 * DAY // 1000}]})
    mepu = cfg.get("min_events_per_user", 0)
    whole, n_a, n_lines = export_days(cfg, a.fraction, ctx.host_array)
    A, B = whole[:n_a], whole[n_a:]
    window = ur.EventWindow("30 days", True)
    out = {"config": a.config, "fraction": a.fraction, "export_bytes": len(whole), "n_lines": n_lines, "new_bytes": len(B),
           "chunk_bytes": a.chunk_bytes, "remove_duplicates": True}
    t = {m: {s: [] for s in STAGES} for m in ("interned", "plain")}
    calc_all = []
    for step in range(a.steps + 1):   # alternated; the first round warms up
        bodies = {}
        for mode in ("interned", "plain"):
            ms, bodies[mode], log = cycle(ctx, torch, A, B, window, a.chunk_bytes, mode == "interned", ap, names, mepu)
            if step == 0:
                out[f"resident_bytes_{mode}"] = log.resident_bytes()
                if mode == "interned":
                    out["intern_stats"] = list(log.intern_stats())
            if mode == "plain":
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                body = ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx)
                tc = (time.perf_counter() - t0) * 1e3
                assert body == bodies["plain"], "calc_all_from_events differs from its stages"
                if step:
                    calc_all.append(tc)
            log.free()
            if step:
                for s in STAGES:
                    t[mode][s].append(ms[s])
        assert bodies["interned"] == bodies["plain"], "the interned log trains differently"
    out["bodies_equal"] = True
    for mode, st in t.items():
        for s, v in st.items():
            out[f"{mode}_{s}_ms"] = round(statistics.median(v), 2)
    out["plain_calc_all_ms"] = round(statistics.median(calc_all), 2)
    ctx.host_free(whole)
    name, plimit = gpu_info()
    out.update(gpu=name, power_limit_w=plimit)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
