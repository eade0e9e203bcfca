"""Cost of the DataSource's eventWindow on the device (CcoContext.read_events(window=...)): the same export read, and
calc_all_from_events run, with and without the window, alternated.

The export is event_stream_bench.py's (events_bench.py's line templates; times uniform over the 30 days before END_MS),
streamed from pinned memory in chunks of --chunk-bytes.  The window's duration is --days: about 1 - days / 30 of the
training lines expire; the synthetic generator repeats (user, item) pairs of a type at other times, and those collapse
under removeDuplicates.  Prints one JSON line:
  - export_bytes, n_lines, chunk_bytes, n_expired and n_duplicates (EventLog.window_stats)
  - plain_read_ms / window_read_ms and plain_calc_all_ms / window_calc_all_ms: medians over --steps alternated rounds
    (one warm-up round first); read = read_events to a finished log, calc_all = calc_all_from_events from that log
  - plain_high_bytes / window_high_bytes: the default memory pool's used-memory high-water mark over a read
  - gpu name and power limit, read in the same run
usage: python tools/event_window_bench.py --config C2 --steps 5
       python tools/event_window_bench.py --config C3 --chunk-bytes 268435456 --steps 3
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from event_stream_bench import PoolHigh, export_blocks  # noqa: E402
from events_bench import END_MS, WINDOW_MS  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, default=256 << 20)
    ap_.add_argument("--days", type=float, default=27.0)
    ap_.add_argument("--steps", type=int, default=3)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_window_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    pool = PoolHigh()
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": names, "duration": WINDOW_MS // 1000}]})
    mepu = cfg.get("min_events_per_user", 0)
    n_bytes, n_lines, gen = export_blocks(cfg, a.fraction)
    whole = ctx.host_array(n_bytes, np.uint8)
    at = 0
    for b in gen():
        whole[at:at + len(b)] = b
        at += len(b)
    pieces = [whole[k:k + a.chunk_bytes] for k in range(0, n_bytes, a.chunk_bytes)]
    window = ur.EventWindow(f"{a.days} days", True)
    out = {"config": a.config, "fraction": a.fraction, "export_bytes": n_bytes, "n_lines": n_lines, "chunk_bytes": a.chunk_bytes,
           "days": a.days}
    t = {k: [] for k in ("plain_read", "window_read", "plain_calc_all", "window_calc_all")}
    for step in range(a.steps + 1):   # alternated; the first round warms up
        for kind, w in (("plain", None), ("window", window)):
            torch.cuda.synchronize()
            pool.reset()
            t0 = time.perf_counter()
            log = ctx.read_events(pieces, chunk_bytes=a.chunk_bytes, window=w, now_ms=END_MS)
            tr = (time.perf_counter() - t0) * 1e3
            out[f"{kind}_high_bytes"] = pool.read()
            if w is not None:
                out["n_expired"], out["n_duplicates"] = log.window_stats()
            t0 = time.perf_counter()
            body = ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx)
            tc = (time.perf_counter() - t0) * 1e3
            out[f"{kind}_body_bytes"] = len(body)
            log.free()
            if step:
                t[f"{kind}_read"].append(tr)
                t[f"{kind}_calc_all"].append(tc)
    for k, v in t.items():
        out[f"{k}_ms"] = round(statistics.median(v), 2)
    ctx.host_free(whole)
    name, plimit = gpu_info()
    out.update(gpu=name, power_limit_w=plimit)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
