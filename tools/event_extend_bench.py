"""Cost of keeping an event log resident across retrains with a sliding eventWindow (EventLog.extend) against what a caller
does without it: read the whole window's export again.

The export is event_stream_bench.py's (events_bench.py's line templates and generators) with eventTimes uniform over the
31 days before END_MS: days 0-29 are A, day 30 is B; the items' $set lines (eventTime END_MS, never expiring) are in A.
A is read as an extendable log with a 30-day window at now = END_MS - 1 day.  Then, alternated over --steps rounds (one
warm-up round first):
  (a) extend: EventLog.extend(B) with the window at now = END_MS (the cutoff moves one day: day 0 expires), to a finished
      log.  Each round extends a fresh extendable read of A, made untimed;
  (b) reread: read_events of A followed by B under the same window at END_MS, from pinned memory, to a finished log.
calc_all_from_events of the two logs must give equal bodies.  Both streamed in chunks of --chunk-bytes.  Prints one JSON
line: export_bytes, n_lines, new_bytes (B), extend_ms and reread_ms (medians), calc_all_ms (the reread log, median),
n_expired / n_duplicates of the extended log, resident_bytes of the extended log and of an extendable reread, and the
GPU's name and power limit, read in the same run.
usage: python tools/event_extend_bench.py --config C2 --steps 5
       python tools/event_extend_bench.py --config C3 --steps 3
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
from events_bench import CHUNK, END_MS, EV, SET, _digits, _holes, fill_events  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402

DAY = 86_400_000


def export_days(cfg: dict, fraction: float, host_array):
    """the export in pinned memory as A (days 0-29 and the $set lines) followed by B (day 30) -> (whole, len(A), n_lines)"""
    n_users, n_items, n_types = cfg["n_users"], cfg["n_items"], cfg["n_types"]
    per = int(cfg["n_events"] * fraction) // n_types
    n_bytes = per * n_types * len(EV) + n_items * len(SET)
    whole = host_array(n_bytes, np.uint8)
    rng = np.random.default_rng(5)
    tables_u = synth.user_tables(n_users)
    later = []   # B's blocks, written after A
    at = 0
    for t in range(n_types):
        users, items = synth.events_for_type(n_users, n_items, per, t, (tables_u, synth.item_tables(n_items, t)))
        for s in range(0, per, CHUNK):
            e = min(per, s + CHUNK)
            times = END_MS - rng.integers(1, 31 * DAY, e - s)
            new = times > END_MS - DAY
            for sel, dst in ((~new, None), (new, later)):
                k = int(sel.sum())
                out = np.empty(k * len(EV), np.uint8) if dst is not None else whole[at:at + k * len(EV)]
                fill_events(out, t, users[s:e][sel], items[s:e][sel], times[sel])
                if dst is not None:
                    dst.append(out)
                else:
                    at += k * len(EV)
        del users, items
    h = _holes(SET)
    for s in range(0, n_items, CHUNK):
        j = np.arange(s, min(n_items, s + CHUNK), dtype=np.int64)
        rows = np.empty((len(j), len(SET)), np.uint8)
        rows[:] = np.frombuffer(SET, dtype=np.uint8)
        rows[:, h[0]:h[0] + 9] = _digits(j, 9)
        rows[:, h[9]] = (48 + j % 10).astype(np.uint8)
        rows[:, h[10]] = (48 + j % 7).astype(np.uint8)
        whole[at:at + rows.size] = rows.reshape(-1)
        at += rows.size
    n_a = at
    for b in later:
        whole[at:at + len(b)] = b
        at += len(b)
    assert at == n_bytes
    return whole, n_a, per * n_types + n_items


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, default=256 << 20)
    ap_.add_argument("--no-dedup", action="store_true", help="the window without removeDuplicates")
    ap_.add_argument("--steps", type=int, default=3)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_extend_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": names, "duration": 30 * DAY // 1000}]})
    mepu = cfg.get("min_events_per_user", 0)
    whole, n_a, n_lines = export_days(cfg, a.fraction, ctx.host_array)
    A, B = whole[:n_a], whole[n_a:]
    window = ur.EventWindow("30 days", not a.no_dedup)
    out = {"config": a.config, "fraction": a.fraction, "export_bytes": len(whole), "n_lines": n_lines, "new_bytes": len(B),
           "chunk_bytes": a.chunk_bytes, "remove_duplicates": not a.no_dedup}
    t = {"extend": [], "reread": [], "calc_all": []}
    for step in range(a.steps + 1):   # alternated; the first round warms up
        log = ctx.read_events(A, chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS - DAY, extendable=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        log.extend(B, window=window, now_ms=END_MS)
        te = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        fresh = ctx.read_events(whole, chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS)
        tr = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        body = ur.calc_all_from_events(fresh, ap, mepu, now_ms=END_MS, ctx=ctx)
        tc = (time.perf_counter() - t0) * 1e3
        if step == 0:
            assert ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx) == body, "the extended log trains differently"
            assert log.window_stats() == fresh.window_stats() and log.info() == fresh.info()
            out["bodies_equal"] = True
            out["n_expired"], out["n_duplicates"] = log.window_stats()
            out["resident_bytes_extended"] = log.resident_bytes()
            with ctx.read_events(whole, chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS, extendable=True) as again:
                out["resident_bytes_reread_extendable"] = again.resident_bytes()
        log.free()
        fresh.free()
        if step:
            t["extend"].append(te)
            t["reread"].append(tr)
            t["calc_all"].append(tc)
    for k, v in t.items():
        out[f"{k}_ms"] = round(statistics.median(v), 2)
    ctx.host_free(whole)
    name, plimit = gpu_info()
    out.update(gpu=name, power_limit_w=plimit)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
