"""Cost of erasing users and items from a resident event log (EventLog.erase) against what a caller does without it: filter
the export and read it again.

The export is event_extend_bench.py's: eventTimes uniform over 31 days (event_stream_bench.py's line templates, users
"u#########" and items "i#########"), the items' $set lines among them.  It is read as an extendable log (interned with
--intern) under a 31-day window with removeDuplicates at now = END_MS.  Erase sets, seeded: 0.1 % of the users, 1 % of the
users, 1 % of the items.  Per set, alternated over --steps rounds (one warm-up round first):
  (a) erase: EventLog.erase on a fresh extendable read of X (made untimed), to a finished log;
  (b) reread: read_events of X - E (X without the erased lines, built untimed in pinned memory) under the same window and
      flags, to a finished log.
calc_all_from_events of the two logs must give equal bodies in every round.  Prints one JSON line per set: the sizes, the
lines erased, erase_ms and reread_ms (medians), and the GPU's name and power limit, read in the same run.
usage: python tools/event_erase_bench.py --config C2 --steps 5
       python tools/event_erase_bench.py --config C3 --steps 3 --intern
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
from event_extend_bench import DAY, export_days  # noqa: E402
from events_bench import END_MS, EV, SET, _holes  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402


def _numbers(rows: np.ndarray, at: int) -> np.ndarray:
    """the 9-digit id number at column `at` of fixed-width lines"""
    d = rows[:, at:at + 9].astype(np.int64) - 48
    return d @ (10 ** np.arange(8, -1, -1, dtype=np.int64))


def without(whole: np.ndarray, n_a: int, n_items: int, users: set, items: set, host_array) -> np.ndarray:
    """X - E in pinned memory: the export's event lines (fixed width, A's before the $set lines, B's after) and $set lines
    without the erased ones"""
    he, hs = _holes(EV), _holes(SET)
    n_set = n_items * len(SET)
    n_ev_a = (n_a - n_set) // len(EV)
    u = np.fromiter(users, np.int64, len(users))
    i = np.fromiter(items, np.int64, len(items))
    parts = []
    for lo, hi, width, hole_u, hole_i in ((0, n_ev_a * len(EV), len(EV), he[1], he[10]), (n_ev_a * len(EV), n_a, len(SET), None, hs[0]),
                                          (n_a, len(whole), len(EV), he[1], he[10])):
        rows = whole[lo:hi].reshape(-1, width)
        gone = np.isin(_numbers(rows, hole_i), i)
        if hole_u is not None:
            gone |= np.isin(_numbers(rows, hole_u), u)
        parts.append(rows[~gone].reshape(-1))
    out = host_array(sum(len(p) for p in parts), np.uint8)
    at = 0
    for p in parts:
        out[at:at + len(p)] = p
        at += len(p)
    return out


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, default=256 << 20)
    ap_.add_argument("--intern", action="store_true", help="interned logs (intern_ids=True)")
    ap_.add_argument("--steps", type=int, default=3)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_erase_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": names, "duration": 31 * DAY // 1000}]})
    mepu = cfg.get("min_events_per_user", 0)
    whole, n_a, n_lines = export_days(cfg, a.fraction, ctx.host_array)
    window = ur.EventWindow("31 days", True)
    kw = dict(chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS, extendable=True, intern_ids=a.intern)
    rng = np.random.default_rng(11)
    n_users, n_items = cfg["n_users"], cfg["n_items"]
    sets = {"users_0.1pct": (rng.choice(n_users, max(1, n_users // 1000), replace=False), []),
            "users_1pct": (rng.choice(n_users, max(1, n_users // 100), replace=False), []),
            "items_1pct": ([], rng.choice(n_items, max(1, n_items // 100), replace=False))}
    name, plimit = gpu_info()
    for label, (us, its) in sets.items():
        rest = without(whole, n_a, n_items, set(int(x) for x in us), set(int(x) for x in its), ctx.host_array)
        uid, iid = [f"u{int(x):09d}" for x in us], [f"i{int(x):09d}" for x in its]
        out = {"config": a.config, "fraction": a.fraction, "set": label, "intern": a.intern, "export_bytes": len(whole),
               "n_lines": n_lines, "rest_bytes": len(rest), "n_users": len(uid), "n_items": len(iid), "chunk_bytes": a.chunk_bytes}
        t = {"erase": [], "reread": []}
        for step in range(a.steps + 1):   # alternated; the first round warms up
            log = ctx.read_events(whole, **kw)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = log.erase(users=uid, items=iid)
            te = (time.perf_counter() - t0) * 1e3
            t0 = time.perf_counter()
            fresh = ctx.read_events(rest, **kw)
            tr = (time.perf_counter() - t0) * 1e3
            body = ur.calc_all_from_events(fresh, ap, mepu, now_ms=END_MS, ctx=ctx)
            assert ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx) == body, "the erased log trains differently"
            if step == 0:
                out.update(n_erased=st.n_lines, n_training_erased=st.n_training, n_ranking_erased=st.n_ranking,
                           n_property_erased=st.n_property_events, resident_bytes_erased=log.resident_bytes(),
                           resident_bytes_reread=fresh.resident_bytes())
            log.free()
            fresh.free()
            if step:
                t["erase"].append(te)
                t["reread"].append(tr)
        ctx.host_free(rest)
        out["bodies_equal"] = True
        for k, v in t.items():
            out[f"{k}_ms"] = round(statistics.median(v), 2)
        out.update(gpu=name, power_limit_w=plimit)
        print(json.dumps(out), flush=True)
    ctx.host_free(whole)
    ctx.close()


if __name__ == "__main__":
    main()
