"""Cost of training from a PredictionIO event export parsed on the device (CcoContext.read_events, ingest_event_log,
ur.calc_all_from_events) against the host path that builds Python tuples for calc_all_on_device.

The export of a synth.py config is assembled on the host with numpy, not a Python loop: fixed-width ids ("u%09d",
"i%09d"), event names "t<type>", millisecond ISO times over 30 days ending at END_MS, then one `$set` line per primary item
(a JSON array and a number).  It lives in pinned host memory.  Prints one JSON line:
  - export_bytes, n_lines, copy_ms_median: a host -> device copy of the same pinned bytes alone
  - read_ms_median (cco_event_log_read), ingest_ms_median (cco_event_log_ingest), calc_all_ms_median (the whole
    calc_all_from_events from the bytes: read, ingest, train, rankings, properties, bulk body), medians of --steps
  - parse_gbps: export bytes / read time, against copy_gbps
  - on a sample (the first --sample / n_types lines of each type and every `$set` line): tuple_path_ms
    (events.read_export building the tuples + calc_all_on_device) and device_path_ms (calc_all_from_events on the same
    bytes), each warmed up once, then alternated --steps times (medians), and parity_ok (the two bodies are equal)
  - gpu name and power limit, read in the same run
usage: python tools/events_bench.py --config C2 --steps 5 --warmup 1 --sample 200000 [--fraction 0.25]
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
from ingest_strings_bench import gpu_info  # noqa: E402
from universal_recommender_b200 import events as E  # noqa: E402

END_MS = 1_700_000_000_000
WINDOW_MS = 30 * 86_400_000
EV = (b'{"event":"t#","entityType":"user","entityId":"u#########","targetEntityType":"item","targetEntityId":"i#########",'
      b'"eventTime":"#######################Z"}\n')
SET = b'{"event":"$set","entityType":"item","entityId":"i#########","properties":{"category":["c#"],"defaultRank":#.5},"eventTime":"2023-11-14T22:13:20.000Z"}\n'
CHUNK = 1 << 22


def _holes(tmpl: bytes) -> list[int]:
    return [k for k, c in enumerate(tmpl) if c == ord("#")]


def _digits(x: np.ndarray, width: int) -> np.ndarray:
    return ((x[:, None] // (10 ** np.arange(width - 1, -1, -1, dtype=np.int64))) % 10 + 48).astype(np.uint8)


def fill_events(out: np.ndarray, t: int, users: np.ndarray, items: np.ndarray, times: np.ndarray):
    """write len(users) event lines of type t into out (n x len(EV) bytes)"""
    h = _holes(EV)
    rows = out.reshape(len(users), len(EV))
    rows[:] = np.frombuffer(EV, dtype=np.uint8)
    rows[:, h[0]] = 48 + t
    rows[:, h[1]:h[1] + 9] = _digits(users, 9)
    rows[:, h[10]:h[10] + 9] = _digits(items, 9)
    iso = np.datetime_as_string(times.astype("datetime64[ms]"), unit="ms").astype("S23")
    rows[:, h[19]:h[19] + 23] = iso.view(np.uint8).reshape(len(users), 23)


def build_export(ctx, cfg: dict, fraction: float):
    """-> (pinned uint8 array, n_lines): each type's events as one block of fixed-width lines (type t's block starts at
    line t * per), then the `$set` lines"""
    n_users, n_items, n_types = cfg["n_users"], cfg["n_items"], cfg["n_types"]
    if n_types > 10:
        raise SystemExit("the event line template holds a one-digit event name: at most 10 types")
    per = int(cfg["n_events"] * fraction) // n_types
    n_ev = per * n_types
    total = n_ev * len(EV) + n_items * len(SET)
    buf = ctx.host_array(total, np.uint8)
    tables_u = synth.user_tables(n_users)
    at = 0
    rng = np.random.default_rng(5)
    for t in range(n_types):
        users, items = synth.events_for_type(n_users, n_items, per, t, (tables_u, synth.item_tables(n_items, t)))
        for s in range(0, per, CHUNK):
            e = min(per, s + CHUNK)
            times = END_MS - rng.integers(1, WINDOW_MS, e - s)
            fill_events(buf[at:at + (e - s) * len(EV)], t, users[s:e], items[s:e], times)
            at += (e - s) * len(EV)
    h = _holes(SET)
    rows = buf[at:].reshape(n_items, len(SET))
    rows[:] = np.frombuffer(SET, dtype=np.uint8)
    j = np.arange(n_items, dtype=np.int64)
    rows[:, h[0]:h[0] + 9] = _digits(j, 9)
    rows[:, h[9]] = (48 + j % 10).astype(np.uint8)
    rows[:, h[10]] = (48 + j % 7).astype(np.uint8)
    return buf, n_ev + n_items


def timed(fn, steps: int, warmup: int):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--steps", type=int, default=5)
    ap_.add_argument("--warmup", type=int, default=1)
    ap_.add_argument("--sample", type=int, default=200_000)
    ap_.add_argument("--fraction", type=float, default=1.0)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("events_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    t0 = time.perf_counter()
    buf, n_lines = build_export(ctx, cfg, a.fraction)
    build_s = time.perf_counter() - t0
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": names, "duration": WINDOW_MS // 1000}]})
    mepu = cfg.get("min_events_per_user", 0)

    dev = torch.empty(len(buf), dtype=torch.uint8, device="cuda")
    host = torch.from_numpy(buf)
    copy_ms = timed(lambda: dev.copy_(host, non_blocking=True), a.steps, a.warmup)
    del dev

    def read():
        ctx.read_events(buf).free()
    read_ms = timed(read, a.steps, a.warmup)
    log = ctx.read_events(buf)

    def ingest():
        ds, _, _ = ctx.ingest_event_log(log, names, mepu)
        ctx.free_dataset(ds)
    ingest_ms = timed(ingest, a.steps, a.warmup)
    info = log.info()
    log.free()
    calc_ms = timed(lambda: ur.calc_all_from_events(buf, ap, mepu, now_ms=END_MS, ctx=ctx), a.steps, a.warmup)

    # the tuple path on a sample: the first --sample event lines of each type's block and every `$set` line
    n_ev = n_lines - cfg["n_items"]
    per = n_ev // cfg["n_types"]
    k = min(a.sample // cfg["n_types"], per)
    mv, L = memoryview(buf), len(EV)   # fixed-width lines: type t's block starts at line t * per
    sample = b"".join([bytes(mv[t * per * L:(t * per + k) * L]) for t in range(cfg["n_types"])] + [bytes(mv[n_ev * L:])])
    def tuple_path():
        m = E.read_export(sample)
        return ur.calc_all_on_device(m.events, m.set_events, ap, mepu, now_ms=END_MS, ctx=ctx, ranking_events=m.ranking_events)

    def device_path():
        return ur.calc_all_from_events(sample, ap, mepu, now_ms=END_MS, ctx=ctx)
    want, got = tuple_path(), device_path()   # warm-up
    t_tuple, t_dev = [], []
    for _ in range(a.steps):   # alternated, so that drift on a shared host touches both
        t0 = time.perf_counter()
        tuple_path()
        t_tuple.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        device_path()
        t_dev.append((time.perf_counter() - t0) * 1e3)
    tuple_ms, device_ms = statistics.median(t_tuple), statistics.median(t_dev)
    name, plimit = gpu_info()
    print(json.dumps({
        "config": a.config, "fraction": a.fraction, "export_bytes": len(buf), "n_lines": n_lines, "build_export_s": round(build_s, 2),
        "copy_ms_median": round(copy_ms, 3), "copy_gbps": round(len(buf) / copy_ms / 1e6, 2),
        "read_ms_median": round(read_ms, 3), "parse_gbps": round(len(buf) / read_ms / 1e6, 2),
        "ingest_ms_median": round(ingest_ms, 3), "calc_all_ms_median": round(calc_ms, 3),
        "names": info.names, "n_training": info.n_training, "n_property_events": info.n_property_events,
        "sample_lines": k * cfg["n_types"] + cfg["n_items"], "tuple_path_ms": round(tuple_ms, 1), "device_path_ms": round(device_ms, 1),
        "parity_ok": got == want, "gpu": name, "power_limit_w": plimit}))
    ctx.host_free(buf)
    ctx.close()


if __name__ == "__main__":
    main()
