"""Throughput of the string ingest (cco_ingest_strings): strings -> resident dataset + dictionaries, on one GPU.

Events are synth.py's integer streams of a config (C3, C4, ...), turned into variable-length decimal ids ("u" + user,
"i" + item) vectorised in numpy, straight into pinned host arrays.  Prints one JSON line:
  - ingest_ms_median / events_per_s: cco_ingest_strings wall time (the call ends in a stream synchronise), median of --steps
  - h2d_bytes: bytes the call copies host -> device; h2d_copy_ms: the same buffers copied alone (torch, pinned), the floor
  - host_prepare: ur.prepare on the first --sample events of each type, with the host's core count
  - parity: prepare_on_device == ur.prepare on that sample (dictionaries in order, row_ptr, col_idx); the full-size dataset
    trains (train_dataset, k = 50, m = 500)
  - gpu name and power limit, read in the same run
usage: python tools/ingest_strings_bench.py --config C3 --steps 5 --warmup 1 --sample 500000
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402


def events_for_type(n_users: int, n_items: int, n_events: int, t: int, tables, workers: int):
    """synth.events_for_type (the same counter-based stream, value for value) computed by `workers` threads over chunks"""
    from concurrent.futures import ThreadPoolExecutor
    (ucdf, uperm), (icdf, iperm) = tables
    users = np.empty(n_events, dtype=np.int64)
    items = np.empty(n_events, dtype=np.int64)
    with np.errstate(over="ignore"):
        base = synth._mix64(np.array([synth.type_seed(t)], dtype=np.uint64))[0]
    step = 1 << 22

    def chunk(s):
        with np.errstate(over="ignore"):
            e = np.arange(s + 1, min(n_events, s + step) + 1, dtype=np.uint64)
            h1 = synth._mix64(base + e * synth._GOLDEN)
            h2 = synth._mix64(h1 ^ synth._H2)
        u1 = (h1 >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
        u2 = (h2 >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
        users[s:s + len(e)] = uperm[np.minimum(np.searchsorted(ucdf, u1, side="right"), n_users - 1)]
        items[s:s + len(e)] = iperm[np.minimum(np.searchsorted(icdf, u2, side="right"), n_items - 1)]

    with ThreadPoolExecutor(workers) as ex:
        list(ex.map(chunk, range(0, n_events, step)))
    return users, items


def decimal_ids(ctx, prefix: bytes, x: np.ndarray):
    """prefix + str(x) for every x >= 0 -> (offsets int64[n + 1], bytes uint8[]) in pinned arrays, vectorised"""
    n = len(x)
    nd = np.ones(n, dtype=np.int64)
    p = 10
    while True:
        more = x >= p
        if not more.any():
            break
        nd += more
        p *= 10
    off = ctx.host_array(n + 1, np.int64)
    off[0] = 0
    np.cumsum(nd + len(prefix), out=off[1:])
    data = ctx.host_array(int(off[-1]), np.uint8)
    start = off[:-1]
    for k, ch in enumerate(prefix):
        data[start + k] = ch
    digits_end = off[1:] - 1          # last digit position
    rest = x.astype(np.int64, copy=True)
    for d in range(int(nd.max())):
        m = nd > d
        data[digits_end[m] - d] = (rest[m] % 10 + 48).astype(np.uint8)
        rest //= 10
    return off, data


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        plimit = float(q.stdout.strip().splitlines()[0])
    except Exception:
        plimit = None
    return name, plimit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=500_000, help="events per type for the host prepare and the parity check")
    a = ap.parse_args()
    cfg = synth.CONFIGS[a.config]
    n_types, n_users, n_items = cfg["n_types"], cfg["n_users"], cfg["n_items"]
    per_type = cfg["n_events"] // n_types
    min_ev = cfg.get("min_events_per_user") or 0
    ctx = ur.CcoContext(device=0)

    t0 = time.perf_counter()
    utab = synth.user_tables(n_users)
    columns = []
    for t in range(n_types):
        users, items = events_for_type(n_users, n_items, per_type, t, (utab, synth.item_tables(n_items, t)), os.cpu_count() or 1)
        columns.append((*decimal_ids(ctx, b"u", users), *decimal_ids(ctx, b"i", items)))
        del users, items
    build_s = time.perf_counter() - t0
    h2d_bytes = int(sum(c[0].nbytes + c[2].nbytes + (c[0][-1] - c[0][0]) + (c[2][-1] - c[2][0]) for c in columns))
    id_bytes = int(sum(c[1].nbytes + c[3].nbytes for c in columns))

    # the copy floor: the same pinned buffers host -> device, alone
    import torch
    dev = torch.device("cuda", 0)
    bufs = [torch.from_numpy(arr) for c in columns for arr in c]
    copy_ms = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs = [b.to(dev, non_blocking=True) for b in bufs]
        torch.cuda.synchronize()
        copy_ms.append((time.perf_counter() - t0) * 1e3)
        del outs
    torch.cuda.empty_cache()

    times = []
    ds = None
    for step in range(a.warmup + a.steps):
        if ds is not None:
            ctx.free_dataset(ds)
        t0 = time.perf_counter()
        ds = ctx.ingest_strings_dataset(columns, min_ev)
        dt = (time.perf_counter() - t0) * 1e3
        if step >= a.warmup:
            times.append(dt)
    shapes = [ctx.dataset_shape(ds, t) for t in range(n_types)]
    t0 = time.perf_counter()
    users = ctx.dataset_dictionary(ds, -1)
    items = [ctx.dataset_dictionary(ds, t) for t in range(n_types)]
    decode_ms = (time.perf_counter() - t0) * 1e3
    params = [(500, 50, None)] * n_types
    ctx.train_dataset(ds, params, seed=42, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR)   # warm-up
    t0 = time.perf_counter()
    res = ctx.train_dataset(ds, params, seed=42, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR)
    train_ms = (time.perf_counter() - t0) * 1e3
    trains = all(r[3][-1] > 0 for r in res) and len(users) == shapes[0][0] and all(len(items[t]) == shapes[t][1] for t in range(n_types))
    ctx.free_dataset(ds)

    # host prepare on a sample, and the parity check on the same sample
    S = min(a.sample, per_type)
    actions = []
    for t, (uo, ub, io, ib) in enumerate(columns):
        us = ur.decode_ids(uo[:S + 1], bytes(ub[:uo[S]]))
        its = ur.decode_ids(io[:S + 1], bytes(ib[:io[S]]))
        actions.append((f"e{t}", list(zip(us, its))))
    t0 = time.perf_counter()
    want = ur.prepare(actions, cfg.get("min_events_per_user"))
    host_s = time.perf_counter() - t0
    got = ur.prepare_on_device(actions, cfg.get("min_events_per_user"), ctx=ctx)
    parity = all(list(g.row_ids.inverse) == list(w.row_ids.inverse) and list(g.column_ids.inverse) == list(w.column_ids.inverse)
                 and np.array_equal(g.row_ptr, w.row_ptr) and np.array_equal(g.col_idx, w.col_idx)
                 for (_, g), (_, w) in zip(got, want))

    name, plimit = gpu_info()
    med = float(np.median(times))
    n_ev = per_type * n_types
    print(json.dumps({
        "tool": "ingest_strings_bench", "config": a.config, "gpu": name, "power_limit_w": plimit,
        "n_types": n_types, "events": n_ev, "min_events_per_user": min_ev,
        "ingest_ms_median": round(med, 2), "ingest_ms_all": [round(x, 2) for x in times],
        "events_per_s": round(n_ev / (med / 1e3)), "h2d_bytes": h2d_bytes, "id_bytes": id_bytes,
        "h2d_copy_ms": round(float(np.median(copy_ms)), 2), "h2d_copy_gb_s": round(h2d_bytes / (np.median(copy_ms) / 1e3) / 1e9, 1),
        "shapes": shapes, "dictionary_decode_ms": round(decode_ms, 1), "train_ms": round(train_ms, 2),
        "host_prepare": {"events": S * n_types, "s": round(host_s, 3), "events_per_s": round(S * n_types / host_s),
                         "cpu_count": os.cpu_count(), "threads": 1},
        "column_build_s": round(build_s, 1), "parity_ok": bool(parity), "trains": bool(trains),
    }), flush=True)
    ctx.close()
    if not (parity and trains):
        sys.exit(1)


if __name__ == "__main__":
    main()
