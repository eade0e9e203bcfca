"""Cost of building mixed queries on the device (CcoContext.mixed_queries, cco_mixed_queries): rows that each have any subset
of {user, item, item set}, over the export of tools/events_bench.py (a synth.py config as fixed-width JSON lines, read with
history retention) and the model index that calc_all_from_events writes from it.  --rows rows (default 10^6) in a seeded
mix of all eight member combinations; users and items drawn from the config's id spaces (so some are unknown), sets of 1
to --max-set ids drawn with the config's item popularity; every column passed as Arrow buffers with validity bitmaps.
Prints one JSON line:
  - mixed_queries_ms: the median of --steps calls after --warmup, each bracketed by a device synchronise; the time
    includes the upload, the copy back of the body and its copy into Python bytes
  - n_rows, n_elements, body_bytes, body_gb_per_s (body bytes per second of the median call)
  - single_ms: in the same loop, alternated with the mixed call, the user-, item- and item-set-query builders on the rows
    with only that member (users and items as Python lists, their interface; sets as Arrow buffers), and the mixed
    builder on the same rows (mixed_on_single_ms)
  - parity_ok: the device records equal ur_query.mixed_queries (the host mirror) for --sample rows of the batch, over a
    sample export (the first lines of each event type) and the whole index
  - gpu name and power limit, read in the same run
usage: python tools/mixed_queries_bench.py --config C3 --fraction 0.25 --steps 5 --warmup 1 [--rows 1000000] [--max-set 20]
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
from events_bench import END_MS, EV, _digits, build_export  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from item_set_queries_bench import ID_WIDTH, build_sets  # noqa: E402
from universal_recommender_b200 import events as E  # noqa: E402
from universal_recommender_b200 import ur_query as Q  # noqa: E402


def fixed_ids(prefix: str, x: np.ndarray):
    """-> (offsets, bytes) of the ids prefix + 9 digits"""
    b = np.empty((len(x), ID_WIDTH), dtype=np.uint8)
    b[:, 0] = ord(prefix)
    b[:, 1:] = _digits(x.astype(np.int64), ID_WIDTH - 1)
    return np.arange(len(x) + 1, dtype=np.int64) * ID_WIDTH, b.reshape(-1)


def build_rows(cfg: dict, n: int, max_set: int, seed: int = 13):
    """-> (kind [n] 0..7: bit 0 user, bit 1 item, bit 2 set; users, items, sets as Arrow buffers with validity bitmaps)"""
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 8, n)
    uo, ub = fixed_ids("u", rng.integers(0, cfg["n_users"] + cfg["n_users"] // 20, n))   # about 5 % unknown users
    io, ib = fixed_ids("i", rng.integers(0, cfg["n_items"] + cfg["n_items"] // 20, n))
    so, eo, eb = build_sets(cfg["n_items"], n, max_set, seed)
    bits = lambda b: np.packbits((kind >> b) & 1 == 1, bitorder="little")
    return kind, (uo, ub, bits(0)), (io, ib, bits(1)), (so, eo, eb, bits(2))


def as_lists(kind, users, items, sets, rows):
    """the Python columns (None for an absent member) of the given rows"""
    ub, ib, eb = users[1].tobytes(), items[1].tobytes(), sets[2].tobytes()
    uo, io, so, eo = users[0], items[0], sets[0], sets[1]
    u = [ub[uo[r]:uo[r + 1]].decode() if kind[r] & 1 else None for r in rows]
    i = [ib[io[r]:io[r + 1]].decode() if kind[r] & 2 else None for r in rows]
    s = [[eb[eo[e]:eo[e + 1]].decode() for e in range(so[r], so[r + 1])] if kind[r] & 4 else None for r in rows]
    return u, i, s


def subset(col, rows):
    """the Arrow buffers of a column restricted to rows (every row present)"""
    if len(col) == 3:
        o, b, _ = col
        lens = o[rows + 1] - o[rows]
        off = np.zeros(len(rows) + 1, dtype=np.int64)
        np.cumsum(lens, out=off[1:])
        idx = np.repeat(o[rows], lens) + (np.arange(off[-1]) - np.repeat(off[:-1], lens))
        return off, b[idx], None
    so, eo, eb, _ = col
    n = so[rows + 1] - so[rows]
    nso = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum(n, out=nso[1:])
    elems = np.repeat(so[rows], n) + (np.arange(nso[-1]) - np.repeat(nso[:-1], n))
    eoff, ebytes, _ = subset((eo, eb, None), elems)
    return nso, eoff, ebytes, None


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C3")
    p.add_argument("--fraction", type=float, default=0.25)
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--rows", type=int, default=1_000_000)
    p.add_argument("--max-set", type=int, default=20)
    p.add_argument("--sample", type=int, default=20_000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mixed_queries_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    buf, n_lines = build_export(ctx, cfg, a.fraction)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "availableDateName": "available", "expireDateName": "expires"})
    index = ur.calc_all_from_events(buf, ap, now_ms=END_MS, ctx=ctx, flags=0)
    log = ctx.read_events(buf, keep_history=True)
    kind, users, items, sets = build_rows(cfg, a.rows, a.max_set)
    query = Q.MixedQuery(blacklistItems=["i000000000", "i000000001", "i000000002"])

    # the single-member rows and their columns, in each builder's interface
    only = {k: np.flatnonzero(kind == k) for k in (1, 2, 4)}
    u_list = as_lists(kind, users, items, sets, only[1])[0]
    i_list = as_lists(kind, users, items, sets, only[2])[1]
    u_arrow, i_arrow, s_arrow = subset(users, only[1]), subset(items, only[2]), subset(sets, only[4])
    single = {
        "user_queries": lambda: ctx.user_queries(log, ap, query, u_list, END_MS),
        "item_queries": lambda: ctx.item_queries(index, ap, query, i_list, END_MS),
        "item_set_queries": lambda: ctx.item_set_queries(s_arrow[:3], ap, query, END_MS),
        "mixed_on_user_rows": lambda: ctx.mixed_queries(log, None, ap, query, u_arrow, now_ms=END_MS),
        "mixed_on_item_rows": lambda: ctx.mixed_queries(None, index, ap, query, None, i_arrow, now_ms=END_MS),
        "mixed_on_set_rows": lambda: ctx.mixed_queries(None, None, ap, query, None, None, s_arrow, now_ms=END_MS),
    }
    out = {}
    times = {k: [] for k in ["mixed"] + list(single)}
    for step in range(a.warmup + a.steps):   # alternated
        for k in times:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = ctx.mixed_queries(log, index, ap, query, users, items, sets, now_ms=END_MS) if k == "mixed" else single[k]()
            torch.cuda.synchronize()
            if step >= a.warmup:
                times[k].append((time.perf_counter() - t0) * 1e3)
            out[k] = r if k == "mixed" else r[0]
    ms = {k: round(statistics.median(v), 3) for k, v in times.items()}
    body, off = out["mixed"]
    single_equal = (out["mixed_on_user_rows"] == out["user_queries"] and out["mixed_on_item_rows"] == out["item_queries"]
                    and out["mixed_on_set_rows"] == out["item_set_queries"])
    log.free()

    # parity on a sample export (the first lines of each event type) with the whole index, for rows spread over the batch
    n_ev = n_lines - cfg["n_items"]
    per, L = n_ev // cfg["n_types"], len(EV)
    k = min(100_000 // cfg["n_types"], per)
    mv = memoryview(buf)
    sample = b"".join(bytes(mv[t * per * L:(t * per + k) * L]) for t in range(cfg["n_types"]))
    step = max(a.rows // max(a.sample, 1), 1)
    rows = np.arange(0, a.rows, step)[:a.sample]
    su, si, ss = as_lists(kind, users, items, sets, rows)
    with ctx.read_events(sample, keep_history=True) as slog:
        dev = ctx.mixed_queries(slog, index, ap, query, su, si, ss, now_ms=END_MS)
    host = Q.mixed_queries(E.read_export(sample), index, ap, query, su, si, ss, END_MS)
    parity = dev[0] == host[0] and np.array_equal(dev[1], host[1])
    name, plimit = gpu_info()
    print(json.dumps({
        "config": a.config, "fraction": a.fraction, "n_lines": n_lines, "index_bytes": len(index), "n_rows": a.rows,
        "n_elements": int(sets[0][-1]), "max_set": a.max_set, "mixed_queries_ms": ms["mixed"], "body_bytes": len(body),
        "body_gb_per_s": round(len(body) / (ms["mixed"] * 1e-3) / 1e9, 2), "bytes_per_record": round(len(body) / max(a.rows, 1), 1),
        "single_rows": {"user": len(only[1]), "item": len(only[2]), "item_set": len(only[4])},
        "single_ms": {k: v for k, v in ms.items() if k != "mixed"}, "single_equal": bool(single_equal),
        "parity_rows": len(rows), "parity_ok": bool(parity), "gpu": name, "power_limit_w": plimit}))
    ctx.host_free(buf)
    ctx.close()


if __name__ == "__main__":
    main()
