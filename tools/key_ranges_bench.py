"""Key ranges (CCO_FLAG_KEY_RANGES, DESIGN.md 3.1 "Key ranges") on the H100, in one call.

  1. A C4-shaped train (10M users, 500M events, m = 500, minEventsPerUser 3) over a 16M-item space: past the packed
     word (25 key bits leave 7 count bits, sampled marginals reach ~560), so it runs only with the flag.  Train time with
     the flag, the ranges of each indicator, and parity against the oracle on the same generator at 1/10 of the users and
     events (same item space, so the sample needs ranges too).
  2. The same shape over the 1M-item space of C4, where the word fits: the reference point of the same work unsplit.
  3. The C3 train with the flag on and off, alternated: where the word fits the flag must not move the time.
Every number is printed with the card's name and power limit.  The 16M-item space applies to both event types (synth
shapes share one item count), so the self indicator runs in ranges as well.

    python tools/key_ranges_bench.py [--steps 5] [--warmup 1] [--no-parity] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from universal_recommender_b200._native import FLAG_RESULT_ON_DEVICE  # noqa: E402

N_BIG = 16_777_216
SEED = 42


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def time_trains(ctx, w, flags, warmup, steps):
    """median / min ms of cco_train_dataset on the resident dataset (device events, ms_total), ranges, kept cells"""
    for _ in range(warmup):
        ctx.train_dataset(w.dataset, w.params, SEED, flags | FLAG_RESULT_ON_DEVICE, copy_arrays=False)
    ts = []
    for _ in range(steps):
        ctx.train_dataset(w.dataset, w.params, SEED, flags | FLAG_RESULT_ON_DEVICE, copy_arrays=False)
        ts.append(ctx.last_stats.ms_total)
    st = ctx.last_stats
    return {"ms_median": float(np.median(ts)), "ms_min": float(min(ts)), "ms_per_indicator": st.ms_indicator,
            "key_ranges": ctx.last_key_ranges, "out_nnz": st.out_nnz, "products": st.products,
            "n_kernel_launches": st.n_kernel_launches}


def c4_shape(ctx, n_items, warmup, steps):
    w = synth.make("C4", ctx=ctx, keep_dataset=True, n_items=n_items)
    try:
        r = {"shape": f"C4 generator, {w.n_users} users x {n_items} items, {w.n_events} events, m = 500"}
        if n_items == N_BIG:
            try:
                ctx.train_dataset(w.dataset, w.params, SEED, FLAG_RESULT_ON_DEVICE, copy_arrays=False)
                r["without_flag"] = "trained (unexpected)"
            except ur.CcoError as e:
                r["without_flag"] = f"refused, status {e.status}"
        r.update(time_trains(ctx, w, ur.FLAG_KEY_RANGES, warmup, steps))
        return r
    finally:
        ctx.free_dataset(w.dataset)


def parity_sample(ctx):
    """the C4 generator at 1/10 of the users and events over the 16M-item space, flag on, against the oracle"""
    from oracle import oracle as orc
    from oracle import parity as par
    c = synth.CONFIGS["C4"]
    sw = synth.make("C4", ctx=ctx, n_items=N_BIG, n_users=c["n_users"] // 10, n_events=c["n_events"] // 10)
    got = ctx.train_csr(sw.mats, sw.params, SEED, ur.FLAG_KEY_RANGES)
    ranges = ctx.last_key_ranges
    t0 = time.perf_counter()
    ref = orc.train([orc.Csr(*m) for m in sw.mats], [orc.Params(*p) for p in sw.params], SEED, 0, os.cpu_count() or 1)
    out = par.compare(ref, got, sw.n_users)
    out.update({"sample": f"{sw.n_users} users x {N_BIG} items, {sw.n_events} events", "key_ranges": ranges,
                "oracle_s": time.perf_counter() - t0})
    return out


def c3_flag_ab(ctx, warmup, steps, rounds=3):
    w = synth.make("C3", ctx=ctx, keep_dataset=True)
    try:
        runs = {"off": [], "on": []}
        for _ in range(rounds):
            for tag, fl in (("off", 0), ("on", ur.FLAG_KEY_RANGES)):
                runs[tag].append(time_trains(ctx, w, fl, warmup, steps))
        return {k: {"ms_median": [r["ms_median"] for r in v], "key_ranges": v[-1]["key_ranges"],
                    "n_kernel_launches": v[-1]["n_kernel_launches"]} for k, v in runs.items()}
    finally:
        ctx.free_dataset(w.dataset)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to DIR/key_ranges_bench.json")
    args = ap.parse_args()
    ctx = ur.CcoContext(device=0)
    res = {"card": card()}
    res["c4_16m"] = c4_shape(ctx, N_BIG, args.warmup, args.steps)
    print(json.dumps({"c4_16m": res["c4_16m"], **res["card"]}), flush=True)
    res["c4_1m"] = c4_shape(ctx, synth.CONFIGS["C4"]["n_items"], args.warmup, args.steps)
    print(json.dumps({"c4_1m": res["c4_1m"], **res["card"]}), flush=True)
    res["c3_flag"] = c3_flag_ab(ctx, args.warmup, args.steps)
    print(json.dumps({"c3_flag": res["c3_flag"], **res["card"]}), flush=True)
    if not args.no_parity:
        res["parity_16m_tenth"] = parity_sample(ctx)
        print(json.dumps({"parity_16m_tenth": res["parity_16m_tenth"], **res["card"]}, default=str), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "key_ranges_bench.json"), "w") as f:
            json.dump(res, f, indent=1, default=str)
    ctx.close()


if __name__ == "__main__":
    main()
