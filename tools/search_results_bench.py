"""Cost of reading Elasticsearch _msearch responses into PredictedResults (CcoContext.search_results) over responses
synthesised from the model index that calc_all_from_events writes from the export of tools/events_bench.py: --records
records of --hits hits each, every hit an index document as its _source with a float32 score text (as ES writes them),
streamed in bodies of --per-body records, every record withRanks.  Prints one JSON line:
  - end_to_end_ms / end_to_end_gb_per_s: the median of --steps calls after --warmup (body bytes over wall-clock time of
    the whole call: staging, copies, kernels, the copy back and the Python columns)
  - kernel_ms / kernel_gb_per_s: the sum of the CUDA kernel times of one call under torch.profiler, in a run of its own;
    kernel_ms_by_name: the eight largest, summed over the call's bodies
  - h2d_ms / h2d_gb_per_s: the host-to-device copy of every body alone, from pinned memory (CUDA events)
  - n_exact: numbers converted on the host's exact path; parity_ok: the device text and columns equal ur_predict's on
    --sample records
  - gpu name and power limit, read in the same run
usage: python tools/search_results_bench.py --config C3 --fraction 0.25 [--records 50000] [--steps 3 --warmup 1]
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
from events_bench import END_MS, build_export  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from universal_recommender_b200 import ur_predict as P  # noqa: E402


def build_bodies(index: bytes, n_records: int, n_hits: int, per_body: int, seed: int = 7) -> list[bytes]:
    lines = index.split(b"\n")
    docs = [(json.loads(lines[k])["index"]["_id"], lines[k + 1]) for k in range(0, len(lines) - 1, 2)]
    rng = np.random.default_rng(seed)
    scores = rng.random(n_records * n_hits, dtype=np.float32) * 20
    pick = rng.integers(0, len(docs), n_records * n_hits)
    bodies, els = [], []
    for r in range(n_records):
        hits = []
        for k in range(r * n_hits, (r + 1) * n_hits):
            did, src = docs[pick[k]]
            hits.append(b'{"_index":"urindex","_type":"items","_id":' + json.dumps(did).encode() + b',"_score":'
                        + str(scores[k]).encode() + b',"_source":' + src + b"}")
        els.append(b'{"took":3,"timed_out":false,"hits":{"total":' + str(n_hits).encode() + b',"max_score":1.0,"hits":['
                   + b",".join(hits) + b']},"status":200}')
        if len(els) == per_body or r == n_records - 1:
            bodies.append(b'{"took":5,"responses":[' + b",".join(els) + b"]}")
            els = []
    return bodies


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C3")
    p.add_argument("--fraction", type=float, default=0.25)
    p.add_argument("--records", type=int, default=50_000)
    p.add_argument("--hits", type=int, default=20)
    p.add_argument("--per-body", type=int, default=1000)
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sample", type=int, default=2000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("search_results_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    buf, _ = build_export(ctx, cfg, a.fraction)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names})
    index = ur.calc_all_from_events(buf, ap, now_ms=END_MS, ctx=ctx, flags=0)
    bodies = build_bodies(index, a.records, a.hits, a.per_body)
    nbytes = sum(len(b) for b in bodies)
    counts = [min(a.per_body, a.records - i) for i in range(0, a.records, a.per_body)]
    times, res = [], None
    for it in range(a.warmup + a.steps):
        t0 = time.perf_counter()
        res = ctx.search_results(bodies, ap, with_ranks=True, counts=counts)
        if it >= a.warmup:
            times.append((time.perf_counter() - t0) * 1e3)
    ms = statistics.median(times)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.search_results(bodies, ap, with_ranks=True, counts=counts)
    kern = {e.key: e.device_time_total for e in prof.key_averages() if "Memcpy" not in e.key and "Memset" not in e.key}
    kern_us = sum(kern.values())
    by_kernel = {k.split("(")[0].replace("void ", "").replace("cco::", ""): round(v / 1e3, 3)
                 for k, v in sorted(kern.items(), key=lambda kv: -kv[1])[:8]}
    # the host-to-device copy alone: every body from pinned memory, CUDA events around the copies
    pinned = [torch.frombuffer(bytearray(b), dtype=torch.uint8).pin_memory() for b in bodies]
    dev = torch.empty(max(len(b) for b in bodies), dtype=torch.uint8, device="cuda")
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for x in pinned:
        dev[:len(x)].copy_(x, non_blocking=True)
    t1.record()
    torch.cuda.synchronize()
    h2d_ms = t0.elapsed_time(t1)
    # parity on the first records against the mirror
    k = min(a.sample, a.per_body)
    first = P.predictions(bodies[0], P.ranking_names(ap), True)[:k]
    parity = res.records()[:k] == [x.text() for x in first] and res.ids[:res.hit_offsets[k]] == [i for x in first for i, _ in x.items]
    name, plimit = gpu_info()
    print(json.dumps({"config": a.config, "fraction": a.fraction, "records": a.records, "hits_per_record": a.hits,
                      "records_per_body": a.per_body, "bodies": len(bodies), "body_bytes": nbytes,
                      "end_to_end_ms": round(ms, 3), "end_to_end_gb_per_s": round(nbytes / ms / 1e6, 2),
                      "kernel_ms": round(kern_us / 1e3, 3), "kernel_gb_per_s": round(nbytes / max(kern_us, 1e-9) / 1e3, 2),
                      "kernel_ms_by_name": by_kernel, "h2d_ms": round(h2d_ms, 3), "h2d_gb_per_s": round(nbytes / h2d_ms / 1e6, 2),
                      "n_exact": int(res.n_exact), "parity_records": k, "parity_ok": bool(parity), "gpu": name, "power_limit_w": plimit}))


if __name__ == "__main__":
    main()
