"""Cost of building the queries of a batchpredict query file (CcoContext.query_file: one Query JSON object per line, each
with its own template) over the export of tools/events_bench.py (a synth.py config as fixed-width JSON lines, read with
history retention) and the model index that calc_all_from_events writes from it.  --lines lines (default 10^6): the rows
of tools/mixed_queries_bench.py (a seeded mix of all eight member combinations) as JSON lines, line r drawing template
r % --templates (a template is its own "from"); every third line also has a two-id blacklistItems (a row member).
Prints one JSON line:
  - query_file_ms: the median of --steps calls after --warmup, split into read_ms (cco_query_file_read: upload, line
    split, tokenizer, row members, template ids), plans_ms (the templates decoded and planned on the host) and render_ms
    (cco_query_file_queries, the copy back and the Python bytes); each native step returns after its device work
  - mixed_ms: in the same loop, alternated, the same rows under one template through cco_mixed_queries (Arrow buffers
    with validity bitmaps, no blacklistItems, without a file), so the file path's overhead is
    visible
  - body_bytes, body_gb_per_s (body bytes per second of the median query_file call)
  - parity_ok: the device records equal ur_query.query_file (the host mirror) for --sample lines of the file, over a
    sample export (the first lines of each event type) and the index documents of the sampled items
  - gpu name and power limit, read in the same run
usage: python tools/query_file_bench.py --config C3 --fraction 0.25 --templates 64 [--lines 1000000] [--steps 3 --warmup 1]
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
from events_bench import END_MS, EV, build_export  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from mixed_queries_bench import as_lists, build_rows  # noqa: E402
from universal_recommender_b200 import events as E  # noqa: E402
from universal_recommender_b200 import ur_query as Q  # noqa: E402


def build_file(u, i, s, n_templates: int) -> bytes:
    lines = []
    for r in range(len(u)):
        t = r % n_templates
        d = {"from": t}
        if r % 3 == 0:
            d["blacklistItems"] = ["i%09d" % (r % 1000), "i000000001"]
        for k, v in (("user", u[r]), ("item", i[r]), ("itemSet", s[r])):
            if v is not None:
                d[k] = v
        lines.append(json.dumps(d))
    return ("\n".join(lines) + "\n").encode()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C3")
    p.add_argument("--fraction", type=float, default=0.25)
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--lines", type=int, default=1_000_000)
    p.add_argument("--templates", type=int, default=1)
    p.add_argument("--max-set", type=int, default=20)
    p.add_argument("--sample", type=int, default=300)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("query_file_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    buf, n_lines = build_export(ctx, cfg, a.fraction)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "availableDateName": "available", "expireDateName": "expires"})
    index = ur.calc_all_from_events(buf, ap, now_ms=END_MS, ctx=ctx, flags=0)
    log = ctx.read_events(buf, keep_history=True)
    kind, users, items, sets = build_rows(cfg, a.lines, a.max_set)
    u, i, s = as_lists(kind, users, items, sets, np.arange(a.lines))
    data = build_file(u, i, s, a.templates)

    split = {"read_ms": [], "plans_ms": [], "render_ms": []}

    def query_file():
        t = {}
        r = ctx.query_file(log, index, ap, data, END_MS, timings=t)
        for k in split:
            split[k].append(t[k])
        return r
    runs = {"query_file": query_file, "mixed": lambda: ctx.mixed_queries(log, index, ap, Q.MixedQuery(from_=0), users, items, sets, now_ms=END_MS)}
    times = {k: [] for k in runs}
    out = None
    for step in range(a.warmup + a.steps):   # alternated
        for k, f in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = f()
            torch.cuda.synchronize()
            if step >= a.warmup:
                times[k].append((time.perf_counter() - t0) * 1e3)
            if k == "query_file":
                out = r
        print(f"step {step}: " + ", ".join(f"{k} {v[-1]:.1f} ms" for k, v in times.items() if v), file=sys.stderr, flush=True)
    ms = {k: round(statistics.median(v), 3) for k, v in times.items()}
    parts = {k: round(statistics.median(v[a.warmup:]), 3) for k, v in split.items()}
    body, off = out
    log.free()

    # parity on a sample export (the first lines of each event type) with the whole index, for lines spread over the file
    n_ev = n_lines - cfg["n_items"]
    per, L = n_ev // cfg["n_types"], len(EV)
    k = min(100_000 // cfg["n_types"], per)
    mv = memoryview(buf)
    sample = b"".join(bytes(mv[t * per * L:(t * per + k) * L]) for t in range(cfg["n_types"]))
    step = max(a.lines // max(a.sample, 1), 1)
    lines = Q.query_file_lines(data)
    sub = b"".join(lines[r] + b"\n" for r in range(0, a.lines, step)[:a.sample])
    # the documents of the sampled items only (the mirror parses the index once per line); the others are unknown to both
    wanted = {json.loads(x).get("item") for x in sub.splitlines()}
    ix = index.split(b"\n")
    small = b"".join(ix[k] + b"\n" + ix[k + 1] + b"\n" for k in range(0, len(ix) - 1, 2) if json.loads(ix[k])["index"]["_id"] in wanted)
    with ctx.read_events(sample, keep_history=True) as slog:
        dev = ctx.query_file(slog, small, ap, sub, END_MS)
    host = Q.query_file(E.read_export(sample), small, ap, sub, END_MS)
    parity = dev[0] == host[0] and np.array_equal(dev[1], host[1])
    name, plimit = gpu_info()
    print(json.dumps({
        "config": a.config, "fraction": a.fraction, "n_lines": n_lines, "index_bytes": len(index), "file_lines": a.lines,
        "file_bytes": len(data), "templates": a.templates, "query_file_ms": ms["query_file"], **parts,
        "mixed_ms": ms["mixed"], "body_bytes": len(body), "body_gb_per_s": round(len(body) / (ms["query_file"] * 1e-3) / 1e9, 2),
        "parity_lines": sub.count(b"\n"), "parity_ok": bool(parity), "gpu": name, "power_limit_w": plimit}))
    ctx.host_free(buf)
    ctx.close()


if __name__ == "__main__":
    main()
