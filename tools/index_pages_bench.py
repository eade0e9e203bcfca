"""Cost of reading the model index back from Elasticsearch scroll pages (CcoContext.index_pages / ur.index_from_pages):
the index calc_all_from_events writes from the export of tools/events_bench.py, rendered as the pages a scroll of
--page-hits hits returns, with compact and with pretty-printed (?pretty) bodies.  Prints one JSON line with, per layout:
  - end_to_end_ms / end_to_end_gb_per_s: the median of --steps reads after --warmup (page bytes over the wall-clock time
    of the whole read: staging, copies, kernels, the copy back of the documents and the body's assembly)
  - kernel_ms / kernel_ms_by_name: the CUDA kernel times of one read under torch.profiler, in a run of its own
  - h2d_ms: the host-to-device copy of every page alone, from pinned memory (CUDA events)
  - mirror_ms_per_mb: ur_model.index_from_pages on the first --sample pages, per MB of page
  - parity_ok: the device body equals the index body (and the mirror's, on the sample)
and the GPU's name and power limit, read in the same run.
usage: python tools/index_pages_bench.py --config C3 --fraction 1.0 [--page-hits 1000] [--steps 3 --warmup 1]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from events_bench import END_MS, build_export  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402
from universal_recommender_b200 import ur_model as um  # noqa: E402


def render_pages(index: bytes, page_hits: int, pretty: bool) -> list[bytes]:
    """the scroll pages of the index: ES's hit members around each document, the final empty page"""
    from search_results_data import pretty as reindent
    lines = index.split(b"\n")
    docs = [(json.loads(lines[k])["index"]["_id"], lines[k + 1]) for k in range(0, len(lines) - 1, 2)]
    head = b'{"_scroll_id":"DXF1ZXJ5QW5kRmV0Y2gBAAAAAAAAAD4WYm9laVYtZndUQlNsdDcwakFMNjU1QQ==","took":12,"timed_out":false,' \
        b'"_shards":{"total":1,"successful":1,"skipped":0,"failed":0},"hits":{"total":{"value":' + str(len(docs)).encode() + \
        b',"relation":"eq"},"max_score":1.0,"hits":['
    pages = []
    for a in range(0, len(docs) + 1, page_hits):
        hits = [b'{"_index":"urindex","_type":"_doc","_id":' + json.dumps(i).encode() + b',"_score":1.0,"_source":' + s + b"}"
                for i, s in docs[a:a + page_hits]]
        text = head + b",".join(hits) + b"]}}"
        pages.append((reindent(text.decode()) + "\n").encode() if pretty else text)
    return pages


def measure(ctx, pages, index, steps, warmup, sample):
    import torch
    from torch.profiler import ProfilerActivity, profile
    nbytes = sum(len(p) for p in pages)
    times, body = [], None
    for it in range(warmup + steps):
        t0 = time.perf_counter()
        body = ur.index_from_pages(pages, ctx=ctx)
        if it >= warmup:
            times.append((time.perf_counter() - t0) * 1e3)
    ms = statistics.median(times)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ur.index_from_pages(pages, ctx=ctx)
    kern = {e.key: e.device_time_total for e in prof.key_averages() if "Memcpy" not in e.key and "Memset" not in e.key}
    by_kernel = {k.split("(")[0].replace("void ", "").replace("cco::", ""): round(v / 1e3, 3)
                 for k, v in sorted(kern.items(), key=lambda kv: -kv[1])[:8]}
    pinned = [torch.frombuffer(bytearray(p), dtype=torch.uint8).pin_memory() for p in pages]
    dev = torch.empty(max(len(p) for p in pages), dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for x in pinned:
        dev[:len(x)].copy_(x, non_blocking=True)
    e1.record()
    torch.cuda.synchronize()
    h2d_ms = e0.elapsed_time(e1)
    few = pages[:sample]
    t0 = time.perf_counter()
    mirror, _, _ = um.index_from_pages(few)
    mirror_ms = (time.perf_counter() - t0) * 1e3
    with ctx.index_pages() as r:   # the sample alone: its pages hold fewer documents than hits.total
        for x in few:
            r.append(x)
        got_few = r.finish()
    return {"pages": len(pages), "page_bytes": nbytes, "end_to_end_ms": round(ms, 3), "end_to_end_gb_per_s": round(nbytes / ms / 1e6, 3),
            "kernel_ms": round(sum(kern.values()) / 1e3, 3), "kernel_ms_by_name": by_kernel, "h2d_ms": round(h2d_ms, 3),
            "mirror_ms_per_mb": round(mirror_ms / (sum(len(p) for p in few) / 1e6), 2),
            "parity_ok": bool(body == index and got_few == mirror)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C3")
    p.add_argument("--fraction", type=float, default=1.0)
    p.add_argument("--page-hits", type=int, default=1000)
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sample", type=int, default=3)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("index_pages_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    buf, _ = build_export(ctx, cfg, a.fraction)
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names})
    index = ur.calc_all_from_events(buf, ap, now_ms=END_MS, ctx=ctx, flags=0)
    out = {"config": a.config, "fraction": a.fraction, "page_hits": a.page_hits, "index_bytes": len(index)}
    for layout, pretty in (("compact", False), ("pretty", True)):
        out[layout] = measure(ctx, render_pages(index, a.page_hits, pretty), index, a.steps, a.warmup, a.sample)
    out["gpu"], out["power_limit_w"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
