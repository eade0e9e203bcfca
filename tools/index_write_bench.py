"""Cost of the device side of writing the model index into Elasticsearch (CcoContext.index_write, ur.write_index): the body
format_model writes for a synth.py config's resident train with model_format_bench.py's two property fields per item (no
rankings), and synthesised _bulk responses for every request of the default cut (1000 documents, 1 MiB), all 201, and a
variant where 1 % of the documents are answered 429 and sent again in one retry round.  Prints one JSON line:
  - begin_fields_ms: the median wall time of index_write(body) + fields() (upload, parse, checks, the field scan; the call
    ends in a stream synchronise), begin_fields_gb_per_s the body bytes over it
  - responses_ms / responses_gb_per_s: reading every response (response() per request, each ending in a synchronise), the
    response bytes over that time; with_429 the same plus retry() and the retry round's responses
  - mirror_ms_per_mb: ur_model.index_fields + bulk_requests + bulk_item_statuses on the first --sample documents
  - parity_ok: the device's fields, cuts and statuses equal the mirror's on that sample
and the GPU's name and power limit, read in the same run.
usage: python tools/index_write_bench.py --config C3 [--steps 3 --warmup 1 --sample 20000]
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
from universal_recommender_b200 import ur_model as um  # noqa: E402


def model_body(ctx, config: str) -> bytes:
    cfg = synth.CONFIGS[config]
    n_types, n_items = cfg["n_types"], cfg["n_items"]
    w = synth.make(config, ctx=ctx, keep_dataset=True)
    _, h = ctx.train_dataset(w.dataset, [(500, 50, None)] * n_types, seed=42, flags=ur.FLAG_RESULT_NO_COUNT | ur.FLAG_RESULT_NO_LLR, keep=True)
    names = [f"e{t}" for t in range(n_types)]
    ids = [f"i{j}" for j in range(n_items)]
    j = np.repeat(np.arange(n_items), 2)
    values = [f'["c{x % 50}"]' if k % 2 == 0 else ("true" if x % 3 else "false") for k, x in enumerate(j.tolist())]
    props = (["category", "available"], *ur.encode_ids([ids[int(x)] for x in j]), np.tile(np.arange(2, dtype=np.int32), n_items),
             *ur.encode_ids(values))
    try:
        return ctx.format_model(h, names, ids, [ids] * n_types, props, None)
    finally:
        ctx.free_result(h)
        ctx.free_dataset(w.dataset)


def doc_ids(body: bytes) -> list[str]:
    lines = body.split(b"\n")
    return [json.loads(lines[k])["index"]["_id"] for k in range(0, len(lines) - 1, 2)]


def response(ids, statuses) -> bytes:
    items = []
    for i, st in zip(ids, statuses):
        if st == 201:
            items.append('{"index":{"_index":"urindex_1","_type":"items","_id":%s,"_version":1,"result":"created",'
                         '"_shards":{"total":2,"successful":1,"failed":0},"created":true,"status":201}}' % json.dumps(i))
        else:
            items.append('{"index":{"_index":"urindex_1","_type":"items","_id":%s,"status":429,"error":{"type":'
                         '"es_rejected_execution_exception","reason":"rejected execution of bulk"}}}' % json.dumps(i))
    return ('{"took":30,"errors":%s,"items":[%s]}' % ("true" if any(s != 201 for s in statuses) else "false", ",".join(items))).encode()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--config", default="C3")
    p.add_argument("--steps", type=int, default=3)
    p.add_argument("--warmup", type=int, default=1)
    p.add_argument("--sample", type=int, default=20000)
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("index_write_bench measures on the GPU: no CUDA device")
    ctx = ur.CcoContext(device=0)
    body = model_body(ctx, a.config)
    ids = doc_ids(body)
    db, bb = um.bulk_requests(body, 1000, 1 << 20)
    all_201 = [response(ids[db[q]:db[q + 1]], [201] * (db[q + 1] - db[q])) for q in range(len(db) - 1)]
    rejected = set(range(0, len(ids), 100))
    some_429 = [response(ids[db[q]:db[q + 1]], [429 if d in rejected else 201 for d in range(db[q], db[q + 1])]) for q in range(len(db) - 1)]

    begin_ms, resp_ms, r429_ms, fields = [], [], [], None
    for step in range(a.warmup + a.steps):
        t0 = time.perf_counter()
        w = ctx.index_write(body)
        fields = w.fields()
        t1 = time.perf_counter()
        for q, r in enumerate(all_201):
            w.response(q, r)
        t2 = time.perf_counter()
        res = w.finish()
        w.free()
        assert res.n_ok == len(ids)
        with ctx.index_write(body) as w2:
            w2.fields()
            t3 = time.perf_counter()
            for q, r in enumerate(some_429):
                w2.response(q, r)
            first, parts = w2.retry()
            for k, (dd, _) in enumerate(parts):
                w2.response(first + k, response([ids[d] for d in dd], [201] * len(dd)))
            t4 = time.perf_counter()
            res2 = w2.finish()
        assert res2.n_ok == len(ids) and sum(len(dd) for dd, _ in parts) == len(rejected)
        if step >= a.warmup:
            begin_ms.append((t1 - t0) * 1e3)
            resp_ms.append((t2 - t1) * 1e3)
            r429_ms.append((t4 - t3) * 1e3)
    resp_bytes = sum(len(r) for r in all_201)

    # the host mirror on a sample
    n = min(a.sample, len(ids))
    lines_end = 0
    for _ in range(2 * n):
        lines_end = body.index(b"\n", lines_end) + 1
    sample = body[:lines_end]
    t0 = time.perf_counter()
    m_fields = um.index_fields(sample)
    m_db, m_bb = um.bulk_requests(sample, 1000, 1 << 20)
    m_status = [s for q in range(len(m_db) - 1)
                for s, _, _ in um.bulk_item_statuses(response(ids[m_db[q]:m_db[q + 1]], [201] * (m_db[q + 1] - m_db[q])), ids[m_db[q]:m_db[q + 1]])]
    mirror_ms = (time.perf_counter() - t0) * 1e3
    with ctx.index_write(sample) as w:
        parity = w.fields() == m_fields and [list(x) for x in w.cuts()] == [m_db, m_bb]
        for q in range(len(m_db) - 1):
            w.response(q, response(ids[m_db[q]:m_db[q + 1]], [201] * (m_db[q + 1] - m_db[q])))
        parity = parity and list(w.finish().status) == m_status
    bm, rm, qm = statistics.median(begin_ms), statistics.median(resp_ms), statistics.median(r429_ms)
    out = {"config": a.config, "documents": len(ids), "body_bytes": len(body), "fields": len(fields), "requests": len(db) - 1,
           "begin_fields_ms": round(bm, 3), "begin_fields_gb_per_s": round(len(body) / bm / 1e6, 3),
           "response_bytes": resp_bytes, "responses_ms": round(rm, 3), "responses_gb_per_s": round(resp_bytes / rm / 1e6, 3),
           "with_429": {"rejected": len(rejected), "responses_and_retry_ms": round(qm, 3)},
           "mirror_sample_docs": n, "mirror_ms_per_mb": round(mirror_ms / (len(sample) / 1e6), 2), "parity_ok": bool(parity)}
    out["gpu"], out["power_limit_w"] = gpu_info()
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
