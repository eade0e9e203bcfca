"""Cost of a streamed read of a PredictionIO event export (cco_event_log_begin / _append / _finish through
CcoContext.read_events) against the one-piece read (cco_event_log_read), and what it makes possible: exports larger than
device memory.

The export is events_bench.py's (fill_events, the same line templates and generators), produced chunk by chunk from a
generator, so that no host buffer the size of the export exists.  Prints one JSON line:
  - export_bytes, n_lines, chunk_bytes (with --fit: one "sweep" entry per chunk_bytes)
  - read_ms (the streamed read from the generator: generation excluded, the generator's blocks are made before timing)
    only when --fit: stream_read_ms and whole_read_ms on the same pinned bytes, alternated --steps times (medians), and
    bodies_equal (calcAll bodies of both logs)
  - parse_gbps (export bytes / streamed read time), finish_ms (cco_event_log_finish alone)
  - ingest_ms and calc_all_ms (calc_all_from_events from the streamed log), or the error a stage ended in
  - read_high_bytes: the device's default memory pool's CU_MEMPOOL_ATTR_USED_MEM_HIGH, reset before the read and read
    after it (whole_read_high_bytes likewise with --fit).  The library's large buffers come from cudaMallocAsync on that
    pool; the 64 MB scratch slabs of trains are cudaMalloc and are not in the figure.
  - gpu name and power limit, read in the same run
usage: python tools/event_stream_bench.py --config C3 --chunk-bytes 268435456 1073741824 --fit --steps 3
       python tools/event_stream_bench.py --config C4 --chunk-bytes 1073741824 [--fraction 0.1]
"""
from __future__ import annotations

import argparse
import ctypes as C
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
from events_bench import CHUNK, END_MS, EV, SET, WINDOW_MS, _digits, _holes, fill_events  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402

CU_MEMPOOL_ATTR_USED_MEM_HIGH = 8


class PoolHigh:
    """the default memory pool of device 0: reset / read its used-memory high-water mark through the driver API"""

    def __init__(self):
        self.cu = C.CDLL("libcuda.so.1")
        dev, self.pool = C.c_int(), C.c_void_p()
        assert self.cu.cuDeviceGet(C.byref(dev), 0) == 0
        assert self.cu.cuDeviceGetDefaultMemPool(C.byref(self.pool), dev) == 0

    def reset(self):
        z = C.c_uint64(0)
        assert self.cu.cuMemPoolSetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_HIGH, C.byref(z)) == 0

    def read(self) -> int:
        v = C.c_uint64(0)
        assert self.cu.cuMemPoolGetAttribute(self.pool, CU_MEMPOOL_ATTR_USED_MEM_HIGH, C.byref(v)) == 0
        return v.value


def export_blocks(cfg: dict, fraction: float):
    """the bytes of events_bench.build_export, block by block (at most CHUNK lines each); -> (n_bytes, n_lines, generator)"""
    n_users, n_items, n_types = cfg["n_users"], cfg["n_items"], cfg["n_types"]
    per = int(cfg["n_events"] * fraction) // n_types

    def gen():
        tables_u = synth.user_tables(n_users)
        rng = np.random.default_rng(5)
        buf = np.empty(CHUNK * len(EV), np.uint8)
        for t in range(n_types):
            users, items = synth.events_for_type(n_users, n_items, per, t, (tables_u, synth.item_tables(n_items, t)))
            for s in range(0, per, CHUNK):
                e = min(per, s + CHUNK)
                times = END_MS - rng.integers(1, WINDOW_MS, e - s)
                out = buf[:(e - s) * len(EV)]
                fill_events(out, t, users[s:e], items[s:e], times)
                yield out
            del users, items
        h = _holes(SET)
        for s in range(0, n_items, CHUNK):
            j = np.arange(s, min(n_items, s + CHUNK), dtype=np.int64)
            rows = np.empty((len(j), len(SET)), np.uint8)
            rows[:] = np.frombuffer(SET, dtype=np.uint8)
            rows[:, h[0]:h[0] + 9] = _digits(j, 9)
            rows[:, h[9]] = (48 + j % 10).astype(np.uint8)
            rows[:, h[10]] = (48 + j % 7).astype(np.uint8)
            yield rows.reshape(-1)
    return per * n_types * len(EV) + n_items * len(SET), per * n_types + n_items, gen


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C3")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, nargs="+", default=[1 << 30], help="with --fit, a sweep over several")
    ap_.add_argument("--fit", action="store_true", help="the export also fits in pinned host memory: alternate with the whole read")
    ap_.add_argument("--steps", type=int, default=3)
    ap_.add_argument("--no-train", action="store_true")
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_stream_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    pool = PoolHigh()
    names = [f"t{t}" for t in range(cfg["n_types"])]
    ap = ur.URAlgorithmParams.from_engine_json({"eventNames": names, "seed": 1, "rankings": [
        {"name": "popRank", "type": "popular", "eventNames": names, "duration": WINDOW_MS // 1000}]})
    mepu = cfg.get("min_events_per_user", 0)
    n_bytes, n_lines, gen = export_blocks(cfg, a.fraction)
    out = {"config": a.config, "fraction": a.fraction, "export_bytes": n_bytes, "n_lines": n_lines}
    L = ctx._L

    def stream(blocks, chunk_bytes):
        """a streamed read of the blocks: (log, read ms excluding the blocks' generation, finish ms)"""
        h = C.c_void_p()
        ur._native.check(L.cco_event_log_begin(ctx._h, chunk_bytes, C.byref(h)))
        ms = 0.0
        for b in blocks:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ur._native.check(L.cco_event_log_append(h, b.ctypes.data, len(b)))
            ms += (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        ur._native.check(L.cco_event_log_finish(h))
        fin = (time.perf_counter() - t0) * 1e3
        return ctx._adopt_log(h), ms + fin, fin

    if a.fit:
        whole = ctx.host_array(n_bytes, np.uint8)
        at = 0
        for b in gen():
            whole[at:at + len(b)] = b
            at += len(b)
        out["sweep"] = []
        for cb in a.chunk_bytes:
            pieces = [whole[k:k + cb] for k in range(0, n_bytes, cb)]
            bodies = []
            t_s, t_w, t_f = [], [], []
            for step in range(a.steps + 1):   # alternated; the first round warms up
                pool.reset()
                log, ms, fin = stream(pieces, cb)
                hs = pool.read()
                if step == 0:
                    bodies.append(ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx))
                log.free()
                torch.cuda.synchronize()
                pool.reset()
                t0 = time.perf_counter()
                log = ctx.read_events(whole)
                tw = (time.perf_counter() - t0) * 1e3
                hw = pool.read()
                if step == 0:
                    bodies.append(ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx))
                log.free()
                if step:
                    t_s.append(ms)
                    t_w.append(tw)
                    t_f.append(fin)
            out["sweep"].append(dict(chunk_bytes=cb, stream_read_ms=round(statistics.median(t_s), 2),
                                     whole_read_ms=round(statistics.median(t_w), 2), finish_ms=round(statistics.median(t_f), 2),
                                     read_high_bytes=hs, whole_read_high_bytes=hw,
                                     parse_gbps=round(n_bytes / statistics.median(t_s) / 1e6, 2), bodies_equal=bodies[0] == bodies[1]))
        ctx.host_free(whole)
    else:
        pool.reset()
        out["chunk_bytes"] = a.chunk_bytes[0]
        log, ms, fin = stream(gen(), a.chunk_bytes[0])
        out.update(read_ms=round(ms, 1), finish_ms=round(fin, 1), parse_gbps=round(n_bytes / ms / 1e6, 2), read_high_bytes=pool.read())
        if not a.no_train:
            stage = "ingest"
            try:
                t0 = time.perf_counter()
                ds, _, _ = ctx.ingest_event_log(log, names, mepu)
                torch.cuda.synchronize()
                out["ingest_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                ctx.free_dataset(ds)
                stage = "calc_all_from_events"
                t0 = time.perf_counter()
                body = ur.calc_all_from_events(log, ap, mepu, now_ms=END_MS, ctx=ctx)
                out["calc_all_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                out["body_bytes"] = len(body)
            except ur.CcoError as e:
                out["failed_stage"] = stage
                out["error"] = str(e)
        log.free()
    name, plimit = gpu_info()
    out.update(gpu=name, power_limit_w=plimit)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
