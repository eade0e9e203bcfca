"""Cost of writing a resident log's cleaned events back as a compacted export (EventLog.write_clean) against reading the
export it comes from.

The export is event_extend_bench.py's (event_stream_bench.py's line templates and generators) with eventTimes uniform
over the 31 days before END_MS and the items' $set lines at END_MS.  The window keeps 27 of the 30 days before END_MS, with
removeDuplicates.  Over --steps rounds (one warm-up round first):
  (a) read: read_events of the export from pinned memory as an extendable log, to a finished log;
  (b) write-back: write_clean of that log from the same bytes into a sink that counts what it is handed.
The first round checks the output against the kept line count and the window's stats.  Prints one JSON line: export_bytes,
n_lines, clean_bytes, n_written, read_ms and clean_ms (medians), clean_gb_s (export bytes over clean_ms), the device
memory in use before the clean and the most seen in use at any append return of the clean (torch.cuda.mem_get_info,
sampled), and the GPU's name and power limit, read in the same run.
usage: python tools/event_clean_bench.py --config C2 --steps 5
       python tools/event_clean_bench.py --config C3 --steps 3
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

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from event_extend_bench import export_days  # noqa: E402
from events_bench import END_MS  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402


class Sink:
    """a binary file object that keeps the byte count and samples the device memory in use"""

    def __init__(self, torch):
        self.n, self.peak, self.torch = 0, 0, torch

    def write(self, b) -> int:
        free, total = self.torch.cuda.mem_get_info()
        self.peak = max(self.peak, total - free)
        self.n += len(b)
        return len(b)


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, default=256 << 20)
    ap_.add_argument("--steps", type=int, default=3)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_clean_bench measures on the GPU: no CUDA device")
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    whole, _, n_lines = export_days(cfg, a.fraction, ctx.host_array)
    window = ur.EventWindow("27 days", True)
    out = {"config": a.config, "fraction": a.fraction, "export_bytes": len(whole), "n_lines": n_lines, "chunk_bytes": a.chunk_bytes,
           "window": "27 days, removeDuplicates"}
    t = {"read": [], "clean": []}
    for step in range(a.steps + 1):   # alternated; the first round warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        log = ctx.read_events(whole, chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS, extendable=True)
        tr = (time.perf_counter() - t0) * 1e3
        sink = Sink(torch)
        free, total = torch.cuda.mem_get_info()
        before = total - free
        t0 = time.perf_counter()
        st = log.write_clean(whole, sink, chunk_bytes=a.chunk_bytes)
        tc = (time.perf_counter() - t0) * 1e3
        if step == 0:
            x, d = log.window_stats()
            assert (st.n_lines, st.n_expired, st.n_duplicates) == (n_lines, x, d)
            assert st.n_written == n_lines - x - d and st.n_bytes == sink.n
            out.update(clean_bytes=sink.n, n_written=st.n_written, n_expired=x, n_duplicates=d,
                       device_bytes_before_clean=before, device_bytes_peak_sampled=sink.peak)
        log.free()
        if step:
            t["read"].append(tr)
            t["clean"].append(tc)
    for k, v in t.items():
        out[f"{k}_ms"] = round(statistics.median(v), 2)
    out["clean_gb_s"] = round(len(whole) / out["clean_ms"] / 1e6, 2)
    ctx.host_free(whole)
    name, plimit = gpu_info()
    out.update(gpu=name, power_limit_w=plimit)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
