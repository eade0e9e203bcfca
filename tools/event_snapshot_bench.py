"""Cost of restarting a trainer from a snapshot of its resident event log (EventLog.save, CcoContext.load_events) against
reading its export again.

The export is event_extend_bench.py's (export_days), held in pinned host memory, so that the re-read is the read alone,
without storage; the log is read as a trainer keeps it: extendable, interned ids, a 30-day window with removeDuplicates
at now = END_MS.  The card's name and power limit are read first.  Each round, alternated (one warm-up round first):
  save          EventLog.save to a temporary file (every byte written and the file closed);
  load_file     CcoContext.load_events of that file, in page cache after the save;
  load_pinned   CcoContext.load_events of the image held in pinned host memory (one append);
  reread        CcoContext.read_events of the export (pinned memory) under the same window and flags.
Every loaded log must report the info, window stats, intern stats and resident bytes of the read one.  Prints one JSON
line: medians of each stage, the snapshot's size, the log's resident bytes and the export's size.
The snapshot file goes to --dir (a temporary directory by default).
usage: python tools/event_snapshot_bench.py --config C2 --steps 5
       python tools/event_snapshot_bench.py --config C3 --steps 3
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import synth  # noqa: E402
import universal_recommender_b200 as ur  # noqa: E402
from event_extend_bench import export_days  # noqa: E402
from events_bench import END_MS  # noqa: E402
from ingest_strings_bench import gpu_info  # noqa: E402

STAGES = ("save", "load_file", "load_pinned", "reread")


def same(a, b) -> bool:
    return (a.info(), a.window_stats(), a.intern_stats(), a.resident_bytes()) == (b.info(), b.window_stats(), b.intern_stats(),
                                                                                   b.resident_bytes())


def main():
    ap_ = argparse.ArgumentParser()
    ap_.add_argument("--config", default="C2")
    ap_.add_argument("--fraction", type=float, default=1.0)
    ap_.add_argument("--chunk-bytes", type=int, default=256 << 20)
    ap_.add_argument("--steps", type=int, default=3)
    ap_.add_argument("--dir", default=None)
    a = ap_.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("event_snapshot_bench measures on the GPU: no CUDA device")
    name, plimit = gpu_info()
    cfg = synth.CONFIGS[a.config]
    ctx = ur.CcoContext(device=0)
    torch.cuda.init()
    window = ur.EventWindow("30 days", True)
    flags = dict(extendable=True, intern_ids=True)
    with tempfile.TemporaryDirectory(dir=a.dir) as tmp:
        snap = os.path.join(tmp, "log.snap")
        whole, _, n_lines = export_days(cfg, a.fraction, ctx.host_array)
        out = {"config": a.config, "fraction": a.fraction, "export_bytes": len(whole), "n_lines": n_lines, "chunk_bytes": a.chunk_bytes,
               "remove_duplicates": True, "gpu": name, "power_limit_w": plimit}
        t = {s: [] for s in STAGES}

        def timed(stage, step, f):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = f()
            torch.cuda.synchronize()
            if step:
                t[stage].append((time.perf_counter() - t0) * 1e3)
            return r

        log = ctx.read_events(whole, chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS, **flags)
        out["resident_bytes"] = log.resident_bytes()
        for step in range(a.steps + 1):
            size = timed("save", step, lambda: log.save(snap, chunk_bytes=a.chunk_bytes))
            back = timed("load_file", step, lambda: ctx.load_events(snap, chunk_bytes=a.chunk_bytes))
            assert same(back, log), "the loaded log differs"
            back.free()
            pinned = ctx.host_array(size, "uint8")
            with open(snap, "rb", buffering=0) as f:
                got = 0
                while got < size:
                    got += f.readinto(memoryview(pinned)[got:])
            back = timed("load_pinned", step, lambda: ctx.load_events(pinned))
            assert same(back, log), "the loaded log differs"
            back.free()
            ctx.host_free(pinned)
            again = timed("reread", step, lambda: ctx.read_events(whole, chunk_bytes=a.chunk_bytes, window=window, now_ms=END_MS, **flags))
            assert same(again, log), "the re-read differs"
            again.free()
        out["snapshot_bytes"] = size
        log.free()
        ctx.host_free(whole)
    for s, v in t.items():
        out[f"{s}_ms"] = round(statistics.median(v), 2)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
