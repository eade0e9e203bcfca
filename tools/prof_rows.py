"""Development: the shortest command that runs the resident hot path a few times (what a profiler wraps).
usage: python tools/prof_rows.py [workload=C3] [trains=2] [--bins OUT.json]

--bins: the last train runs under torch.profiler (CUDA activities).  For every indicator it reports, per row-kernel bin,
the start and end of its k_rows launch relative to the start of the indicator's bracket, the CTAs per SM the launch
got (from its grid: 4 waves over the SMs), and which bin ends the bracket.  Bins that share one k_rows instance are told
apart by launch order: an indicator launches its bins in order 0, 1, ..."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import synth
import universal_recommender_b200 as ur
from universal_recommender_b200 import _native as N

args = [a for a in sys.argv[1:] if not a.startswith("--")]
bins_out = sys.argv[sys.argv.index("--bins") + 1] if "--bins" in sys.argv else None
if bins_out in args:
    args.remove(bins_out)
ctx = ur.CcoContext()
w = synth.make(args[0] if args else "C3", ctx=ctx)
ds = ctx.upload(w.mats, ur.FLAG_ASSUME_CANONICAL)
trains = int(args[1]) if len(args) > 1 else 2


def train(it):
    ctx.train_dataset(ds, w.params, 42, ur.FLAG_ASSUME_CANONICAL | N.FLAG_RESULT_ON_DEVICE, copy_arrays=False)
    st = ctx.last_stats
    print(f"train {it}: prep {st.ms_prepare:.2f} indicators {st.ms_cooccurrence:.2f} rows {[round(x, 3) for x in st.ms_indicator]} "
          f"evaluated {st.llr_evaluated} distinct {st.distinct_cells} products {st.products}", flush=True)


for it in range(trains - (1 if bins_out else 0)):
    train(it)
if bins_out:
    import torch
    from torch.profiler import ProfilerActivity, profile
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        train(trains - 1)
        torch.cuda.synchronize()
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        prof.export_chrome_trace(os.path.join(td, "trace.json"))
        with open(os.path.join(td, "trace.json")) as f:
            trace = json.load(f)
    kern = [e for e in trace["traceEvents"] if e.get("cat") == "kernel" and "k_rows<" in e.get("name", "")]
    kern.sort(key=lambda e: e["args"]["correlation"])   # launch order
    n_bins = len(kern) // w.n_types
    assert n_bins * w.n_types == len(kern), f"{len(kern)} k_rows launches for {w.n_types} indicators"
    report = {"gpu": torch.cuda.get_device_name(0), "sms": sms, "indicators": []}
    for i in range(w.n_types):
        ks = kern[i * n_bins:(i + 1) * n_bins]
        t0 = min(e["ts"] for e in ks)
        t1 = max(e["ts"] + e["dur"] for e in ks)
        bins = []
        for b, e in enumerate(ks):
            inst = e["name"][e["name"].index("k_rows<") + 7:e["name"].index(">")]
            bins.append({"bin": b, "k_rows": inst, "ctas_per_sm": e["args"]["grid"][0] // (4 * sms),
                         "start_us": round(e["ts"] - t0, 1), "end_us": round(e["ts"] + e["dur"] - t0, 1), "dur_us": round(e["dur"], 1)})
        last = max(bins, key=lambda x: x["end_us"])
        report["indicators"].append({"indicator": i, "bracket_us": round(t1 - t0, 1), "ends_bracket": last["bin"], "bins": bins})
        print(f"indicator {i}: bracket {t1 - t0:.0f} us, ended by bin {last['bin']} (k_rows<{last['k_rows']}>)")
        for x in bins:
            print(f"  bin {x['bin']} k_rows<{x['k_rows']}> {x['ctas_per_sm']:2d} CTAs/SM: "
                  f"{x['start_us']:8.1f} .. {x['end_us']:8.1f} us ({x['dur_us']:.1f})")
    with open(bins_out, "w") as f:
        json.dump(report, f, indent=1)
