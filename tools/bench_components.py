"""Cost of the forecast components on config #5 (100k fitted models x 672 15-min periods; DESIGN §12).

    python tools/bench_components.py [--models 100000] [--reps 5]

Four legs, alternated rep by rep after one warm-up call each, timed with CUDA events on the context's stream:
predict alone, predict with the six component planes, 1000-draw intervals alone (predict + mc_kernel), and intervals with
the trend bounds.  The models are fitted config-#3 series tiled up to --models, as bench.py's scorer section does.  Also
checks that the components legs leave yhat and the yhat bounds byte for byte.  Prints one JSON line with the card's
name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402


def _smi():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), (v.strip() for v in r.stdout.splitlines()[0].split(","))))
    except Exception as exc:       # the numbers still stand; say why the card could not be read
        return {"error": repr(exc)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", type=int, default=100_000)
    ap.add_argument("--fit", type=int, default=4096, help="config-#3 series fitted and tiled up to --models")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    ctx = L.Context(0)
    dev = torch.device("cuda", 0)
    H, STEP = 672, 15 * 60 * 10**9
    b = synth.config3(n=a.fit)
    fb = batched.fit_batch_device(ctx, batched.make_options(), torch.from_numpy(b.ds).to(dev),
                                  torch.from_numpy(b.y).to(dev), b.offsets, 0.0, 1.1)
    idx = torch.arange(a.models, device=dev) % fb.n
    sub = batched.FittedBatch(*(x[idx].contiguous() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)),
                              fb.smax, fb.kmax)
    last = torch.from_numpy(b.ds[b.offsets[1:] - 1].copy()).to(dev)[idx]
    fut = (last[:, None] + STEP * torch.arange(1, H + 1, device=dev, dtype=torch.int64)[None, :]).contiguous()
    fl = torch.zeros(a.models, dtype=torch.float64, device=dev)
    cap = sub.meta_f64[:, 2].float().double().contiguous()
    o_det = batched.make_options(uncertainty_samples=0)
    o_mc = batched.make_options(uncertainty_samples=1000)
    legs = {"predict": (o_det, False, False), "predict_components": (o_det, False, True),
            "intervals": (o_mc, True, False), "intervals_trend_bounds": (o_mc, True, True)}
    bufs = {k: batched.predict_batch_device(ctx, o, sub, fut, fl, cap, seed=1, intervals=iv, components=c)
            for k, (o, iv, c) in legs.items()}
    same = (torch.equal(bufs["predict"].yhat, bufs["predict_components"].yhat)
            and torch.equal(bufs["intervals"].yhat_lower, bufs["intervals_trend_bounds"].yhat_lower)
            and torch.equal(bufs["intervals"].yhat_upper, bufs["intervals_trend_bounds"].yhat_upper))
    st = torch.cuda.ExternalStream(ctx.stream, device=dev)
    times = {k: [] for k in legs}
    clock = None
    for r in range(a.reps):
        for k, (o, iv, c) in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            batched.predict_batch_device(ctx, o, sub, fut, fl, cap, seed=1, intervals=iv, components=c, sync=False,
                                         out=bufs[k])
            e1.record(st)
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
            if r == a.reps - 1 and k == "intervals_trend_bounds":
                clock = _smi()
    ms = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    pts = a.models * H
    out = {"workload": f"{a.models} fitted config-#3 models x {H} 15-min periods", "reps": a.reps,
           "median_ms": ms, "min_ms": {k: min(v) for k, v in times.items()},
           "components_extra_ms": ms["predict_components"] - ms["predict"],
           "trend_bounds_extra_ms": ms["intervals_trend_bounds"] - ms["intervals"],
           "component_plane_bytes": pts * 8 * L.N_COMPONENTS,
           "component_planes_at_3_35_TBps_ms": pts * 8 * L.N_COMPONENTS / 3.35e12 * 1e3,
           "yhat_and_bounds_unchanged": bool(same), "gpu": clock}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
