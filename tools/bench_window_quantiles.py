"""Cost of the quantiles of window totals (DESIGN §21) next to the totals' call without levels.

    python tools/bench_window_quantiles.py [--models 100000] [--month-models 20000] [--reps 5]

Config #5 (config-#3-fitted models tiled to 100k x 672 15-minute points, 1000 draws), daily totals: Q = 0 (the
pb200_predict_sums_device call as it is), Q = 2 at levels 0.1 / 0.9 (the 80 % interval's percentiles), Q = 9 (deciles)
and Q = 32.  Then 20k models x 8 832 points (92 days), monthly totals (pb200_predict_period_sums_device): Q = 0, 9, 32.
The legs of each workload alternate rep by rep after one warm-up call each, timed with CUDA events on the context's
stream; medians are reported.  A timed call is the whole batched.* call (its output allocations from torch's caching
allocator, and the copy of each frame's first and last point that sizes the slots).  Checks at full size that every
output of the Q = 32 calls other than the planes is the Q = 0 call's, bit for bit.  Prints one JSON line with the card's
name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from bench_aggregate import _smi  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402

STEP, DAY = 15 * 60 * 10**9, 86400 * 10**9
LEVELS = {0: None, 2: [0.1, 0.9], 9: [0.1 * k for k in range(1, 10)], 32: [k / 31 for k in range(32)]}


def _same(x, y):
    """Bit for bit, NaN (an empty slot) equal to NaN."""
    if not x.is_floating_point():
        return torch.equal(x, y)
    return bool(torch.equal(x.view(torch.int64), y.view(torch.int64)))


def _models(ctx, fb, b, n, H, dev):
    idx = torch.arange(n, device=dev) % fb.n
    sub = batched.FittedBatch(*(x[idx].contiguous() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)),
                              fb.smax, fb.kmax)
    last = torch.from_numpy(b.ds[b.offsets[1:] - 1].copy()).to(dev)[idx]
    fut = (last[:, None] + STEP * torch.arange(1, H + 1, device=dev, dtype=torch.int64)[None, :]).contiguous()
    return sub, fut, torch.zeros(n, dtype=torch.float64, device=dev), sub.meta_f64[:, 2].float().double().contiguous()


def _measure(ctx, legs, reps, dev):
    """Warm up every leg, check the Q = 32 leg's other outputs against Q = 0, then time the legs alternately."""
    first = {k: f() for k, f in legs.items()}
    ctx.synchronize()
    (f0, w0), (f32, w32) = first["q0"], first["q32"]
    same = all(_same(getattr(w0, f.name), getattr(w32, f.name)) for f in batched.fields(batched.WindowSums))
    same &= _same(f0.yhat, f32.yhat) and _same(f0.yhat_int, f32.yhat_int)
    windows = [int(w0.n_windows.min()), int(w0.n_windows.max())]
    del first, f0, w0, f32, w32
    torch.cuda.empty_cache()
    st = torch.cuda.ExternalStream(ctx.stream, device=dev)
    times = {k: [] for k in legs}
    for _ in range(reps):
        for k, f in legs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            res = f()
            e1.record(st)
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1))
            del res
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    return {"median_ms": med, "min_ms": {k: min(v) for k, v in times.items()},
            "max_ms": {k: max(v) for k, v in times.items()},
            "added_over_q0_pct": {k: 100.0 * (v / med["q0"] - 1.0) for k, v in med.items() if k != "q0"},
            "windows_per_model": windows, "other_outputs_equal_q0": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", type=int, default=100_000)
    ap.add_argument("--month-models", type=int, default=20_000)
    ap.add_argument("--fit", type=int, default=4096, help="config-#3 series fitted and tiled up to the model counts")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    ctx = L.Context(0)
    dev = torch.device("cuda", 0)
    b = synth.config3(n=a.fit)
    fb = batched.fit_batch_device(ctx, batched.make_options(), torch.from_numpy(b.ds).to(dev),
                                  torch.from_numpy(b.y).to(dev), b.offsets, 0.0, 1.1)
    opts = batched.make_options(uncertainty_samples=1000)
    out = {}
    sub, fut, fl, cap = _models(ctx, fb, b, a.models, 672, dev)
    daily = {f"q{q}": (lambda lv=lv: batched.predict_sums_device(ctx, opts, sub, fut, fl, cap, DAY, 0, seed=1, levels=lv))
             for q, lv in LEVELS.items()}
    out["daily_config5"] = _measure(ctx, daily, a.reps, dev)
    del sub, fut, fl, cap, daily
    torch.cuda.empty_cache()
    sub, fut, fl, cap = _models(ctx, fb, b, a.month_models, 8832, dev)
    monthly = {f"q{q}": (lambda lv=lv: batched.predict_period_sums_device(ctx, opts, sub, fut, fl, cap, 1, 0, seed=1,
                                                                          levels=lv))
               for q, lv in LEVELS.items() if q != 2}
    out["monthly_8832"] = _measure(ctx, monthly, a.reps, dev)
    out["gpu"] = _smi()
    out["workload"] = (f"daily totals: {a.models} config-#3-fitted models x 672 15-min points; monthly totals: "
                       f"{a.month_models} x 8832; 1000 draws; reps {a.reps}")
    print(json.dumps(out))
    if not all(v["other_outputs_equal_q0"] for k, v in out.items() if isinstance(v, dict) and "median_ms" in v):
        raise SystemExit("the calls with levels changed an output of the call without them")


if __name__ == "__main__":
    main()
