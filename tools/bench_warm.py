"""What warm starts buy a scheduled refit, on one GPU (DESIGN §11).  synth config #3 with 1536 15-minute points per
series: the first 1440 (the headline problem: span 14 d 23:45, weekly + daily, S = 25) are fitted cold and their
records kept; then all 1536 (one appended day) are refitted cold and warm from those records, alternated, ``--reps``
times each.

Per leg it prints one JSON line: ms per fit call and series/s, evaluations per series (mean, p50, p99, max) and
iterations, the status histogram and the warm reason counts; then one line comparing the last warm and cold fits:
warm - cold objective relative to |cold| (median, max) and the 672-period forecast difference over y_scale (median,
max).  The card's name, power limit and SM clock are read in the same run.

    python tools/bench_warm.py [--n 50000] [--reps 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_backtest import card  # noqa: E402
from time_series_spark_b200 import _lib as L, batched, synth  # noqa: E402

T_OLD, T_NEW, HORIZON, STEP = 1440, 1536, 672, 15 * 60 * 10**9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    b = synth.config3(n=args.n, T=T_NEW)
    keep = (np.arange(b.offsets[-1]) - np.repeat(b.offsets[:-1], np.diff(b.offsets))) < T_OLD
    old_off = np.concatenate(([0], np.cumsum(np.minimum(np.diff(b.offsets), T_OLD)))).astype(np.int64)
    ctx = L.Context(0)
    dev = torch.device("cuda:0")
    opts = batched.make_options(uncertainty_samples=0)
    y_new = torch.from_numpy(b.y.astype(np.int32)).to(dev)
    ds_new = torch.from_numpy(b.ds).to(dev)
    ds_old, y_old = ds_new[torch.from_numpy(keep).to(dev)].contiguous(), y_new[torch.from_numpy(keep).to(dev)].contiguous()
    print("card:", card(), flush=True)

    def fit(ds, y, off, init=None):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f = batched.fit_batch_device(ctx, opts, ds, y, off, 0.0, 1.1, init=init)      # ends in a synchronisation
        return f.to_host(), time.perf_counter() - t0

    old, t_old = fit(ds_old, y_old, old_off)      # also the warm-up of every kernel the legs use
    init = batched.FittedBatch(old.params, old.tchange, old.meta_i32, old.meta_i64, old.meta_f64, old.smax, old.kmax)
    fit(ds_new, y_new, b.offsets, init)
    print(json.dumps({"leg": "records", "series": b.n, "points": T_OLD, "ms": round(1e3 * t_old, 1),
                      "status": dict(zip(*map(lambda a: a.tolist(), np.unique(old.status, return_counts=True))))}), flush=True)
    last = {}
    times = {"cold": [], "warm": []}
    for rep in range(args.reps):
        for leg in ("cold", "warm"):
            f, t = fit(ds_new, y_new, b.offsets, init if leg == "warm" else None)
            times[leg].append(t)
            last[leg] = f
    for leg in ("cold", "warm"):
        f = last[leg]
        ev, it = f.meta_i32[:, 6].astype(np.float64), f.meta_i32[:, 5]
        line = {"leg": leg, "series": b.n, "points": T_NEW, "ms_per_fit": [round(1e3 * t, 1) for t in times[leg]],
                "series_per_s": round(b.n / min(times[leg])), "evals_mean": round(float(ev.mean()), 1),
                "evals_p50": float(np.percentile(ev, 50)), "evals_p99": float(np.percentile(ev, 99)),
                "evals_max": int(ev.max()), "iters_mean": round(float(it.mean()), 1),
                "status": {int(k): int(c) for k, c in zip(*np.unique(f.status, return_counts=True))}}
        if f.warm is not None:
            line["warm"] = {int(k): int(c) for k, c in zip(*np.unique(f.warm, return_counts=True))}
        print(json.dumps(line), flush=True)
    c, w = last["cold"], last["warm"]
    ok = (c.status >= 0) & (w.status >= 0)
    fc, fw = c.meta_f64[ok, 3], w.meta_f64[ok, 3]
    rel = (fw - fc) / np.maximum(np.abs(fc), 1e-300)
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], HORIZON, STEP)
    fl, cap = c.meta_f64[:, 1].copy(), c.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    pc = batched.predict_batch_host(ctx, opts, c, fut, fl, cap, intervals=False)
    pw = batched.predict_batch_host(ctx, opts, w, fut, fl, cap, intervals=False)
    dy = (np.abs(pw.yhat - pc.yhat).max(axis=1) / c.meta_f64[:, 0])[ok]
    print(json.dumps({"both_fitted": int(ok.sum()), "warm_minus_cold_rel_median": float(np.median(rel)),
                      "warm_minus_cold_rel_max": float(rel.max()), "warm_minus_cold_rel_min": float(rel.min()),
                      "warm_lower_share": float(np.mean(rel < 0)),
                      "forecast_diff_over_y_scale_median": float(np.median(dy)),
                      "forecast_diff_over_y_scale_max": float(dy.max()), "card": card()}), flush=True)


if __name__ == "__main__":
    main()
