"""Tuning throughput on one GPU: synth config #3 (``--n`` series x 1440 15-minute points), a 4 x 4 grid of prior scales
(fbprophet's documented changepoint_prior_scale x seasonality_prior_scale), horizon 1 day, period 12 h, initial 3 days --
22 cutoffs per series, 16 cutoff fits per cutoff.  Two legs in one run:

  (a) batched.tune_device: every grid point's cutoff fits in the same fit calls, then the final fit;
  (b) the loop a user writes without it: 16 cross_validation_device calls, one per grid point, uniform options.

Prints one JSON line per leg (seconds per stage -- each stage ends in a synchronisation, so its wall time is its GPU
time -- fits/s and history points/s of the cutoff fits) and one with the largest score difference between the legs,
plus the card's name, power limit and SM clock read in the same run.

    python tools/bench_tune.py [--n 5000]
"""
import argparse
import itertools
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

D = 86400 * 10**9
CP = (0.001, 0.01, 0.1, 0.5)
SP = (0.01, 0.1, 1.0, 10.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=5000)
    args = ap.parse_args()
    grid = list(itertools.product(CP, SP))
    b = synth.config3(n=args.n)
    ctx = L.Context(0)
    dev = torch.device("cuda:0")
    ds = torch.from_numpy(b.ds).to(dev)
    y = torch.from_numpy(b.y.astype(np.int32)).to(dev)
    cap = torch.tensor(np.maximum.reduceat(b.y.astype(np.float64), b.offsets[:-1]) * 1.1, dtype=torch.float64, device=dev)
    opts = batched.make_options(uncertainty_samples=0)
    print("card:", card(), flush=True)
    # warm-up: module loads and the first launch of every kernel either leg uses
    w = b.take(0, 64)
    batched.tune_device(ctx, opts, ds[:int(w.offsets[-1])], y[:int(w.offsets[-1])], w.offsets, 0.0, 1.1, D, D // 2, 3 * D,
                        grid[:2])
    torch.cuda.synchronize()

    plan = batched.cv_plan_device(ctx, opts, ds, b.offsets, D, D // 2, 3 * D)
    ps = np.repeat(np.arange(b.n), plan.n_cutoffs)
    hist_rows = int((plan.hist_end.cpu().numpy() - b.offsets[:-1][ps]).sum())
    fits, points = plan.n_pairs * len(grid), hist_rows * len(grid)

    def report(leg, tm, wall):
        line = {"leg": leg, "series": b.n, "grid_points": len(grid), "cutoff_fits": fits, "history_points": points,
                "wall_s": round(wall, 3), "stages_s": {k: round(v, 3) for k, v in tm.items()},
                "fits_per_s": round(fits / tm["fit"], 1), "fit_points_per_s": round(points / tm["fit"]),
                "cv_fits_per_s_wall": round(fits / (wall - tm.get("final_fit", 0.0)), 1), "card": card()}
        print(json.dumps(line), flush=True)

    tm_a = {}
    t0 = time.perf_counter()
    tuned = batched.tune_device(ctx, opts, ds, y, b.offsets, 0.0, 1.1, D, D // 2, 3 * D, grid, timings=tm_a)
    report("a_tune_device", tm_a, time.perf_counter() - t0)

    tm_b = {}
    scores_b = np.full((b.n, len(grid)), np.nan)
    t0 = time.perf_counter()
    for j, (cp, sp) in enumerate(grid):
        o = batched.make_options(uncertainty_samples=0, changepoint_prior_scale=cp, seasonality_prior_scale=sp)
        res = batched.cross_validation_device(ctx, o, ds, y, b.offsets, 0.0, cap, D, D // 2, 3 * D, rolling_window=1.0,
                                              timings=tm_b)
        scores_b[res.metrics["series"], j] = res.metrics["rmse"]
    report("b_python_loop", tm_b, time.perf_counter() - t0)
    d = np.abs(tuned.scores - scores_b)
    rel = d / np.maximum(np.abs(scores_b), 1e-300)
    print(json.dumps({"max_abs_score_diff": float(np.nanmax(d)), "max_rel_score_diff": float(np.nanmax(rel)),
                      "bit_equal_scores": int(np.sum(tuned.scores.view(np.int64) == scores_b.view(np.int64))),
                      "scores": int(scores_b.size), "chosen_histogram": np.bincount(tuned.chosen + 1, minlength=len(grid) + 1).tolist(),
                      "final_fit_failed": int((tuned.fitted.meta_i32[:, 4] < 0).sum().item())}), flush=True)


if __name__ == "__main__":
    main()
