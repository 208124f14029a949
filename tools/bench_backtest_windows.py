"""Backtest window totals on one GPU (DESIGN §14): synth config #3 (50k series x 1440 15-minute points), horizon 2
days, period 12 h, initial 3 days, 1000 draws.  Legs: point forecasts and 1000-draw intervals, each without windows,
with daily ('1D') and with hourly ('1h') windows.  Prints seconds per stage (each stage ends in a synchronisation, so its
wall time is its GPU time) and what the windows add to each leg, then the held-out coverage per horizon of the
daily-total intervals against the nominal width, beside two naive intervals built from the same pointwise bounds:
summed bounds, and independent points (half-width sqrt(sum (hi - lo)^2) / 2 around the sum of the midpoints).  The
card's name, power limit and SM clock are read in the same run.  One JSON line per leg, then one for the coverage.

    python tools/bench_backtest_windows.py [--n 50000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from time_series_spark_b200 import _lib as L, batched, synth  # noqa: E402

H = 3600 * 10**9
D = 24 * H


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # the numbers still mean something without it; say so
        return f"unavailable ({e})"


def naive_coverage(res, W):
    """Per horizon (j + 1) W: (joint-draw, summed-bounds, independent-points) coverage of the window totals, over the
    pairs whose fits all succeeded."""
    w = res.windows
    key = np.stack([res.row_series, res.cutoff, (res.ds - res.cutoff - 1) // W])
    first = np.flatnonzero(np.concatenate(([True], np.any(key[:, 1:] != key[:, :-1], axis=0))))
    assert first.size == w.y.size and np.array_equal(np.diff(np.append(first, res.ds.size)), w.points)
    lo_sum = np.add.reduceat(res.yhat_lower, first)
    hi_sum = np.add.reduceat(res.yhat_upper, first)
    mid = np.add.reduceat((res.yhat_lower + res.yhat_upper) / 2, first)
    half = np.sqrt(np.add.reduceat((res.yhat_upper - res.yhat_lower) ** 2, first)) / 2
    bad = np.zeros(int(res.pair_series.max()) + 1, bool)
    bad[res.pair_series[res.pair_status < 0]] = True
    ok = ~bad[w.series]
    out = {}
    for h in np.unique(w.horizon):
        g = ok & (w.horizon == h)
        y = w.y[g]
        out[f"{h // H}h"] = {"windows": int(g.sum()),
                             "joint_draws": float(np.mean((w.yhat_lower[g] <= y) & (y <= w.yhat_upper[g]))),
                             "summed_bounds": float(np.mean((lo_sum[g] <= y) & (y <= hi_sum[g]))),
                             "independent_points": float(np.mean((mid[g] - half[g] <= y) & (y <= mid[g] + half[g]))),
                             "joint_width_over_summed": float(np.median((w.yhat_upper[g] - w.yhat_lower[g])
                                                                        / (hi_sum[g] - lo_sum[g]))),
                             "joint_width_over_independent": float(np.median((w.yhat_upper[g] - w.yhat_lower[g])
                                                                             / (2 * half[g])))}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50_000)
    args = ap.parse_args()
    b = synth.config3(n=args.n)
    ctx = L.Context(0)
    dev = torch.device("cuda:0")
    ds = torch.from_numpy(b.ds).to(dev)
    y = torch.from_numpy(b.y.astype(np.int32)).to(dev)
    cap = torch.tensor(np.maximum.reduceat(b.y.astype(np.float64), b.offsets[:-1]) * 1.1, dtype=torch.float64, device=dev)
    print("card:", card(), flush=True)
    cov = None
    for intervals in (False, True):
        opts = batched.make_options(uncertainty_samples=1000 if intervals else 0)
        base = None
        for name, W in (("none", None), ("1D", D), ("1h", H)):
            tm = {}
            t0 = time.perf_counter()
            res = batched.cross_validation_device(ctx, opts, ds, y, b.offsets, 0.0, cap, 2 * D, D // 2, 3 * D,
                                                  intervals=intervals, rolling_window=0.1, timings=tm, aggregate_ns=W)
            wall = time.perf_counter() - t0
            line = {"leg": ("intervals" if intervals else "point") + f"/windows={name}", "series": b.n,
                    "fits": int(res.pair_series.size), "held_out_rows": int(res.ds.size),
                    "failed_fits": int((res.pair_status < 0).sum()), "wall_s": round(wall, 3),
                    "stages_s": {k: round(v, 3) for k, v in tm.items()}, "card": card()}
            if W is None:
                base = tm
            else:
                line["window_rows"] = int(res.windows.y.size)
                line["window_metrics_rows"] = int(res.windows.metrics["horizon"].size)
                # what the windows add: the predict stage's growth (the anchored sums with intervals) and the new stages
                line["added_s"] = {"predict": round(tm["predict"] - base["predict"], 3),
                                   "windows": round(tm.get("windows", 0.0), 3),
                                   "window_metrics": round(tm.get("window_metrics", 0.0), 3)}
                if intervals and W == D:
                    cov = naive_coverage(res, W)
            print(json.dumps(line), flush=True)
            del res
    print(json.dumps({"daily_total_coverage_by_horizon": cov, "nominal": 0.8}), flush=True)


if __name__ == "__main__":
    main()
