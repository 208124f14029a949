"""Backtest throughput on one GPU: synth config #3 (50k series x 1440 15-minute points), horizon 1 day, period 12 h,
initial 3 days -- 22 cutoffs per series.  Prints the exact pair / row counts, seconds per stage (plan, gather, fit,
predict, metrics; each stage ends in a synchronisation, so its wall time is its GPU time) and fits/s, without and with
intervals, plus the card's name, power limit and SM clock read in the same run.  One JSON line per leg.

    python tools/bench_backtest.py [--n 50000] [--reps 2]
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

D = 86400 * 10**9


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        return q
    except Exception as e:      # the numbers still mean something without it; say so
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    b = synth.config3(n=args.n)
    ctx = L.Context(0)
    dev = torch.device("cuda:0")
    ds = torch.from_numpy(b.ds).to(dev)
    y = torch.from_numpy(b.y.astype(np.int32)).to(dev)
    cap = torch.tensor(np.maximum.reduceat(b.y.astype(np.float64), b.offsets[:-1]) * 1.1, dtype=torch.float64, device=dev)
    print("card:", card(), flush=True)
    for intervals in (False, True):
        opts = batched.make_options(uncertainty_samples=1000 if intervals else 0)
        for rep in range(args.reps):
            tm = {}
            t0 = time.perf_counter()
            res = batched.cross_validation_device(ctx, opts, ds, y, b.offsets, 0.0, cap, D, D // 2, 3 * D,
                                                  intervals=intervals, rolling_window=0.1, timings=tm)
            wall = time.perf_counter() - t0
        pairs = int(res.pair_series.size)
        po = np.concatenate(([0], np.cumsum(np.bincount(res.pair_series, minlength=b.n))))
        hist_rows = sum(int(np.searchsorted(b.ds[b.offsets[s]:b.offsets[s + 1]], res.pair_cutoff[po[s]:po[s + 1]],
                                            side="right").sum()) for s in range(b.n))
        line = {"leg": "intervals" if intervals else "point", "series": b.n, "fits": pairs,
                "cutoffs_per_series": pairs / b.n, "held_out_rows": int(res.ds.size),
                "history_rows": hist_rows, "mean_history_rows": round(hist_rows / pairs, 1),
                "metrics_rows": int(res.metrics["horizon"].size), "failed_fits": int((res.pair_status < 0).sum()),
                "wall_s": round(wall, 3), "stages_s": {k: round(v, 3) for k, v in tm.items()},
                "fits_per_s": round(pairs / tm.get("fit", float("nan")), 1),
                "fit_points_per_s": round(hist_rows / tm.get("fit", float("nan"))),
                "last_fit_variant_counts": ctx.last_fit_variant_counts().tolist(), "card": card()}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
