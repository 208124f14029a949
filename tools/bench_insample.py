"""Cost of the in-sample predict, its outlier flags and the refit without them (DESIGN §16) on config #3 (50k x 1440
15-min points) and config #4 (500k ragged series, T_i ~ U{48..96}).

    python tools/bench_insample.py [--c3 50000] [--c4 500000] [--reps 3] [--width 0.99]

Per workload: the fit (once), then -- alternated rep by rep after one warm-up call each -- (1) the ragged in-sample
predict without bounds; (2) the same with 1000-draw bounds; (3) the padded alternative, pb200_predict_device on
[n, Tmax] frames that repeat each history's last timestamp, without and (4) with bounds; (5) flags and compaction;
then the refit (once).  Each leg's time is a host clock around calls that end in a device synchronise; the median of
the reps is reported.  Checks at full size that the ragged rows are the padded frames' rows byte for byte.  Prints one
JSON line per workload with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_aggregate import _smi  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402


def _timed(ctx, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    ctx.synchronize()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run(ctx, name, b, reps, width):
    dev = torch.device("cuda", 0)
    opts = batched.make_options(uncertainty_samples=1000, interval_width=width)
    ds = torch.from_numpy(b.ds).to(dev)
    y = torch.from_numpy(b.y).to(dev)
    off = b.offsets
    T = np.diff(off)
    t_fit, fitted = _timed(ctx, lambda: batched.fit_batch_device(ctx, opts, ds, y, off, 0.0, 1.1))
    fl = fitted.meta_f64[:, 1].contiguous()
    cp = fitted.meta_f64[:, 2].contiguous()
    # the padded frames: row i is history i, then its last timestamp repeated up to the longest history
    tmax = int(T.max())
    d_off = torch.from_numpy(off).to(dev)
    d_T = torch.from_numpy(T).to(dev)
    j = torch.arange(tmax, device=dev)[None, :]
    idx = d_off[:-1, None] + torch.minimum(j, d_T[:, None] - 1)
    fut = ds[idx].contiguous()
    valid = (j < d_T[:, None])
    legs = {
        "history": lambda: batched.predict_history_device(ctx, opts, fitted, ds, off, fl, cp, seed=1, intervals=False),
        "history_bounds": lambda: batched.predict_history_device(ctx, opts, fitted, ds, off, fl, cp, seed=1),
        "padded": lambda: batched.predict_batch_device(ctx, opts, fitted, fut, fl, cp, seed=1, intervals=False),
        "padded_bounds": lambda: batched.predict_batch_device(ctx, opts, fitted, fut, fl, cp, seed=1),
    }
    times = {k: [] for k in legs}
    times["flags_compact"] = []
    outs = {k: fn() for k, fn in legs.items()}            # warm-up
    hb = outs["history_bounds"]
    ol = batched.outliers_device(ctx, ds, y, off, hb.yhat_lower, hb.yhat_upper)
    for _ in range(reps):
        for k, fn in legs.items():
            t, outs[k] = _timed(ctx, fn)
            times[k].append(t)
        t, ol = _timed(ctx, lambda: batched.outliers_device(ctx, ds, y, off, hb.yhat_lower, hb.yhat_upper))
        times["flags_compact"].append(t)
    hb, pb = outs["history_bounds"], outs["padded_bounds"]
    same = all(torch.equal(getattr(hb, f).view(torch.int64), getattr(pb, f)[valid].view(torch.int64))
               for f in ("yhat", "yhat_lower", "yhat_upper"))
    short = int(np.count_nonzero(np.diff(ol.offsets) < 2))
    t_refit = None
    if short == 0:
        t_refit, _ = _timed(ctx, lambda: batched.fit_batch_device(ctx, opts, ol.ds, ol.y, ol.offsets, 0.0, 1.1))
    med = {k: float(np.median(v)) * 1e3 for k, v in times.items()}
    return {"workload": name, "series": int(b.n), "rows": int(off[-1]), "tmax": tmax, "padded_rows": int(b.n * tmax),
            "fit_ms": t_fit * 1e3, **{f"{k}_ms": round(v, 2) for k, v in med.items()},
            "refit_ms": None if t_refit is None else t_refit * 1e3, "rows_flagged": int(off[-1] - ol.offsets[-1]),
            "series_flagged": int(np.count_nonzero(ol.kept < T)), "series_short_after_filter": short,
            "ragged_equals_padded_bytes": bool(same), "width": width, "samples": 1000, "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c3", type=int, default=50_000)
    ap.add_argument("--c4", type=int, default=500_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--width", type=float, default=0.99)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    ctx = L.Context(0)
    card = _smi()
    for name, n, make in (("config3", a.c3, synth.config3), ("config4", a.c4, synth.config4)):
        if n <= 0:
            continue
        r = run(ctx, name, make(n=n), a.reps, a.width)
        print(json.dumps({**r, "card": card}), flush=True)


if __name__ == "__main__":
    main()
