"""Cost of extra regressors (DESIGN §19) against the default model, on bench.py's workload.

    python tools/bench_regressors.py [--n 50000] [--reps 3] [--predict-n 100000]

Fit stage, config #3 (50k series x 1440 15-minute points, logistic, multiplicative), four legs alternated rep by rep
after one warm-up call each, each a batched.fit_batch_device call timed with CUDA events on the context's stream:
  (a) default    the default model on the grouped kernels;
  (b) as_table   the same model written as a table: weekly2 (7, 3) and daily2 (1, 4), built-ins off
                 (bench_seasonalities.py's leg (b));
  (c) promo      (b) plus one binary promotion flag (20 % of the points on; not standardised);
  (d) four       (b) plus four continuous regressors (standard normal values; standardised).
Per leg: series/s from the median time, the median and maximum evaluations (meta_i32[:, 6]) and the table count
(pb200_last_fit_table_count).  Then predict and 1000-draw intervals at 100k models x 672 15-minute points (one week),
default against (b) plus two regressors (the flag and one continuous), each with its own leg's fits tiled.  Prints one
JSON line with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_aggregate import _smi  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402

OFF = dict(yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False)
TABLE = [dict(name="weekly2", period=7, fourier_order=3), dict(name="daily2", period=1, fourier_order=4)]
CONT = [dict(name=f"x{i}") for i in range(4)]
LEGS = {
    "default": (lambda: batched.make_options(), 0),
    "as_table": (lambda: batched.make_table_options(seasonalities=TABLE, **OFF), 0),
    "promo": (lambda: batched.make_regressor_options([dict(name="promo")], seasonalities=TABLE, **OFF), 1),
    "four": (lambda: batched.make_regressor_options(CONT, seasonalities=TABLE, **OFF), 4),
    "two": (lambda: batched.make_regressor_options([dict(name="promo"), CONT[0]], seasonalities=TABLE, **OFF), 2),
}
FIT_LEGS = ("default", "as_table", "promo", "four")


def _values(kind, R, rows, dev, seed):
    """[R, rows] float64 on the device: the promotion flag first when kind has one, then standard normal values."""
    g = torch.Generator(device=dev).manual_seed(seed)
    out = torch.randn((R, rows), generator=g, device=dev, dtype=torch.float64)
    if kind in ("promo", "two"):
        out[0] = (torch.rand(rows, generator=g, device=dev) < 0.2).double()
    return out.contiguous()


def _table_count(ctx) -> int:
    n = np.zeros(1, np.int64)
    L.check(L.load().pb200_last_fit_table_count(ctx.handle, n.ctypes.data_as(C.c_void_p)), "pb200_last_fit_table_count")
    return int(n[0])


def _timed(st, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    out = fn()
    e1.record(st)
    e1.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50_000, help="config-#3 series fitted per leg")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--predict-n", type=int, default=100_000, help="models of the predict legs")
    ap.add_argument("--horizon", type=int, default=672, help="15-minute points of the predict legs")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark only runs on the GPU")
    ctx = L.Context(0)
    dev = torch.device("cuda", 0)
    st = torch.cuda.ExternalStream(ctx.stream, device=dev)
    b = synth.config3(n=a.n)
    ds, y = torch.from_numpy(b.ds).to(dev), torch.from_numpy(b.y).to(dev)
    opts = {k: f() for k, (f, _) in LEGS.items()}
    regs = {k: _values(k, R, b.ds.size, dev, 1) if R else None for k, (_, R) in LEGS.items()}

    def fit(k):
        return batched.fit_batch_device(ctx, opts[k], ds, y, b.offsets, 0.0, 1.1, regressors=regs[k])

    fits, counts = {}, {}
    for k in FIT_LEGS:                               # warm-up: module load, shared-memory attributes, allocator
        fits[k] = fit(k).to_host()
        counts[k] = _table_count(ctx)
    times = {k: [] for k in FIT_LEGS}
    clock = None
    for r in range(a.reps):
        for k in FIT_LEGS:
            ms, _ = _timed(st, lambda: fit(k))
            times[k].append(ms)
            if r == a.reps - 1 and k == "as_table":
                clock = _smi()
    fit_res = {}
    for k in FIT_LEGS:
        med = sorted(times[k])[len(times[k]) // 2]
        ev = fits[k].meta_i32[:, 6]
        ok = fits[k].meta_i32[:, 4] >= 0
        fit_res[k] = {"median_ms": med, "min_ms": min(times[k]), "max_ms": max(times[k]),
                      "series_per_s": a.n / (med / 1e3), "evals_median": float(np.median(ev[ok])),
                      "evals_max": int(ev[ok].max()), "table_count": counts[k], "failed": int((~ok).sum()),
                      "status_codes": sorted(int(s) for s in np.unique(fits[k].meta_i32[:, 4]))}
    del fits
    torch.cuda.empty_cache()

    # predict legs: the default and the two-regressor fits tiled to predict-n models, one week of 15-minute points
    STEP = 15 * 60 * 10**9
    PL = ("default", "two")
    pred = {}
    for k in PL:
        fb = fit(k)
        idx = torch.arange(a.predict_n, device=dev) % fb.n
        pred[k] = batched.FittedBatch(*(x[idx].contiguous() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64,
                                                                      fb.meta_f64)), fb.smax, fb.kmax,
                                      reg_scale=None if fb.reg_scale is None else fb.reg_scale[idx].contiguous())
    fregs = {"default": None, "two": _values("two", 2, a.predict_n * a.horizon, dev, 2)}
    last = torch.from_numpy(b.ds[b.offsets[1:] - 1].copy()).to(dev)[torch.arange(a.predict_n, device=dev) % b.n]
    fut = (last[:, None] + STEP * torch.arange(1, a.horizon + 1, device=dev, dtype=torch.int64)[None, :]).contiguous()
    fl = torch.zeros(a.predict_n, dtype=torch.float64, device=dev)
    cap = pred["default"].meta_f64[:, 2].float().double().contiguous()
    mc = {k: batched.copy_options(opts[k]) for k in PL}
    det = {k: batched.copy_options(opts[k]) for k in PL}
    for k in mc:
        mc[k].uncertainty_samples = 1000
        det[k].uncertainty_samples = 0

    def run(leg):
        k, kind = leg
        o = mc[k] if kind == "intervals" else det[k]
        return batched.predict_batch_device(ctx, o, pred[k], fut, fl, cap, seed=1, intervals=kind == "intervals",
                                            regressors=fregs[k])

    plegs = [(k, kind) for kind in ("predict", "intervals") for k in PL]
    outs = {leg: run(leg) for leg in plegs}                 # warm-up
    ctx.synchronize()
    finite = {f"{k}_{kind}": bool(torch.isfinite(outs[(k, kind)].yhat).all()) for k, kind in plegs}
    del outs
    ptimes = {leg: [] for leg in plegs}
    for r in range(a.reps):
        for leg in plegs:
            ms, res = _timed(st, lambda: run(leg))
            ptimes[leg].append(ms)
            del res
    pred_res = {f"{k}_{kind}": {"median_ms": sorted(v)[len(v) // 2], "min_ms": min(v), "max_ms": max(v)}
                for (k, kind), v in ptimes.items()}
    res = {"workload": f"fit: config #3, {a.n} series x 1440 15-min points; predict: {a.predict_n} models x "
                       f"{a.horizon} 15-min points, intervals 1000 draws", "reps": a.reps, "fit": fit_res,
           "predict": pred_res, "predict_yhat_finite": finite,
           "fit_slowdown_vs_default": {k: fit_res[k]["median_ms"] / fit_res["default"]["median_ms"] for k in FIT_LEGS},
           "gpu": clock}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
