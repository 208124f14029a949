"""Numpy restatement of the backtest's semantics (DESIGN §9): fbprophet.diagnostics' generate_cutoffs and
cross_validation (fbprophet 0.5, restated from recall -- fbprophet is not importable here) and performance_metrics
(the per-horizon rolling_mean_by_h of later fbprophet releases, also from recall).  TEST INFRASTRUCTURE ONLY: the
backtest tests hold csrc/cv_kernel.cuh and batched.cross_validation_device to it.  The fits and predictions it makes
come from oracle/prophet_oracle.py, unchanged."""
from __future__ import annotations

import math
from typing import Optional

import numpy as np

from oracle.prophet_oracle import ProphetOptions, auto_seasonalities, fit, predict


def generate_cutoffs(ds_sorted, horizon_ns: int, period_ns: int, initial_ns: int) -> np.ndarray:
    """fbprophet 0.5 diagnostics.generate_cutoffs (restated from recall), in the binary-search form cv_kernel.cuh runs:
    start at ``last - horizon``; while the latest cutoff is >= ``first + initial`` step back by ``period``, and when no
    row lies in ``(c, c + horizon]`` move to ``(latest row <= c) - horizon`` (no such row: fbprophet's NaT, which ends
    the loop); drop the last cutoff; ascending.  ValueError for fbprophet's two cases."""
    ds = np.asarray(ds_sorted, dtype=np.int64)
    first, last = int(ds[0]), int(ds[-1])
    prev = last - int(horizon_ns)
    if prev < first:
        raise ValueError("Less data than horizon.")
    out = []
    while prev >= first + int(initial_ns):
        c = prev - int(period_ns)
        u = int(np.searchsorted(ds, c, side="right"))           # first row > c
        stop = False
        if not (u < ds.size and ds[u] <= c + int(horizon_ns)):
            if u == 0:
                stop = True
            else:
                c = int(ds[u - 1]) - int(horizon_ns)
        out.append(prev)
        if stop:
            break
        prev = c
    if not out:
        raise ValueError("Less data than horizon after initial window. Make horizon or initial shorter.")
    return np.array(out[::-1], dtype=np.int64)


def seasonality_mask(ds_sorted, opts: Optional[ProphetOptions] = None) -> int:
    """1 yearly | 2 weekly | 4 daily of auto_seasonalities on this history."""
    bit = {"yearly": 1, "weekly": 2, "daily": 4}
    return sum(bit[s.name] for s in auto_seasonalities(np.asarray(ds_sorted, np.int64), opts or ProphetOptions()))


def cross_validation(ds_ns, y, horizon_ns: int, period_ns: int, initial_ns: int, floor: float = 0.0,
                     cap_multiplier: float = 1.1, opts: Optional[ProphetOptions] = None):
    """fbprophet 0.5 diagnostics.cross_validation for one series (restated from recall): per cutoff, a fit on the rows
    ``ds <= cutoff`` with the full model's options except the seasonalities, which are the FULL history's (prophet_copy
    turns auto off and copies the fitted seasonalities), the full-history float64 cap, and a prediction of the rows
    ``cutoff < ds <= cutoff + horizon``.  Returns (rows dict ds / cutoff / y / yhat, list of FitResult)."""
    opts = opts or ProphetOptions()
    ds_ns = np.asarray(ds_ns, dtype=np.int64)
    y = np.asarray(y, dtype=np.float64)
    order = np.argsort(ds_ns, kind="stable")
    ds, yy = ds_ns[order], y[order]
    cap = float(np.max(yy)) * cap_multiplier
    mask = seasonality_mask(ds, opts)
    oc = ProphetOptions(**{**opts.__dict__, "yearly_seasonality": bool(mask & 1), "weekly_seasonality": bool(mask & 2),
                           "daily_seasonality": bool(mask & 4)})
    rows = {"ds": [], "cutoff": [], "y": [], "yhat": []}
    fits = []
    for c in generate_cutoffs(ds, horizon_ns, period_ns, initial_ns):
        he = int(np.searchsorted(ds, c, side="right"))
        we = int(np.searchsorted(ds, c + horizon_ns, side="right"))
        if he < 2:
            raise ValueError("Less than two datapoints before cutoff. Increase initial window.")
        fr = fit(ds[:he], yy[:he], floor, cap, oc)
        pr = predict(fr, ds[he:we], floor, cap, oc)
        rows["ds"].append(ds[he:we])
        rows["cutoff"].append(np.full(we - he, c, np.int64))
        rows["y"].append(yy[he:we])
        rows["yhat"].append(pr["yhat"])
        fits.append(fr)
    return {k: np.concatenate(v) for k, v in rows.items()}, fits


def performance_metrics(horizon_ns, y, yhat, yhat_lower=None, yhat_upper=None, rolling_window: float = 0.1):
    """performance_metrics of ONE series (per-horizon form; rolling_mean_by_h of later fbprophet releases, restated
    from recall).  With n rows and w = min(n, max(1, int(rolling_window n))), each distinct horizon h gets the mean over
    w rows: every row of h, then rows of smaller horizons nearest first, the group where the window stops contributing
    its mean times the rows it still needs (computed as sum * (need / count)); horizons with fewer than w rows at or
    below them get no row.  mape = |y - yhat| / |y|, NaN for every horizon when some |y| < 1e-8; coverage only with
    intervals.  Within a horizon rows are summed in their given order, as the kernel does."""
    if not (0.0 <= rolling_window <= 1.0):
        raise ValueError(f"rolling_window must be in [0, 1] (got {rolling_window!r})")
    h = np.asarray(horizon_ns, np.int64)
    y = np.asarray(y, np.float64)
    e = y - np.asarray(yhat, np.float64)
    n = h.size
    iv = yhat_lower is not None
    cov = ((np.asarray(yhat_lower) <= y) & (y <= np.asarray(yhat_upper))).astype(np.float64) if iv else np.zeros(n)
    tiny = bool(np.any(np.abs(y) < 1e-8))
    w = min(n, max(1, int(rolling_window * n)))
    order = np.argsort(h, kind="stable")
    hs = []
    sums = []          # per distinct horizon: [se, ae, ape, cov, count]
    for i in order:
        if not hs or hs[-1] != h[i]:
            hs.append(h[i])
            sums.append([0.0, 0.0, 0.0, 0.0, 0])
        s = sums[-1]
        s[0] += e[i] * e[i]
        s[1] += abs(e[i])
        s[2] += abs(e[i]) / abs(y[i])
        s[3] += cov[i]
        s[4] += 1
    out = {k: [] for k in ("horizon", "mse", "rmse", "mae", "mape", "coverage")}
    for k in range(len(hs)):
        acc = [0.0, 0.0, 0.0, 0.0]
        need = w
        for g in range(k, -1, -1):
            if need <= 0:
                break
            c = sums[g][4]
            f = need / c if c >= need else 1.0
            for j in range(4):
                acc[j] += sums[g][j] * f if c >= need else sums[g][j]
            need = 0 if c >= need else need - c
        if need > 0:
            continue
        mse = acc[0] / w
        out["horizon"].append(hs[k])
        out["mse"].append(mse)
        out["rmse"].append(math.sqrt(mse))
        out["mae"].append(acc[1] / w)
        out["mape"].append(float("nan") if tiny else acc[2] / w)
        out["coverage"].append(acc[3] / w if iv else float("nan"))
    res = {k: np.array(v, dtype=np.int64 if k == "horizon" else np.float64) for k, v in out.items()}
    if not iv:
        res["coverage"] = None
    return res
