"""Numpy restatement of the backtest's window rows (DESIGN §14): the held-out rows after each cutoff summed per
fixed-width window anchored at the cutoff.  TEST INFRASTRUCTURE ONLY: the window tests hold csrc/cv_kernel.cuh's
cv_window_kernel and batched.cross_validation_device(aggregate_ns=...) to it; the window metrics are
tests/backtest_oracle.performance_metrics on these rows, and the window bounds tests/window_oracle.window_sums with
origin c + 1."""
import numpy as np


def window_rows(ds, cutoff, y, yhat, width_ns: int):
    """The backtest's window rows (DESIGN §14) of one series' held-out rows, given ordered by (cutoff, ds) as
    cross_validation returns them.  Per cutoff c, row r lies in window j = floor((ds_r - (c + 1)) / W) -- the window
    (c + j W, c + (j + 1) W], closed on the right like the held-out span -- and every window that holds a row gives, in
    ascending j: cutoff, horizon (j + 1) W, points, and y / yhat summed sequentially in row order (s = 0.0; s = s + v,
    plain fp64 adds).  ``first`` [windows + 1] indexes each window's first row in the input (the last entry: its
    length), for references that need the rows themselves."""
    ds = np.asarray(ds, np.int64)
    cutoff = np.asarray(cutoff, np.int64)
    y = np.asarray(y, np.float64)
    yhat = np.asarray(yhat, np.float64)
    W = int(width_ns)
    out = {k: [] for k in ("cutoff", "horizon", "points", "y", "yhat", "first")}
    r, n = 0, ds.size
    while r < n:
        c = int(cutoff[r])
        j = (int(ds[r]) - (c + 1)) // W
        e = r
        sy, sf = 0.0, 0.0
        while e < n and int(cutoff[e]) == c and (int(ds[e]) - (c + 1)) // W == j:
            sy = sy + float(y[e])
            sf = sf + float(yhat[e])
            e += 1
        for k, v in (("cutoff", c), ("horizon", (j + 1) * W), ("points", e - r), ("y", sy), ("yhat", sf), ("first", r)):
            out[k].append(v)
        r = e
    res = {k: np.array(out[k], dtype=np.float64 if k in ("y", "yhat") else np.int64) for k in out}
    res["first"] = np.append(res["first"], n).astype(np.int64)
    return res
