"""Reference for forecast quantiles and their backtest calibration (DESIGN §15), on the CPU.

``quantiles`` restates the kernel's percentile over the draws of oracle/mc_stream.draws; ``quantile_metrics`` the
per-horizon rule of backtest_oracle.performance_metrics for the pinball loss and the share of y at or below the
quantile, through that function itself."""
import numpy as np

import backtest_oracle as bo


def quantiles(d: np.ndarray, percentiles) -> np.ndarray:
    """[Q, H]: for each percentile p, x = p / 100 (n - 1), i = floor(x), f = x - i, s_i + (s_{min(i+1, n-1)} - s_i) f over
    each point's sorted draws s (d: [H, n])."""
    s = np.sort(np.asarray(d, np.float64), axis=1)
    n = s.shape[1]
    out = []
    for p in percentiles:
        x = float(p) / 100.0 * (n - 1)
        i = int(np.floor(x))
        f = x - np.floor(x)
        v0, v1 = s[:, i], s[:, min(i + 1, n - 1)]
        out.append(v0 + (v1 - v0) * f)
    return np.array(out).reshape(len(out), s.shape[0])


def pinball(y, yq, level):
    """max(q e, (q - 1) e) with e = y - yq, per row."""
    e = np.asarray(y, np.float64) - np.asarray(yq, np.float64)
    return np.maximum(level * e, (level - 1.0) * e)


def quantile_metrics(horizon, y, yq, levels, rolling_window: float = 0.1):
    """ONE series' rows: {level index: {"horizon", "pinball", "share_below"}}.  The pinball loss is the rolling mean of
    the per-row loss (performance_metrics' mae of the loss against 0: the loss is >= 0), the share the rolling mean of
    [y <= yq] (performance_metrics' coverage of the interval [-inf, yq])."""
    h = np.asarray(horizon, np.int64)
    y = np.asarray(y, np.float64)
    out = {}
    for q, lv in enumerate(levels):
        yqq = np.asarray(yq[q], np.float64)
        m1 = bo.performance_metrics(h, pinball(y, yqq, lv), np.zeros(h.size), rolling_window=rolling_window)
        m2 = bo.performance_metrics(h, y, y, np.full(h.size, -np.inf), yqq, rolling_window=rolling_window)
        out[q] = {"horizon": m1["horizon"], "pinball": m1["mae"], "share_below": m2["coverage"]}
    return out
