"""Numpy restatement of mc_sum_kernel's windows and window sums (DESIGN §13), on top of the draws that
oracle/mc_stream.draws restates: the reference every window bound of the GPU is held to."""
import numpy as np

from oracle import mc_stream as mcs


def window_runs(ds, width_ns: int, origin_ns: int = 0):
    """The windows of an ascending frame under w(ds) = floor((ds - origin) / width): (index of each run's first point
    [W + 1, the last entry is the frame's length], start of each window [W] = origin + w * width)."""
    ds = np.asarray(ds, np.int64)
    w = (ds - np.int64(origin_ns)) // np.int64(width_ns)
    first = np.concatenate([[0], np.flatnonzero(np.diff(w) != 0) + 1, [ds.size]]) if ds.size else np.zeros(1, np.int64)
    return first.astype(np.int64), np.int64(origin_ns) + w[first[:-1]] * np.int64(width_ns)


def window_sums(d: np.ndarray, ds, width_ns: int, origin_ns: int, width: float):
    """mc_sum_kernel's window bounds from the draws ``d`` [H, n_samples] of ``mc_stream.draws(...)`` on the frame ``ds``:
    (window_start [W], n_points [W], lower [W], upper [W]).  Each draw's sum is sequential over the window's points
    (s = 0.0; s = s + d[h]), the bounds numpy's linear-interpolation percentiles over the sums."""
    first, start = window_runs(ds, width_ns, origin_ns)
    W = start.size
    sums = np.zeros((W, d.shape[1]))
    for j in range(W):
        for h in range(first[j], first[j + 1]):
            sums[j] = sums[j] + d[h]
    lo, hi = mcs.bounds(sums, width) if W else (np.zeros(0), np.zeros(0))
    return start, np.diff(first).astype(np.int64), lo, hi
