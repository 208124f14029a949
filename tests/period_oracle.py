"""Pandas restatement of the calendar periods of mc_sum_kernel's calendar instance (DESIGN §17) and of its period sums,
on top of the draws that oracle/mc_stream.draws restates: the reference every period bound of the GPU is held to."""
import numpy as np
import pandas as pd

from oracle import mc_stream as mcs


def period_runs(ds, alias: str):
    """The periods of an ascending frame under pandas' ``DatetimeIndex.to_period(alias)``: (index of each run's first
    point [W + 1, the last entry is the frame's length], start of each period [W] from ``start_time``)."""
    ds = np.asarray(ds, np.int64)
    if ds.size == 0:
        return np.zeros(1, np.int64), np.zeros(0, np.int64)
    per = pd.DatetimeIndex(ds.astype("datetime64[ns]")).to_period(alias)
    code = np.asarray(per.asi8, np.int64)
    first = np.concatenate([[0], np.flatnonzero(np.diff(code) != 0) + 1, [ds.size]]).astype(np.int64)
    start = per[first[:-1]].start_time.values.astype("datetime64[ns]").astype(np.int64)
    return first, start


def period_sums(d: np.ndarray, ds, alias: str, width: float):
    """The period bounds of the draws ``d`` [H, n_samples] of ``mc_stream.draws(...)`` on the frame ``ds``, as
    window_oracle.window_sums: (period_start [W], n_points [W], lower [W], upper [W]); each draw's sum is sequential over
    the period's points (s = 0.0; s = s + d[h]), the bounds numpy's linear-interpolation percentiles over the sums."""
    first, start = period_runs(ds, alias)
    W = start.size
    sums = np.zeros((W, d.shape[1]))
    for j in range(W):
        for h in range(first[j], first[j + 1]):
            sums[j] = sums[j] + d[h]
    lo, hi = mcs.bounds(sums, width) if W else (np.zeros(0), np.zeros(0))
    return start, np.diff(first).astype(np.int64), lo, hi
