"""Reference for the quantiles of window and period totals (DESIGN §21), on the CPU: the draws of
oracle/mc_stream.draws summed per window as window_oracle / period_oracle sum them (s = 0.0; s = s + d[h] in frame
order), then quantile_oracle.quantiles over each window's sums."""
import numpy as np

import period_oracle as pdo
import quantile_oracle as qo
import window_oracle as wo


def run_sums(d: np.ndarray, first) -> np.ndarray:
    """[W, n_samples]: each draw of ``d`` [H, n_samples] summed over the runs [first[j], first[j + 1])."""
    W = len(first) - 1
    sums = np.zeros((W, d.shape[1]))
    for j in range(W):
        for h in range(first[j], first[j + 1]):
            sums[j] = sums[j] + d[h]
    return sums


def window_quantiles(d: np.ndarray, ds, width_ns: int, origin_ns: int, percentiles) -> np.ndarray:
    """[Q, W]: plane q of each fixed-width window floor((ds - origin) / width) of the frame ``ds``."""
    first, _ = wo.window_runs(ds, width_ns, origin_ns)
    return qo.quantiles(run_sums(d, first), percentiles)


def period_quantiles(d: np.ndarray, ds, alias: str, percentiles) -> np.ndarray:
    """[Q, W]: plane q of each calendar period (pandas' ``to_period(alias)``) of the frame ``ds``."""
    first, _ = pdo.period_runs(ds, alias)
    return qo.quantiles(run_sums(d, first), percentiles)
