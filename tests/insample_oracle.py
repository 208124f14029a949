"""Reference for the in-sample predict, its outlier flags and the batch without the flagged rows (DESIGN §16), on the
CPU.

``yhat`` is prophet_oracle's predict on the history timestamps; ``bounds`` mc_stream's interval over the history frame
(the model's own rows: the same key, counters and Tmax as the kernel); ``flags`` / ``kept_batch`` the flags, the kept
counts and the filtered batch."""
import numpy as np

from oracle import mc_stream as mcs
from oracle import prophet_oracle as po


def yhat(fr, ds_ns, floor, cap, opts=None) -> np.ndarray:
    """fbprophet's m.predict() yhat at the history timestamps ``ds_ns`` of the fit ``fr``."""
    return po.predict(fr, ds_ns, floor, cap, opts)["yhat"]


def bounds(fitted, i: int, ds_ns, floor: float, cap: float, logistic: bool, multiplicative: bool, n_samples: int,
           width: float, seed: int):
    """(yhat_lower, yhat_upper) of model row ``i`` over its history frame ``ds_ns``."""
    d = mcs.draws(fitted, i, ds_ns, floor, cap, logistic, multiplicative, n_samples, seed)
    return mcs.bounds(d, width)


def flags(y, lower, upper) -> np.ndarray:
    """y < lower or y > upper, with y as float64; a NaN bound never flags."""
    y = np.asarray(y).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return (y < np.asarray(lower)) | (y > np.asarray(upper))


def kept_batch(ds_ns, y, offsets, flag):
    """The batch without the flagged rows: (kept [N] int64, offsets [N + 1] int64, ds, y), rows in their order and y in
    its own dtype."""
    offsets = np.asarray(offsets, np.int64)
    keep = ~np.asarray(flag, bool)
    series = np.repeat(np.arange(offsets.size - 1), np.diff(offsets))
    kept = np.bincount(series[keep], minlength=offsets.size - 1).astype(np.int64)
    off = np.concatenate(([0], np.cumsum(kept))).astype(np.int64)
    return kept, off, np.asarray(ds_ns)[keep], np.asarray(y)[keep]
