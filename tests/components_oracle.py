"""References for the forecast components (DESIGN §12): fbprophet 0.5's per-seasonality columns of Prophet.predict, and
the noise-free trend draws of mc_kernel's own stream.

* ``predict`` is oracle/prophet_oracle.py's ``predict`` plus one column per seasonality, computed as fbprophet's
  predict_seasonal_components does: ``X_c @ (beta_c * s)`` with s the mode's indicator, times y_scale for an additive
  seasonality; a seasonality the model does not have is 0.
* ``trend_draws`` is the ``tr`` that oracle/mc_stream.py's ``draws`` forms before it adds the seasonality and the noise:
  the same key, the same simulated changepoints, the same fitted-changepoint state, so that the trend bounds can be held
  to it draw for draw as the yhat bounds are held to ``draws``.
"""
from __future__ import annotations

import numpy as np

from oracle import mc_stream as mcs
from oracle import prophet_oracle as po

SEASONALITIES = ("yearly", "weekly", "daily")


def predict(fr: po.FitResult, ds_ns, floor=None, cap=None, opts: po.ProphetOptions = None) -> dict:
    """po.predict's dict with ``yearly`` / ``weekly`` / ``daily`` added."""
    opts = opts or po.ProphetOptions()
    out = po.predict(fr, ds_ns, floor, cap, opts)
    p = fr.prep
    ds_ns = np.asarray(ds_ns, np.int64)
    X, _, s_a, s_m = po.seasonal_features(ds_ns, p.seasonalities, opts)
    for name in SEASONALITIES:
        out[name] = np.zeros(ds_ns.size)
    col = 0
    for s in p.seasonalities:
        blk = slice(col, col + 2 * s.order)
        if opts.seasonality_mode == "multiplicative":
            out[s.name] = X[:, blk] @ (fr.beta[blk] * s_m[blk])
        else:
            out[s.name] = (X[:, blk] @ (fr.beta[blk] * s_a[blk])) * p.y_scale
        col += 2 * s.order
    return out


def trend_draws(fitted, i: int, future_ds, floor: float, cap: float, logistic: bool, n_samples: int,
                seed: int) -> np.ndarray:
    """[H, n_samples] noise-free trend draws of model row ``i`` of a FittedBatch (numpy arrays), the stream of
    mc_stream.draws: ``draws == trend (1 + s) + noise`` (multiplicative) or ``trend + s y_scale + noise``."""
    pr = np.asarray(fitted.params[i], np.float64)
    S = int(fitted.meta_i32[i, 1])
    start, t_scale = int(fitted.meta_i64[i, 0]), int(fitted.meta_i64[i, 1])
    y_scale = float(fitted.meta_f64[i, 0])
    ds = np.asarray(future_ds, np.int64)
    assert np.all(np.diff(ds) >= 0), "mc_kernel wants ascending future timestamps"
    H, n = ds.size, int(n_samples)
    k0, k1 = mcs.model_key(seed, pr, fitted.tchange[i], start, t_scale, y_scale, floor, cap)
    t = (ds - start).astype(np.float64) / float(t_scale)
    fl = float(floor) if logistic else 0.0
    cap_s = (float(cap) - fl) / y_scale if logistic else 0.0
    k, m = float(pr[0]), float(pr[1])
    delta = [float(pr[3 + s]) for s in range(S)]
    tc = [float(fitted.tchange[i, s]) for s in range(S)]
    kh, mh, lam_acc, acc, kc = [k], [m], 0.0, 0.0, k
    for s in range(S):
        kn = kc + delta[s]
        if logistic:
            g = (tc[s] - m - acc) * (1.0 - kc / kn)
            acc += g
        else:
            g = -tc[s] * delta[s]
        kc = kn
        lam_acc += abs(delta[s])
        kh.append(kh[-1] + delta[s])
        mh.append(mh[-1] + g)
    lam = lam_acc / S + 1e-8
    s_hist = np.searchsorted(np.array(tc), t, side="right") if S else np.zeros(H, np.int64)
    nsim = np.zeros((n, H), np.int64)
    ks = np.full((n, 1), kh[-1])
    ms_ = np.full((n, 1), mh[-1])
    if t.max() > 1.0:
        pos, dl = mcs.simulated_changepoints(k0, k1, n, float(S), lam, t.max())
        kcol, mcol = [ks[:, 0]], [ms_[:, 0]]
        kk, mm = ks[:, 0].copy(), ms_[:, 0].copy()
        for c in range(pos.shape[1]):
            kn = kk + dl[:, c]
            if logistic:
                mm = mm + (pos[:, c] - mm) * (1.0 - kk / kn)
            else:
                mm = mm + -pos[:, c] * dl[:, c]
            kk = kn
            kcol.append(kk)
            mcol.append(mm)
        ks, ms_ = np.stack(kcol, axis=1), np.stack(mcol, axis=1)
        for c in range(pos.shape[1]):
            nsim += pos[:, c:c + 1] <= t[None, :]
    kt = np.where(nsim > 0, np.take_along_axis(ks, nsim, axis=1), np.array(kh)[s_hist][None, :])
    mt = np.where(nsim > 0, np.take_along_axis(ms_, nsim, axis=1), np.array(mh)[s_hist][None, :])
    with np.errstate(over="ignore"):
        tr = cap_s / (1.0 + np.exp(-kt * (t[None, :] - mt))) if logistic else kt * t[None, :] + mt
    return (tr * y_scale + fl).T
