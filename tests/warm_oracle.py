"""Warm-started fit restated on the numpy oracle (DESIGN §11): fbprophet's ``m.fit(df, init=stan_init(m_old))``.

fbprophet 0.5's ``Prophet.fit(df, **kwargs)`` passes ``kwargs`` into PyStan's ``optimizing`` after its own
``init=stan_init``, so a user's ``init`` replaces the cold start of the L-BFGS run and of the Newton retry that reuses
the same arguments, while the linear constant-``y`` shortcut keeps the local ``stan_init``.  This is
``oracle.prophet_oracle.fit`` with that one change, built from the oracle's own pieces; without ``init`` it is that
function."""
from __future__ import annotations

import math
from typing import Optional

import numpy as np

from oracle import prophet_oracle as po


def fit(ds_ns, y, floor: float = 0.0, cap: Optional[float] = None, opts: Optional[po.ProphetOptions] = None,
        cap_multiplier: float = 1.1, algorithm: str = "LBFGS+Newton", trace: Optional[list] = None,
        init: Optional[np.ndarray] = None, crit: Optional[list] = None) -> po.FitResult:
    """``po.fit`` started from ``init`` (Stan's unconstrained order k, m, delta[S], log sigma_obs, beta[K]) when given."""
    if init is None:
        return po.fit(ds_ns, y, floor, cap, opts, cap_multiplier, algorithm, trace, crit)
    opts = opts or po.ProphetOptions()
    ds_ns = np.asarray(ds_ns, dtype=np.int64)
    y = np.asarray(y, dtype=np.float64)
    if cap is None:
        cap = float(np.nanmax(y)) * cap_multiplier
    p = po.prepare(ds_ns, y, floor, cap, opts)
    x0 = np.array(init, dtype=np.float64)
    if x0.shape != (p.S + p.K + 3,):
        raise ValueError(f"init has {x0.size} values; the model has {p.S + p.K + 3}")   # PyStan: a dimension mismatch
    if p.constant_linear_shortcut:
        th, f, it, ret, ne = po.initial_theta(p), float("nan"), 0, po.TERM_SUCCESS, 0
        sigma = 1e-9
    else:
        fun = lambda x: po.neg_logp_grad(x, p)     # noqa: E731
        if algorithm == "Newton":
            th, f, it, ret, ne = po.stan_newton(fun, x0, opts)
        else:
            th, f, it, ret, ne = po.stan_lbfgs(fun, x0, opts, trace=trace, crit=crit)
            if ret == po.TERM_LSFAIL and algorithm == "LBFGS+Newton":
                th, f, it2, ret, ne2 = po.stan_newton(fun, x0, opts)
                it, ne = it + it2, ne + ne2
        sigma = math.exp(th[2 + p.S])
    S = p.S
    k, m, delta, beta = th[0], th[1], th[2:2 + S].copy(), th[3 + S:].copy()
    if p.n_changepoints_real == 0:
        k = k + float(delta[0])
        delta = np.zeros_like(delta)
    return po.FitResult(prep=p, k=float(k), m=float(m), delta=delta, sigma_obs=float(sigma), beta=beta,
                        theta=th, neg_logp=float(f), iters=it, n_evals=ne, ret=ret, last_ds_ns=int(np.max(ds_ns)))


def season_mask(p: po.Prepared) -> int:
    """The seasonality mask (1 yearly | 2 weekly | 4 daily) of a prepared history."""
    bits = {"yearly": 1, "weekly": 2, "daily": 4}
    return sum(bits[s.name] for s in p.seasonalities)


def record_of(fr: po.FitResult, smax: int, kmax: int):
    """An oracle fit as a model record's (params row, meta_i32 row): what the fit kernels would have written."""
    p = fr.prep
    row = np.zeros(3 + smax + kmax)
    row[0], row[1], row[2] = fr.k, fr.m, fr.sigma_obs
    row[3:3 + p.S] = fr.delta
    row[3 + smax:3 + smax + p.K] = fr.beta
    meta = np.array([p.t.size, p.S, p.n_changepoints_real, season_mask(p), 31, fr.iters, fr.n_evals, 0], np.int32)
    return row, meta
