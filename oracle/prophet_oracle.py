"""CPU float64 oracle for the batched-Prophet hot path.  TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED.  The reference (mageky/time-series-spark) keeps all of its
arithmetic in two un-vendored third-party pins, ``fbprophet==0.5`` and
``pystan==2.19.1.1`` (reference environment.yml:12-13).  Neither is
installed here, neither can be fetched (no network), and the reference's own
tests pin no numerical value (tests/unit/*.py assert row counts and column
names only).  This file therefore *restates the published algorithm* of those
two pins from knowledge of the upstream sources; it has NOT been checked
against a real fbprophet run.  What anchors it instead:

  * the reference's call sites: ``Prophet(growth='logistic',
    seasonality_mode='multiplicative').fit(pdf)`` (src/jobs/prophet_modeler.py:65-66),
    ``make_future_dataframe`` / ``predict`` (src/jobs/prophet_scorer.py:64-70);
  * finite-difference checks of the analytic gradient (tests/test_oracle.py);
  * an independent optimiser (scipy L-BFGS-B) reaching the same optimum;
  * an independent C restatement (oracle/prophet_oracle.c) agreeing with this file.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline
legs may import this module.  The product path (``time_series_spark_b200``)
never does; it fails loudly if the CUDA library is missing.

Upstream functions restated (facebook/prophet tag v0.5,
python/fbprophet/forecaster.py and python/stan/unix/prophet.stan;
stan-dev/stan v2.19 src/stan/optimization/{bfgs,bfgs_linesearch,lbfgs_update}.hpp,
src/stan/services/optimize/lbfgs.hpp; PyStan 2.19.1.1 ``StanModel.optimizing``
defaults).  Every function names the upstream routine it follows.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

NS_PER_DAY = 86400 * 10**9
EPS = np.finfo(np.float64).eps


# --------------------------------------------------------------------------
# options (Prophet.__init__ defaults, fbprophet 0.5) with the two overrides the
# reference hard-codes at src/jobs/prophet_modeler.py:65
# --------------------------------------------------------------------------
@dataclass
class ProphetOptions:
    growth: str = "logistic"                 # prophet_modeler.py:65
    seasonality_mode: str = "multiplicative"  # prophet_modeler.py:65
    n_changepoints: int = 25
    changepoint_range: float = 0.8
    yearly_seasonality: object = "auto"
    weekly_seasonality: object = "auto"
    daily_seasonality: object = "auto"
    seasonality_prior_scale: float = 10.0
    changepoint_prior_scale: float = 0.05
    interval_width: float = 0.80
    uncertainty_samples: int = 1000
    # PyStan 2.19.1.1 optimizing() defaults, iter overridden by fbprophet.fit (iter=1e4)
    max_iter: int = 10000
    history_size: int = 5
    init_alpha: float = 1e-3
    tol_obj: float = 1e-12
    tol_rel_obj: float = 1e4
    tol_grad: float = 1e-8
    tol_rel_grad: float = 1e7
    tol_param: float = 1e-8


@dataclass
class Seasonality:
    name: str
    period: float
    order: int


@dataclass
class Prepared:
    """Everything Prophet.fit hands to Stan (the ``dat`` dict) plus scaling meta."""
    T: int
    S: int
    K: int
    t: np.ndarray
    y: np.ndarray            # y_scaled
    cap: np.ndarray          # cap_scaled per row (zeros for linear)
    X: np.ndarray            # T x K
    sigmas: np.ndarray       # K prior scales
    s_a: np.ndarray
    s_m: np.ndarray
    t_change: np.ndarray     # S (dummy [0] if no changepoints)
    tau: float
    logistic: bool
    start_ns: int
    t_scale_ns: int
    y_scale: float
    floor: float
    cap_value: float
    seasonalities: List[Seasonality]
    n_changepoints_real: int  # 0 if dummy
    ds_sorted: np.ndarray
    y_raw_sorted: np.ndarray
    A: np.ndarray = field(default=None, repr=False)
    constant_linear_shortcut: bool = False


@dataclass
class FitResult:
    prep: Prepared
    k: float
    m: float
    delta: np.ndarray
    sigma_obs: float
    beta: np.ndarray
    theta: np.ndarray        # unconstrained (k, m, delta, log sigma, beta)
    neg_logp: float
    iters: int
    n_evals: int
    ret: int                 # Stan TerminationCondition code
    last_ds_ns: int = 0


# Stan TerminationCondition (bfgs.hpp)
TERM_SUCCESS, TERM_ABSX, TERM_ABSF, TERM_RELF = 0, 10, 20, 21
TERM_ABSGRAD, TERM_RELGRAD, TERM_MAXIT, TERM_LSFAIL = 30, 31, 40, -1
TERM_NEWTON = 60     # not a Stan code: the model came from fbprophet's Newton retry (stan_newton below)


# --------------------------------------------------------------------------
# preprocessing  (Prophet.fit -> setup_dataframe / initialize_scales /
# set_auto_seasonalities / make_all_seasonality_features / set_changepoints)
# --------------------------------------------------------------------------
def fourier_series(ds_ns: np.ndarray, period: float, order: int) -> np.ndarray:
    """Prophet.fourier_series: days since epoch as float; columns sin,cos per order.

    ``t = (dates - 1970-01-01).dt.total_seconds() / (3600*24.)`` where pandas
    0.25's total_seconds is ``1e-9 * asi8``; argument evaluated left to right
    as ``2.0 * (i + 1) * np.pi * t / period``.
    """
    t = (1e-9 * ds_ns.astype(np.float64)) / (3600 * 24.)
    cols = []
    for i in range(order):
        arg = 2.0 * (i + 1) * np.pi * t / period
        cols.append(np.sin(arg))
        cols.append(np.cos(arg))
    return np.column_stack(cols) if cols else np.zeros((len(ds_ns), 0))


def _parse_seasonality_arg(arg, auto_disable: bool, default_order: int) -> int:
    """Prophet.parse_seasonality_args."""
    if isinstance(arg, str) and arg == "auto":
        return 0 if auto_disable else default_order
    if arg is True:
        return default_order
    if arg is False:
        return 0
    return int(arg)


def auto_seasonalities(ds_sorted: np.ndarray, opts: ProphetOptions) -> List[Seasonality]:
    """Prophet.set_auto_seasonalities (yearly 365.25/10, weekly 7/3, daily 1/4)."""
    first, last = int(ds_sorted[0]), int(ds_sorted[-1])
    span = last - first
    dt = np.diff(ds_sorted)
    nz = dt[dt != 0]
    min_dt = int(nz.min()) if nz.size else None
    out = []
    yearly_disable = span < 730 * NS_PER_DAY
    weekly_disable = (span < 14 * NS_PER_DAY) or (min_dt is not None and min_dt >= 7 * NS_PER_DAY)
    daily_disable = (span < 2 * NS_PER_DAY) or (min_dt is not None and min_dt >= 1 * NS_PER_DAY)
    for name, arg, dis, period, order in (
        ("yearly", opts.yearly_seasonality, yearly_disable, 365.25, 10),
        ("weekly", opts.weekly_seasonality, weekly_disable, 7.0, 3),
        ("daily", opts.daily_seasonality, daily_disable, 1.0, 4),
    ):
        fo = _parse_seasonality_arg(arg, dis, order)
        if fo > 0:
            out.append(Seasonality(name, period, fo))
    return out


def seasonal_features(ds_ns: np.ndarray, seas: Sequence[Seasonality], opts: ProphetOptions):
    """Prophet.make_all_seasonality_features + regressor_column_matrix.

    Returns X, prior scales, s_a, s_m.  With no seasonality a single all-zero
    column with prior scale 1 and s_a = s_m = 0 (the 'zeros' placeholder).
    """
    blocks, sig = [], []
    for s in seas:
        blocks.append(fourier_series(ds_ns, s.period, s.order))
        sig += [opts.seasonality_prior_scale] * (2 * s.order)
    if not blocks:
        X = np.zeros((len(ds_ns), 1))
        return X, np.array([1.0]), np.zeros(1), np.zeros(1)
    X = np.column_stack(blocks)
    K = X.shape[1]
    if opts.seasonality_mode == "multiplicative":
        s_a, s_m = np.zeros(K), np.ones(K)
    else:
        s_a, s_m = np.ones(K), np.zeros(K)
    return X, np.array(sig, dtype=np.float64), s_a, s_m


def changepoint_indexes(T: int, opts: ProphetOptions) -> np.ndarray:
    """Prophet.set_changepoints: indices into the sorted history (may be empty)."""
    hist_size = int(np.floor(T * opts.changepoint_range))
    n_cp = opts.n_changepoints
    if n_cp + 1 > hist_size:
        n_cp = hist_size - 1
    if n_cp > 0:
        idx = np.linspace(0, hist_size - 1, n_cp + 1).round().astype(np.int64)
        return idx[1:]
    return np.zeros(0, dtype=np.int64)


def prepare(ds_ns, y, floor: float, cap: float, opts: ProphetOptions) -> Prepared:
    """Prophet.fit up to the ``dat`` dict.  ``ds_ns`` int64 ns since epoch, any order;
    ``y`` float (NaN = null).  ``floor``/``cap`` are the per-series constants the
    reference UDF writes into the frame (prophet_modeler.py:56-60)."""
    ds_ns = np.asarray(ds_ns, dtype=np.int64)
    y = np.asarray(y, dtype=np.float64)
    keep = ~np.isnan(y)
    ds_ns, y = ds_ns[keep], y[keep]
    if ds_ns.size < 2:
        raise ValueError("Dataframe has less than 2 non-NaN rows.")
    if np.isinf(y).any():
        raise ValueError("Found infinity in column y.")
    order = np.argsort(ds_ns, kind="stable")
    ds, yr = ds_ns[order], y[order]
    logistic = opts.growth == "logistic"
    # initialize_scales: floor only honoured for logistic growth
    fl = float(floor) if logistic else 0.0
    y_scale = float(np.abs(yr - fl).max())
    if y_scale == 0:
        y_scale = 1.0
    start = int(ds[0])
    t_scale = int(ds[-1]) - start
    if logistic:
        if cap <= fl:
            raise ValueError("cap must be greater than floor (which defaults to 0).")
        cap_s = np.full(ds.size, (float(cap) - fl) / y_scale)
    else:
        cap_s = np.zeros(ds.size)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (ds - start).astype(np.float64) / np.float64(t_scale)
    y_s = (yr - fl) / y_scale
    seas = auto_seasonalities(ds, opts)
    X, sig, s_a, s_m = seasonal_features(ds, seas, opts)
    idx = changepoint_indexes(ds.size, opts)
    if idx.size:
        t_change = np.sort(t[idx])
    else:
        t_change = np.array([0.0])
    A = (t[:, None] >= t_change[None, :]).astype(np.float64)
    const = bool(yr.min() == yr.max()) and not logistic
    return Prepared(T=ds.size, S=t_change.size, K=X.shape[1], t=t, y=y_s, cap=cap_s, X=X,
                    sigmas=sig, s_a=s_a, s_m=s_m, t_change=t_change,
                    tau=opts.changepoint_prior_scale, logistic=logistic, start_ns=start,
                    t_scale_ns=t_scale, y_scale=y_scale, floor=fl, cap_value=float(cap),
                    seasonalities=list(seas), n_changepoints_real=int(idx.size),
                    ds_sorted=ds, y_raw_sorted=yr, A=A, constant_linear_shortcut=const)


def initial_theta(p: Prepared) -> np.ndarray:
    """Prophet.linear_growth_init / logistic_growth_init + stan_init (delta=0, beta=0,
    sigma_obs=1 -> log sigma = 0).  idxmin/idxmax pick the FIRST min / FIRST max ds."""
    i0 = 0
    i1 = int(np.argmax(p.ds_sorted))          # first occurrence of the max
    Tspan = p.t[i1] - p.t[i0]
    if p.logistic:
        C0, C1 = p.cap[i0], p.cap[i1]
        y0 = max(0.01 * C0, min(0.99 * C0, p.y[i0]))
        y1 = max(0.01 * C1, min(0.99 * C1, p.y[i1]))
        r0, r1 = C0 / y0, C1 / y1
        if abs(r0 - r1) <= 0.01:
            r0 = 1.05 * r0
        L0, L1 = math.log(r0 - 1), math.log(r1 - 1)
        m = L0 * Tspan / (L0 - L1)
        k = (L0 - L1) / Tspan
    else:
        k = (p.y[i1] - p.y[i0]) / Tspan
        m = p.y[i0] - k * p.t[i0]
    th = np.zeros(p.S + p.K + 3)
    th[0], th[1] = k, m
    return th


# --------------------------------------------------------------------------
# Stan model: -log_prob and its gradient (propto=true, jacobian=false)
# --------------------------------------------------------------------------
def neg_logp_grad(theta: np.ndarray, p: Prepared) -> Tuple[int, float, np.ndarray]:
    """prophet.stan ``model`` block, negated, with analytic reverse-mode gradient.

    Unconstrained order is the Stan declaration order: k, m, delta[S],
    sigma_obs (log-transformed, lower=0), beta[K].  Returns (err, f, g) with the
    error convention of stan::optimization::ModelAdaptor::operator():
    1 = model threw (non-finite location / non-positive or infinite scale),
    2 = non-finite f, 3 = non-finite gradient.
    """
    S, K, T = p.S, p.K, p.T
    g = np.zeros_like(theta)
    if not np.all(np.isfinite(theta)):
        return 1, np.nan, g
    k, m = theta[0], theta[1]
    delta = theta[2:2 + S]
    u = theta[2 + S]
    beta = theta[3 + S:]
    with np.errstate(all="ignore"):
        sigma = math.exp(u) if u < 709.0 else math.inf
        if not (sigma > 0 and math.isfinite(sigma)):
            return 1, np.nan, g
        A, t = p.A, p.t
        if p.logistic:
            k_s = np.concatenate(([k], k + np.cumsum(delta)))
            gamma = np.zeros(S)
            m_prs = np.zeros(S)
            m_pr = m
            for i in range(S):
                m_prs[i] = m_pr
                gamma[i] = (p.t_change[i] - m_pr) * (1 - k_s[i] / k_s[i + 1])
                m_pr = m_pr + gamma[i]
            kt = k + A @ delta
            mt = m + A @ gamma
            z = kt * (t - mt)
            sg = 1.0 / (1.0 + np.exp(-z))
            trend = p.cap * sg
        else:
            kt = k + A @ delta
            mt = m + A @ (-p.t_change * delta)
            trend = kt * t + mt
        Xm = p.X @ (beta * p.s_m)
        Xa = p.X @ (beta * p.s_a)
        mu = trend * (1 + Xm) + Xa
        if not np.all(np.isfinite(mu)):
            return 1, np.nan, g
        r = p.y - mu
        ss = float(r @ r)
        inv_s2 = float(np.float64(1.0) / np.float64(sigma * sigma))   # sigma^2 may underflow to 0: inf, reported as a non-finite objective
        f = (0.5 * ss * inv_s2 + T * u + k * k / 50.0 + m * m / 50.0
             + np.abs(delta).sum() / p.tau + 2.0 * sigma * sigma
             + float(np.sum(beta * beta / (2.0 * p.sigmas ** 2))))
        w = -r * inv_s2                                  # df/dmu
        g[3 + S:] = (p.X.T @ (w * trend)) * p.s_m + (p.X.T @ w) * p.s_a + beta / p.sigmas ** 2
        q = w * (1 + Xm)                                 # df/dtrend
        if p.logistic:
            dz = q * p.cap * sg * (1 - sg)
            dkt = dz * (t - mt)
            dmt = dz * (-kt)
            gk = dkt.sum()
            gdelta = A.T @ dkt
            gm = dmt.sum()
            ggamma = A.T @ dmt
            a_ks = np.zeros(S + 1)
            a_mpr = 0.0
            for i in range(S - 1, -1, -1):
                a_gam = ggamma[i] + a_mpr
                ratio = k_s[i] / k_s[i + 1]
                d = p.t_change[i] - m_prs[i]
                a_ks[i] += a_gam * d * (-1.0 / k_s[i + 1])
                a_ks[i + 1] += a_gam * d * ratio / k_s[i + 1]
                a_mpr = a_mpr + a_gam * (-(1 - ratio))
            gm += a_mpr
            gk += a_ks.sum()
            suffix = np.cumsum(a_ks[::-1])[::-1]          # suffix[i] = sum_{j>=i} a_ks[j]
            gdelta = gdelta + suffix[1:]
        else:
            dkt = q * t
            gk = dkt.sum()
            gm = q.sum()
            gdelta = A.T @ dkt + (-p.t_change) * (A.T @ q)
        g[0] = gk + k / 25.0
        g[1] = gm + m / 25.0
        g[2:2 + S] = gdelta + np.sign(delta) / p.tau
        g[2 + S] = -ss * inv_s2 + T + 4.0 * sigma * sigma
    if not np.all(np.isfinite(g)):
        return 3, f, g
    if not math.isfinite(f):
        return 2, f, g
    return 0, float(f), g


# --------------------------------------------------------------------------
# Stan L-BFGS (bfgs.hpp BFGSMinimizer + LBFGSUpdate + bfgs_linesearch.hpp)
# --------------------------------------------------------------------------
def _cubic_interp(df0, x1, f1, df1, loX, hiX):
    """bfgs_linesearch.hpp CubicInterp(df0, x1, f1, df1, loX, hiX): minimiser on
    [loX, hiX] of the cubic through (0,0) slope df0 and (x1,f1) slope df1."""
    # numpy float64 scalars give the IEEE semantics of the C++ (x/0 = inf, sqrt(<0) = nan)
    df0, x1, f1, df1 = np.float64(df0), np.float64(x1), np.float64(f1), np.float64(df1)
    with np.errstate(all="ignore"):
        c3 = (-12 * f1 + 6 * x1 * (df0 + df1)) / (x1 * x1 * x1)
        c2 = -(4 * df0 + 2 * df1) / x1 + 6 * f1 / (x1 * x1)
        c1 = df0
        t_s = np.sqrt(c2 * c2 - 2.0 * c1 * c3)
        s1 = -(c2 + t_s) / c3
        s2 = -(c2 - t_s) / c3

    def poly(x):
        with np.errstate(all="ignore"):
            return x * (x * (x * c3 / 3.0 + c2) / 2.0 + c1)

    minF, minX = poly(loX), loX
    tmpF = poly(hiX)
    if tmpF < minF:
        minF, minX = tmpF, hiX
    if loX < s1 < hiX:
        tmpF = poly(s1)
        if tmpF < minF:
            minF, minX = tmpF, s1
    if loX < s2 < hiX:
        tmpF = poly(s2)
        if tmpF < minF:
            minF, minX = tmpF, s2
    return minX


class _Counter:
    def __init__(self, fun):
        self.fun, self.n = fun, 0

    def __call__(self, x):
        self.n += 1
        return self.fun(x)


def _wolfe_zoom(func, x, f, dfp, c1dfp, c2dfp, p, alo, aloF, aloDFp, ahi, ahiF, ahiDFp, min_range):
    """bfgs_linesearch.hpp WolfLSZoom.  Returns (ret, alpha, newX, newF, newDF)."""
    itNum = 0
    alpha, newX, newF, newDF = 0.0, x, f, None
    while True:
        itNum += 1
        if abs(alo - ahi) < min_range:
            return 1, alpha, newX, newF, newDF
        mid = 0.5 * (alo + ahi)
        if mid == alo or mid == ahi:
            # [guard, not in Stan] alo and ahi are adjacent doubles wider than min_range (|alpha| > ~0.5):
            # upstream's loop cannot shrink the bracket any further and spins forever when the
            # gradient has a kink (Laplace prior) inside it.  Observed on 1 of 200k config-#4 series.
            return 1, alpha, newX, newF, newDF
        if itNum % 5 == 0:
            alpha = 0.5 * (alo + ahi)
        else:
            with np.errstate(all="ignore"):
                d1 = aloDFp + ahiDFp - 3 * (aloF - ahiF) / (alo - ahi)
                rad = d1 * d1 - aloDFp * ahiDFp
                d2 = math.sqrt(rad) if rad >= 0 else math.nan
                if ahi < alo:
                    d2 = -d2
                den = (ahiDFp - aloDFp + 2 * d2)
                alpha = ahi - (ahi - alo) * (ahiDFp + d2 - d1) / den if den != 0 else math.nan
            lo, hi = min(alo, ahi), max(alo, ahi)
            if (not math.isfinite(alpha)) or alpha < lo + 0.01 * abs(alo - ahi) or alpha > hi - 0.01 * abs(alo - ahi):
                alpha = 0.5 * (alo + ahi)
        newX = x + alpha * p
        while True:
            err, newF, newDF = func(newX)
            if not err:
                break
            alpha = 0.5 * (alpha + min(alo, ahi))
            if abs(min(alo, ahi) - alpha) < min_range:
                return 1, alpha, newX, newF, newDF
            newX = x + alpha * p
        newDFp = float(newDF @ p)
        if newF > (f + alpha * c1dfp) or newF >= aloF:
            ahi, ahiF, ahiDFp = alpha, newF, newDFp
        else:
            if abs(newDFp) <= -c2dfp:
                break
            if newDFp * (ahi - alo) >= 0:
                ahi, ahiF, ahiDFp = alo, aloF, aloDFp
            alo, aloF, aloDFp = alpha, newF, newDFp
    return 0, alpha, newX, newF, newDF


def _wolfe_line_search(func, alpha, p, x0, f0, g0, c1, c2, min_alpha, max_ls_its, max_ls_restarts):
    """bfgs_linesearch.hpp WolfeLineSearch.  Returns (ret, alpha, x1, f1, g1)."""
    dfp = float(g0 @ p)
    c1dfp, c2dfp = c1 * dfp, c2 * dfp
    alpha0 = min_alpha
    prevF, prevDFp = f0, dfp
    nits = 0
    ls_restarts = 0
    x1, f1, g1 = x0, f0, g0
    while True:
        if nits >= max_ls_its:
            return 1, alpha, x1, f1, g1
        x1 = x0 + alpha * p
        err, f1, g1 = func(x1)
        if err:
            if ls_restarts >= max_ls_restarts:
                return 1, alpha, x1, f1, g1
            alpha = 0.5 * (alpha0 + alpha)
            ls_restarts += 1
            continue
        ls_restarts = 0
        newDFp = float(g1 @ p)
        if f1 > f0 + alpha * c1dfp or (f1 >= prevF and nits > 0):
            ret, alpha, x1, f1, g1 = _wolfe_zoom(func, x0, f0, dfp, c1dfp, c2dfp, p,
                                                 alpha0, prevF, prevDFp, alpha, f1, newDFp, 1e-16)
            return ret, alpha, x1, f1, g1
        if abs(newDFp) <= -c2dfp:
            return 0, alpha, x1, f1, g1
        if newDFp >= 0:
            ret, alpha, x1, f1, g1 = _wolfe_zoom(func, x0, f0, dfp, c1dfp, c2dfp, p,
                                                 alpha, f1, newDFp, alpha0, prevF, prevDFp, 1e-16)
            return ret, alpha, x1, f1, g1
        alpha0, prevF, prevDFp = alpha, f1, newDFp
        alpha *= 10.0
        nits += 1


def stan_lbfgs(fun, x0: np.ndarray, opts: ProphetOptions, trace: Optional[list] = None,
               crit: Optional[list] = None):
    """stan::optimization::BFGSMinimizer<…, LBFGSUpdate>::initialize + step loop as
    driven by stan::services::optimize::lbfgs.  ``fun(x) -> (err, f, g)`` minimised.

    Returns (x, f, iters, ret, n_evals).  ret < 0 is what PyStan turns into the
    RuntimeError fbprophet 0.5 answers with a Newton retry.  ``trace`` (a list) receives one
    ``(iteration, f_k, alpha_k, n_evals)`` tuple per accepted iteration -- the record the GPU
    kernel's trajectory hook (pb200_fit_trace_host) writes, compared in tests/test_gpu_trajectory.py.
    ``crit`` (a list) receives, per accepted iteration, what the convergence tests compare with their
    tolerances: ``(iteration, |f_{k-1} - f_k|, max(|f_{k-1}|, |f_k|, 1), ||g_k||, |g_k . p_k|,
    max(|f_k|, 1), ||s_k||)`` (tests/test_gpu_stop_rules.py).
    """
    func = _Counter(fun)
    c1, c2, min_alpha, max_ls_its, max_ls_restarts = 1e-4, 0.9, 1e-12, 20, 10
    xk = np.array(x0, dtype=np.float64)
    err, fk, gk = func(xk)
    if err:
        raise RuntimeError("Error evaluating initial BFGS point.")
    pk = -gk
    hist: List[Tuple[float, np.ndarray, np.ndarray]] = []   # (1/s.y, y, s), oldest first
    gammak = 1.0
    it = 0
    xk_1 = fk_1 = gk_1 = pk_1 = None
    alphak_1 = alpha = 0.0
    while True:
        it += 1
        resetB = 1 if it == 1 else 0
        while True:
            if resetB:
                pk = -gk
            if it > 1 and resetB != 2:
                alpha0 = alpha = min(1.0, 1.01 * _cubic_interp(float(gk_1 @ pk_1), alphak_1, fk - fk_1,
                                                               float(gk @ pk), min_alpha, 1.0))
            else:
                alpha0 = alpha = opts.init_alpha
            ret, alpha, xn, fn, gn = _wolfe_line_search(func, alpha, pk, xk, fk, gk, c1, c2,
                                                        min_alpha, max_ls_its, max_ls_restarts)
            if ret:
                if resetB:
                    return xk, fk, it, TERM_LSFAIL, func.n
                resetB = 2
                continue
            break
        # swap: k <- newest
        xk_1, fk_1, gk_1, pk_1 = xk, fk, gk, pk
        xk, fk, gk = xn, fn, gn
        if trace is not None:
            trace.append((it, float(fk), float(alpha), func.n))
        sk = xk - xk_1
        yk = gk - gk_1
        grad_norm = float(np.linalg.norm(gk))
        step_norm = float(np.linalg.norm(sk))
        skyk = float(yk @ sk)
        if resetB:
            B0fact = float(yk @ yk) / skyk
            hist.clear()
            pk_1 = pk_1 / B0fact
            alphak_1 = alpha * B0fact
        else:
            alphak_1 = alpha
        gammak = skyk / float(yk @ yk)
        hist.append((1.0 / skyk, yk, sk))
        if len(hist) > opts.history_size:
            hist.pop(0)
        # LBFGSUpdate::search_direction (two-loop recursion)
        pk = -gk
        alphas = [0.0] * len(hist)
        for j in range(len(hist) - 1, -1, -1):
            rho, yi, si = hist[j]
            a = rho * float(si @ pk)
            pk = pk - a * yi
            alphas[j] = a
        pk = pk * gammak
        for j in range(len(hist)):
            rho, yi, si = hist[j]
            b = rho * float(yi @ pk)
            pk = pk + (alphas[j] - b) * si
        # convergence tests
        df = abs(fk_1 - fk)
        if crit is not None:
            crit.append((it, df, max(abs(fk_1), max(abs(fk), 1.0)), grad_norm, abs(float(gk @ pk)),
                         max(abs(fk), 1.0), step_norm))
        if df < opts.tol_obj:
            ret = TERM_ABSF
        elif df < opts.tol_rel_obj * EPS * max(abs(fk_1), max(abs(fk), 1.0)):
            ret = TERM_RELF
        elif grad_norm < opts.tol_grad:
            ret = TERM_ABSGRAD
        elif abs(float(gk @ pk)) < opts.tol_rel_grad * EPS * max(abs(fk), 1.0):
            # g' * Hhat^{-1} * g / max(|f|, fScale) < tolRelGrad * eps, with pk = -Hhat^{-1} g
            ret = TERM_RELGRAD
        elif step_norm < opts.tol_param:
            ret = TERM_ABSX
        elif it >= opts.max_iter:
            ret = TERM_MAXIT
        else:
            ret = TERM_SUCCESS
        if ret != TERM_SUCCESS:
            return xk, fk, it, ret, func.n


# --------------------------------------------------------------------------
# Stan Newton (fbprophet 0.5 fit(): ``except RuntimeError: model.optimizing(..., algorithm='Newton')``)
# --------------------------------------------------------------------------
NEWTON_FD_EPS = 1e-3


def _grad_hess(func, x: np.ndarray):
    """stan::model::grad_hess_log_prob<true, false>: analytic gradient plus a Hessian from 4-point
    central finite differences of GRADIENTS (perturbations -2e, -e, e, 2e with e = 1e-3,
    coefficients 1/12, -2/3, 2/3, -1/12), accumulated into rows and columns with half weight each
    (so the result is symmetric).  An evaluation that fails throws in Stan and surfaces in PyStan as
    RuntimeError -- which the reference UDF turns into a dropped series (prophet_modeler.py:81-85).

    [UPSTREAM-RECALL, unsure] Stan 2.19's source writes the increment as
    ``half_epsilon * coefficients[i] * temp_grad[dd]`` with ``half_epsilon = 0.5 * epsilon``; read
    literally that scales the Hessian by epsilon^2.  The derivative the stencil computes needs
    ``0.5 / epsilon``, which is what is used here (and in the C port and the GPU kernel).  Only the
    length of the Newton direction depends on it -- newton_step's step halving absorbs a wrong scale,
    and the iteration stops on |delta lp| < 1e-8, i.e. at the same optimum either way."""
    n = x.size
    err, f, g = func(x)
    if err:
        raise RuntimeError("grad_hess_log_prob: error evaluating the log probability")
    H = np.zeros((n, n))
    pert = (-2 * NEWTON_FD_EPS, -NEWTON_FD_EPS, NEWTON_FD_EPS, 2 * NEWTON_FD_EPS)
    coef = (1.0 / 12.0, -2.0 / 3.0, 2.0 / 3.0, -1.0 / 12.0)
    half_inv_eps = 0.5 / NEWTON_FD_EPS
    xp = x.copy()
    for d in range(n):
        for pe, co in zip(pert, coef):
            xp[d] = x[d] + pe
            e2, _, gi = func(xp)
            if e2:
                raise RuntimeError("grad_hess_log_prob: error evaluating a perturbed gradient")
            inc = half_inv_eps * co * gi
            H[d, :] += inc
            H[:, d] += inc
        xp[d] = x[d]
    return f, g, H


def _abs_hessian_solve(H: np.ndarray, g: np.ndarray) -> np.ndarray:
    """stan::optimization::make_negative_definite_and_solve, in terms of f = -lp: every eigenvalue
    of the Hessian is replaced by its absolute value before solving, u = V diag(1/|lambda|) V' g."""
    lam, V = np.linalg.eigh(H)
    with np.errstate(all="ignore"):
        return V @ ((V.T @ g) / np.abs(lam))


def stan_newton(fun, x0: np.ndarray, opts: ProphetOptions):
    """stan::services::optimize::newton + stan::optimization::newton_step (Stan 2.19), minimising
    f = -lp.  Each iteration: gradient and finite-difference Hessian at x, Newton direction with
    |H|, then step sizes 1, 1/2, 1/4, ... until f does not increase (an evaluation error counts as
    an increase; below 1e-50 the iteration returns the old point).  Stops when an iteration changes
    lp by less than 1e-8 (absolute) or after ``iter`` (fbprophet passes 1e4) iterations.  The first
    comparison in Stan is against lp computed WITH the normalising constants (log_prob<false,false>)
    while newton_step returns the propto value, so it cannot fire on iteration 1; neither does it here.

    Returns (x, f, iters, ret, n_evals) with ret = TERM_NEWTON; raises RuntimeError where Stan throws."""
    func = _Counter(fun)
    x = np.array(x0, dtype=np.float64)
    err, f, _ = func(x)
    if err:
        f = math.inf           # services::newton catches this and carries on with lp = -inf
    it = 0
    for it in range(1, opts.max_iter + 1):
        f0, g, H = _grad_hess(func, x)
        u = _abs_hessian_solve(H, g)
        step, f1, xn = 2.0, math.inf, x
        moved = False
        while True:
            step *= 0.5
            if step < 1e-50:
                break
            xn = x - step * u
            e1, f1, _ = func(xn)
            if e1 or not (f1 <= f0):
                continue
            moved = True
            break
        last = f
        if moved:
            x, f = xn, f1
        else:
            f = f0
        if it > 1 and abs(f - last) < 1e-8:
            break
    return x, float(f), it, TERM_NEWTON, func.n


# --------------------------------------------------------------------------
# fit / predict
# --------------------------------------------------------------------------
def fit(ds_ns, y, floor: float = 0.0, cap: Optional[float] = None,
        opts: Optional[ProphetOptions] = None, cap_multiplier: float = 1.1,
        algorithm: str = "LBFGS+Newton", trace: Optional[list] = None,
        crit: Optional[list] = None) -> FitResult:
    """model_time_series_udf body (prophet_modeler.py:56-66): cap = max(y)*cap_multiplier,
    then Prophet(...).fit.  ``algorithm``: "LBFGS+Newton" is fbprophet 0.5's fit() -- L-BFGS, and on
    PyStan's RuntimeError (line-search failure) a Newton run from the same initial point; "LBFGS" /
    "Newton" run one of them alone (tests).  ``trace`` / ``crit``: stan_lbfgs's records."""
    opts = opts or ProphetOptions()
    ds_ns = np.asarray(ds_ns, dtype=np.int64)
    y = np.asarray(y, dtype=np.float64)
    if cap is None:
        cap = float(np.nanmax(y)) * cap_multiplier          # prophet_modeler.py:59
    p = prepare(ds_ns, y, floor, cap, opts)
    th0 = initial_theta(p)
    if p.constant_linear_shortcut:
        th, f, it, ret, ne = th0.copy(), float("nan"), 0, TERM_SUCCESS, 0
        sigma = 1e-9
    else:
        fun = lambda x: neg_logp_grad(x, p)     # noqa: E731
        if algorithm == "Newton":
            th, f, it, ret, ne = stan_newton(fun, th0, opts)
        else:
            th, f, it, ret, ne = stan_lbfgs(fun, th0, opts, trace=trace, crit=crit)
            if ret == TERM_LSFAIL and algorithm == "LBFGS+Newton":
                th, f, it2, ret, ne2 = stan_newton(fun, th0, opts)
                it, ne = it + it2, ne + ne2
        sigma = math.exp(th[2 + p.S])
    S = p.S
    k, m, delta, beta = th[0], th[1], th[2:2 + S].copy(), th[3 + S:].copy()
    if p.n_changepoints_real == 0:
        k = k + float(delta[0])        # "Fold delta into the base rate k"
        delta = np.zeros_like(delta)
    return FitResult(prep=p, k=float(k), m=float(m), delta=delta, sigma_obs=float(sigma), beta=beta,
                     theta=th, neg_logp=float(f), iters=it, n_evals=ne, ret=ret,
                     last_ds_ns=int(np.max(ds_ns)))


def make_future_ns(last_ns: int, periods: int, freq_ns: int) -> np.ndarray:
    """Prophet.make_future_dataframe(include_history=False) for a fixed-width (Tick)
    frequency: date_range(start=last, periods+1, freq)[> last][:periods]
    (prophet_scorer.py:64-66; 'W' is mapped to a 7-day tick at :61-62)."""
    return last_ns + freq_ns * np.arange(1, periods + 1, dtype=np.int64)


def _piecewise_trend(t, cap_s, deltas, k, m, cps, logistic):
    """Prophet.piecewise_linear / piecewise_logistic."""
    deltas = np.asarray(deltas, dtype=np.float64)
    cps = np.asarray(cps, dtype=np.float64)
    if logistic:
        k_cum = np.concatenate(([k], np.cumsum(deltas) + k))
        gammas = np.zeros(len(cps))
        acc = 0.0
        with np.errstate(all="ignore"):
            for i, t_s in enumerate(cps):
                gammas[i] = (t_s - m - acc) * (1 - k_cum[i] / k_cum[i + 1])
                acc += gammas[i]
    else:
        gammas = -cps * deltas
    k_t = k * np.ones_like(t)
    m_t = m * np.ones_like(t)
    for s, t_s in enumerate(cps):
        indx = t >= t_s
        k_t[indx] += deltas[s]
        m_t[indx] += gammas[s]
    if logistic:
        with np.errstate(all="ignore"):
            return cap_s / (1 + np.exp(-k_t * (t - m_t)))
    return k_t * t + m_t


def predict(fr: FitResult, ds_ns, floor: Optional[float] = None, cap: Optional[float] = None,
            opts: Optional[ProphetOptions] = None):
    """Prophet.predict deterministic part: setup_dataframe(future) -> predict_trend ->
    predict_seasonal_components -> yhat = trend*(1+multiplicative)+additive.
    ``floor``/``cap`` are the values the scorer writes into the future frame
    (prophet_scorer.py:67-68; cap there is the float32-rounded one)."""
    opts = opts or ProphetOptions()
    p = fr.prep
    ds_ns = np.asarray(ds_ns, dtype=np.int64)
    t = (ds_ns - p.start_ns).astype(np.float64) / np.float64(p.t_scale_ns)
    if p.logistic:
        fl = p.floor if floor is None else float(floor)
        cp = p.cap_value if cap is None else float(cap)
        cap_s = np.full(t.size, (cp - fl) / p.y_scale)
    else:
        fl, cap_s = 0.0, np.zeros(t.size)
    trend = _piecewise_trend(t, cap_s, fr.delta, fr.k, fr.m, p.t_change, p.logistic) * p.y_scale + fl
    X, _, s_a, s_m = seasonal_features(ds_ns, p.seasonalities, opts)
    mult = X @ (fr.beta * s_m)
    add = (X @ (fr.beta * s_a)) * p.y_scale
    yhat = trend * (1 + mult) + add
    return {"t": t, "trend": trend, "multiplicative_terms": mult, "additive_terms": add,
            "yhat": yhat, "cap_scaled": cap_s, "floor": fl}


def scorer_epilogue(yhat: np.ndarray, floor: float) -> np.ndarray:
    """prophet_scorer.py:73-84: astype(int) truncates toward zero; values < floor -> floor."""
    yi = np.trunc(yhat).astype(np.int64)
    return np.where(yi < floor, floor, yi)


def predict_uncertainty(fr: FitResult, ds_ns, pred: dict, rng: np.random.RandomState,
                        opts: Optional[ProphetOptions] = None):
    """Prophet.predict_uncertainty -> sample_posterior_predictive -> sample_model ->
    sample_predictive_trend, 1 MAP 'iteration' x uncertainty_samples draws, then
    np.nanpercentile at 100*(1-w)/2 and 100*(1+w)/2 (linear interpolation).
    fbprophet uses the unseeded global np.random; the call ORDER per draw is kept:
    poisson, rand(n), laplace(n), then normal(T)."""
    opts = opts or ProphetOptions()
    p = fr.prep
    t = pred["t"]
    n = opts.uncertainty_samples
    Tmax = t.max()
    S = len(p.t_change)
    mult, add = pred["multiplicative_terms"], pred["additive_terms"]
    yh = np.empty((t.size, n))
    tr = np.empty((t.size, n))
    for j in range(n):
        if Tmax > 1:
            n_changes = rng.poisson(S * (Tmax - 1))
        else:
            n_changes = 0
        if n_changes > 0:
            cp_new = 1 + rng.rand(n_changes) * (Tmax - 1)
            cp_new.sort()
        else:
            cp_new = np.zeros(0)
        lam = np.mean(np.abs(fr.delta)) + 1e-8
        d_new = rng.laplace(0, lam, n_changes)
        cps = np.concatenate((p.t_change, cp_new))
        ds_ = np.concatenate((fr.delta, d_new))
        trend = _piecewise_trend(t, pred["cap_scaled"], ds_, fr.k, fr.m, cps, p.logistic) * p.y_scale + pred["floor"]
        noise = rng.normal(0, fr.sigma_obs, t.size) * p.y_scale
        yh[:, j] = trend * (1 + mult) + add + noise
        tr[:, j] = trend
    lower_p = 100 * (1.0 - opts.interval_width) / 2
    upper_p = 100 * (1.0 + opts.interval_width) / 2
    return {"yhat_lower": np.nanpercentile(yh, lower_p, axis=1),
            "yhat_upper": np.nanpercentile(yh, upper_p, axis=1),
            "trend_lower": np.nanpercentile(tr, lower_p, axis=1),
            "trend_upper": np.nanpercentile(tr, upper_p, axis=1)}
