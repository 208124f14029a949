"""Helpers the GPU fit tests share: contexts built under the environment switches pb200_create reads, start points near
the oracle's initial one, the oracle's per-iteration record, the trajectory comparison, and a host mirror of the grouped
kernel's chunk rule.  TEST INFRASTRUCTURE ONLY."""
import dataclasses
import os

import numpy as np

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L


def ctx_with_env(**env):
    """A context created while ``env`` is set (the switches are read once, at pb200_create)."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return L.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def grp_chunk(T, P, G, U=2):
    """Host mirror of fit_kernel.cuh grp_chunk: the grouped kernel's points per lane, -1 when no chunk keeps the bins of
    one step apart (the series then leaves the grouped kernel)."""
    c0 = (T + G - 1) // G
    for c in range(c0, c0 + 25):
        if all(U - 1 < (c * dl) % P < P - (U - 1) for dl in range(1, G)):
            return c
    return -1


def thetas(b, oopts, lay, rng, steep=False):
    """Per series of RaggedBatch ``b``: a point near the oracle's initial_theta, zero-padded to the layout's pstride, and
    the oracle's Prepared.  Returns ``(rows, [(prepared, theta)])``."""
    rows, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        if steep:
            # a steep falling logistic trend: k (t - m) = -520 t stays inside +-600 on the series' own t in [0, 1], so the
            # kernel takes its exp-ratio recurrence; past t ~ 1.36 exp(520 t) overflows a double
            th[0], th[1], th[2:2 + p.S] = -520.0, 0.0, 0.0
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        rows.append(row)
        preps.append((p, th))
    return np.array(rows), preps


def oracle_rows(ds, y, oopts):
    """The oracle's L-BFGS fit and its per-iteration record ``(iteration, f_k, alpha_k, n_evals)``."""
    rows = []
    fr = po.fit(ds, y, opts=oopts, algorithm="LBFGS", trace=rows)
    return fr, np.array(rows).reshape(-1, 4)


def assert_trajectory_head(tr, n_gpu, rows, what, n_head=6):
    """The first accepted iterations against the oracle, at the tolerances of test_lbfgs_trajectory_matches_oracle."""
    head = min(n_gpu, len(rows), n_head)
    assert head >= 1, what
    g, o = tr[:head], rows[:head]
    assert np.array_equal(g[:, 0], np.arange(1, head + 1)), what
    assert np.array_equal(g[:, 3], o[:, 3]), (what, g[:, 3], o[:, 3])
    df = np.abs(g[:, 1] - o[:, 1]) / np.maximum(1.0, np.abs(o[:, 1]))
    assert np.all(df <= 1e-11), (what, df)
    da = np.abs(g[:, 2] - o[:, 2]) / np.abs(o[:, 2])
    assert np.all(da <= 1e-7), (what, da)


# ---------------------------------------------------------------------------------------------------------------------
# fbprophet's Newton run held per iteration (tests/test_newton_steps.py, tests/test_wide_params.py)
# ---------------------------------------------------------------------------------------------------------------------
def seasonal_k(mask):
    """Fourier columns of a seasonality mask (yearly 20 | weekly 6 | daily 8), fbprophet's one zero column without any."""
    k = 20 * bool(mask & 1) + 6 * bool(mask & 2) + 8 * bool(mask & 4)
    return k if k else 1


def record_theta(fb, i):
    """Row i of a fitted batch as Stan's unconstrained point (k, m, delta[S], log sigma_obs, beta[K]), in the record's
    folded form: without changepoints (n_cp_real 0) k holds k + delta[0] and delta is zero, and the single zero column of a
    history without seasonality is recorded as 0."""
    mi, p = fb.meta_i32[i], fb.params[i]
    S, K = int(mi[1]), seasonal_k(int(mi[3]))
    return np.concatenate(([p[0], p[1]], p[3:3 + S], [np.log(p[2])], p[3 + fb.smax:3 + fb.smax + K]))


def folded(theta, S, ncp, mask):
    """An oracle's unconstrained point in record_theta's form."""
    th = np.array(theta, dtype=np.float64)
    if ncp == 0:
        th[0] += th[2]
        th[2:2 + S] = 0.0
    if mask == 0:
        th[3 + S:] = 0.0
    return th


def c_newton_opts(growth, mode, extra, n_changepoints, max_iter):
    """The C oracle's options for fbprophet's Newton run alone (``extra``: the Prophet seasonality switches)."""
    from oracle import c_oracle as co
    sw = {True: 1, False: 0}
    o = co.options(growth=growth, seasonality_mode=mode, yearly=sw.get(extra.get("yearly_seasonality"), -1),
                   weekly=sw.get(extra.get("weekly_seasonality"), -1), daily=sw.get(extra.get("daily_seasonality"), -1))
    o.n_changepoints = n_changepoints
    o.max_iter = max_iter
    o.algorithm = co.ALG_NEWTON
    return o


def newton_bound(gpu, ref, other, scale, floor=1e-10):
    """|gpu - ref|, and the bound it is held to: ten times the two CPU oracles' disagreement |other - ref| plus a floor of
    ``floor`` of the quantity's size (max norm over a vector)."""
    d = float(np.max(np.abs(np.asarray(gpu) - ref)))
    return d, 10.0 * float(np.max(np.abs(np.asarray(other) - ref))) + floor * max(1.0, float(np.max(np.abs(scale))))


def assert_newton_row(fb, i, fr, c_theta, c_f, c_info, measured, what):
    """Row i of a Newton fit against the numpy oracle's FitResult ``fr`` and the C oracle's (theta, f, info) row: status
    60, iteration and evaluation counts equal to both, changepoints exact, theta and objective within newton_bound."""
    p = fr.prep
    S, P, mask = p.S, p.S + p.K + 3, sum({"yearly": 1, "weekly": 2, "daily": 4}[s.name] for s in p.seasonalities)
    mi = fb.meta_i32[i]
    assert (int(mi[0]), int(mi[1]), int(mi[3])) == (p.T, S, mask), (what, mi)
    assert mi[4] == 60 == fr.ret == c_info[0], (what, mi, fr.ret, c_info)
    assert (mi[5], mi[6]) == (fr.iters, fr.n_evals) == (c_info[1], c_info[2]), (what, mi, fr.iters, fr.n_evals, c_info)
    assert np.array_equal(fb.tchange[i, :S], p.t_change) and np.all(fb.tchange[i, S:] == 0.0), what
    # the objective's floor is 1e-8: away from the optimum f moves with g . dtheta, and the two oracles' objectives can
    # agree far more closely than their theta does (GPU measured up to 5.3e-9 relative where numpy and C are 1e-10 apart)
    df, bf = newton_bound(fb.meta_f64[i, 3], fr.neg_logp, c_f, fr.neg_logp, floor=1e-8)
    th_np = folded(fr.theta, S, p.n_changepoints_real, mask)
    th_c = folded(c_theta[:P], S, p.n_changepoints_real, mask)
    # theta's floor is 1e-10, and 1e-7 on yearly + weekly + daily series: their Hessian is ill-conditioned along the
    # Laplace kinks, the two oracles' theta spread there to 2.4e-7, and they can happen to agree much more closely
    # (GPU measured 3.8e-8 at P = 65 after five iterations where numpy and C were 6e-10 apart)
    dt, bt = newton_bound(record_theta(fb, i), th_np, th_c, th_np, floor=1e-7 if mask == 7 else 1e-10)
    measured["f"] = max(measured.get("f", 0.0), df / bf)
    measured["theta"] = max(measured.get("theta", 0.0), dt / bt)
    assert df <= bf, (what, fb.meta_f64[i, 3], fr.neg_logp, c_f)
    assert dt <= bt, (what, dt, bt, np.abs(record_theta(fb, i) - th_np))


# ---------------------------------------------------------------------------------------------------------------------
# Stan's L-BFGS stop rules bracketed through the status alone (tests/test_stop_rules_oracle.py,
# tests/test_gpu_stop_rules.py): run with max_iter = j, every other tolerance 0 and one rule's tolerance just above (just
# below) the oracle's value at iteration j, a fit must end with that rule's status (with MAXIT) at iteration j
# ---------------------------------------------------------------------------------------------------------------------
EPS = 2.220446049250313e-16
RULES = ("ABSF", "RELF", "ABSGRAD", "RELGRAD", "ABSX")            # the order BFGSMinimizer::step tests them in
RULE_TOL = dict(zip(RULES, ("tol_obj", "tol_rel_obj", "tol_grad", "tol_rel_grad", "tol_param")))
RULE_STATUS = dict(zip(RULES, (po.TERM_ABSF, po.TERM_RELF, po.TERM_ABSGRAD, po.TERM_RELGRAD, po.TERM_ABSX)))
ZERO_TOLS = {t: 0.0 for t in RULE_TOL.values()}
RECORD_MARGIN = 1.01          # a target's earlier values are all at least 1 % above its own


class StopRun:
    """The oracle's L-BFGS run with every tolerance 0: its trace rows ``(iteration, f_k, alpha_k, n_evals)``, the fit,
    and per rule the value each accepted iteration compares with the rule's tolerance."""

    def __init__(self, ds, y, oopts, max_iter=12, history=5, init=None):
        import warm_oracle as wo
        o = dataclasses.replace(oopts, max_iter=max_iter, history_size=history, **ZERO_TOLS)
        rows, crit = [], []
        self.fr = wo.fit(ds, np.asarray(y, np.float64), opts=o, algorithm="LBFGS", trace=rows, crit=crit, init=init)
        self.rows = np.array(rows).reshape(-1, 4)
        self.crit = np.array(crit).reshape(-1, 7)
        c = self.crit
        self.values = {"ABSF": c[:, 1], "RELF": c[:, 1] / (EPS * c[:, 2]), "ABSGRAD": c[:, 3],
                       "RELGRAD": c[:, 4] / (EPS * c[:, 5]), "ABSX": c[:, 6]}
        self.history = history

    def f(self, j):
        """f_j; f_0 is the start point's objective (each accepted step lowers f, so f_{j-1} = f_j + df_j)."""
        return self.rows[j - 1, 1] if j >= 1 else self.rows[0, 1] + self.crit[0, 1]

    def record_lows(self, rule):
        """The iterations j whose value of ``rule`` every earlier one exceeds by RECORD_MARGIN."""
        v = self.values[rule]
        return [j for j in range(1, v.size + 1) if np.isfinite(v[j - 1]) and v[j - 1] > 0
                and np.all(v[:j - 1] >= RECORD_MARGIN * v[j - 1])]

    def targets(self, rule):
        """Iteration 1 (the reset path), 2 when it is a record low, and the last record low past the history size (the
        ring buffer has wrapped)."""
        lows = self.record_lows(rule)
        out = [j for j in lows if j <= 2]
        past = [j for j in lows if j > self.history]
        return out + past[-1:]

    def delta(self, rule, j):
        """The bracket's half width: 1e-6, and for the rules on df, 1e-9 |f_j| / df_j (df is the difference of two
        values each exact to about 1e-11 relative)."""
        if rule in ("ABSF", "RELF"):
            return max(1e-6, 1e-9 * abs(self.rows[j - 1, 1]) / self.crit[j - 1, 1])
        return 1e-6

    def bracket(self, rule, j, side, delta):
        """(tolerances, expected (status, iters, n_evals)) of the run with max_iter j and ``rule``'s tolerance at
        v_j (1 + side delta)."""
        tols = dict(ZERO_TOLS)
        tols[RULE_TOL[rule]] = float(self.values[rule][j - 1] * (1.0 + side * delta))
        want = (RULE_STATUS[rule] if side > 0 else po.TERM_MAXIT, j, int(self.rows[j - 1, 3]))
        return tols, want
