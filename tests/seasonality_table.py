"""fbprophet's seasonality table on top of the numpy oracle (DESIGN §18): custom seasonalities (add_seasonality) and
built-in Fourier orders, in fbprophet's column order -- custom entries as added, then yearly, weekly, daily -- with a
prior scale per column (Stan's ``sigmas``).  Test reference only."""
import numpy as np

from oracle import prophet_oracle as po

NS_PER_DAY = 86400 * 10**9
BUILTINS = (("yearly", 365.25, 10), ("weekly", 7.0, 3), ("daily", 1.0, 4))


def seasonalities(ds_sorted, builtin, custom, prior_scale):
    """[(name, period, order, prior_scale)] of one history.  ``builtin``: {name: 'auto' | True | False | int order};
    ``custom``: dicts {name, period, fourier_order, prior_scale?} in the order they were added.  An 'auto' built-in
    follows set_auto_seasonalities' rules at its default order; a custom entry of the same name replaces it."""
    first, last = int(ds_sorted[0]), int(ds_sorted[-1])
    span = last - first
    dt = np.diff(ds_sorted)
    nz = dt[dt != 0]
    min_dt = int(nz.min()) if nz.size else None
    disable = {"yearly": span < 730 * NS_PER_DAY,
               "weekly": span < 14 * NS_PER_DAY or (min_dt is not None and min_dt >= 7 * NS_PER_DAY),
               "daily": span < 2 * NS_PER_DAY or (min_dt is not None and min_dt >= NS_PER_DAY)}
    out = [(c["name"], float(c["period"]), int(c["fourier_order"]), float(c.get("prior_scale") or prior_scale))
           for c in custom]
    names = {c["name"] for c in custom}
    for name, period, order in BUILTINS:
        arg = builtin.get(name, "auto")
        if name in names:
            continue
        fo = po._parse_seasonality_arg(arg, disable[name], order)
        if fo > 0:
            out.append((name, period, fo, prior_scale))
    return out


def prepare(ds_ns, y, floor, cap, opts: po.ProphetOptions, builtin, custom):
    """po.prepare with the table's Fourier columns and per-column prior scales."""
    p = po.prepare(ds_ns, y, floor, cap, opts)
    seas = seasonalities(p.ds_sorted, builtin, custom, opts.seasonality_prior_scale)
    p.seasonalities = [po.Seasonality(n, per, o) for n, per, o, _ in seas]
    X, _, s_a, s_m = po.seasonal_features(p.ds_sorted, p.seasonalities, opts)
    p.X, p.s_a, p.s_m, p.K = X, s_a, s_m, X.shape[1]
    p.sigmas = np.array([ps for _, _, o, ps in seas for _ in range(2 * o)]) if seas else np.array([1.0])
    return p, seas


def fit(p: po.Prepared, opts: po.ProphetOptions, trace=None) -> po.FitResult:
    """po.fit's L-BFGS on a prepared table model (no Newton retry)."""
    th0 = po.initial_theta(p)
    th, f, it, ret, ne = po.stan_lbfgs(lambda x: po.neg_logp_grad(x, p), th0, opts, trace=trace)
    S = p.S
    k, m, delta, beta = th[0], th[1], th[2:2 + S].copy(), th[3 + S:].copy()
    if p.n_changepoints_real == 0:
        k = k + float(delta[0])
        delta = np.zeros_like(delta)
    return po.FitResult(prep=p, k=float(k), m=float(m), delta=delta, sigma_obs=float(np.exp(th[2 + S])), beta=beta,
                        theta=th, neg_logp=float(f), iters=it, n_evals=ne, ret=ret, last_ds_ns=int(np.max(p.ds_sorted)))
