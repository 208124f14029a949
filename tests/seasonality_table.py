"""fbprophet's seasonality table on top of the numpy oracle (DESIGN §18): custom seasonalities (add_seasonality) and
built-in Fourier orders, in fbprophet's column order -- custom entries as added, then yearly, weekly, daily -- with a
prior scale per column (Stan's ``sigmas``).  Test reference only.

Two sets of Fourier columns (``columns``):

* ``"numpy"``: fbprophet's own, ``sin / cos(2.0 * (i + 1) * np.pi * t / period)`` with every harmonic's argument rounded
  on its own -- about ulp(arg) / 2 off the angle, more than 1e-9 at harmonic 32 of a 6-hour period on 2021 dates;
* ``"exact"``: what the table fit kernel computes.  fit_table.cu stages one base angle per seasonality,
  theta = fl(fl(2 pi) t / period), and builds harmonic h from it by the three-term recurrence, which follows
  sin / cos(h theta) far more closely than numpy's columns do.  Here h theta is formed exactly in extended precision
  and its sin / cos rounded to double.  The fit kernel is held to this reference; the predict kernels, which evaluate numpy's arguments, and the MC
  consumers to ``"numpy"``.
"""
import numpy as np

from oracle import prophet_oracle as po

NS_PER_DAY = 86400 * 10**9
BUILTINS = (("yearly", 365.25, 10), ("weekly", 7.0, 3), ("daily", 1.0, 4))
COLUMNS = ("numpy", "exact")
TWO_PI_FL = 2.0 * 3.141592653589793     # fl(2 pi), as fit_kernel.cuh stages it

# h * theta is exact in np.longdouble when its significand holds theta's 53 bits times h: x87 extended precision (64
# bits) does for h < 2^11.  A host without it needs a double-double form of h * theta, not a silent float64 fall-back.
_LD_BITS = np.finfo(np.longdouble).nmant + 1


def tau_days(ds_ns) -> np.ndarray:
    """Days since 1970 as pandas 0.25's total_seconds / 86400, fbprophet's t of fourier_series."""
    return (1e-9 * np.asarray(ds_ns, np.int64).astype(np.float64)) / 86400.0


def base_angle(ds_ns, period: float) -> np.ndarray:
    """The base angle the table fit kernel stages per point, fl(fl(2 pi) tau / period), in float64."""
    return TWO_PI_FL * tau_days(ds_ns) / float(period)


def fourier_columns(ds_ns, period: float, order: int, columns: str = "numpy") -> np.ndarray:
    """[T, 2 order] sin, cos per harmonic, as Prophet.fourier_series orders them; ``columns`` as the module says."""
    if columns == "numpy":
        return po.fourier_series(np.asarray(ds_ns, np.int64), period, order)
    if columns != "exact":
        raise ValueError(f"columns must be one of {COLUMNS} (got {columns!r})")
    assert np.finfo(np.longdouble).nmant >= 63, "np.longdouble is not x87 extended precision: h * theta is not exact"
    assert order < 2 ** (_LD_BITS - 53), order
    th = base_angle(ds_ns, period).astype(np.longdouble)
    arg = th[:, None] * np.arange(1, order + 1, dtype=np.longdouble)[None, :]
    out = np.empty((th.size, 2 * order))
    out[:, 0::2] = np.sin(arg).astype(np.float64)
    out[:, 1::2] = np.cos(arg).astype(np.float64)
    return out


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


def table_entries(builtin, custom):
    """[(name, period, order)] of the whole table as the library normalises it: the custom entries, then each built-in
    not replaced by one and not switched off, at its order ('auto' and True: the default).  A history's table mask has
    bit j set when entry j is among its ``seasonalities``."""
    out = [(c["name"], float(c["period"]), int(c["fourier_order"])) for c in custom]
    names = {c["name"] for c in custom}
    for name, period, order in BUILTINS:
        arg = builtin.get(name, "auto")
        if name in names or arg is False or (not isinstance(arg, str) and arg is not True and int(arg) == 0):
            continue
        out.append((name, period, order if isinstance(arg, str) or arg is True else int(arg)))
    return out


def table_mask(seas, entries) -> int:
    """The table mask of a history's ``seasonalities`` within the table's ``entries``."""
    on = {s[0] for s in seas}
    return sum(1 << j for j, e in enumerate(entries) if e[0] in on)


def prepare(ds_ns, y, floor, cap, opts: po.ProphetOptions, builtin, custom, columns: str = "numpy"):
    """po.prepare with the table's Fourier columns (``columns``: "numpy" or "exact") and per-column prior scales."""
    p = po.prepare(ds_ns, y, floor, cap, opts)
    seas = seasonalities(p.ds_sorted, builtin, custom, opts.seasonality_prior_scale)
    p.seasonalities = [po.Seasonality(n, per, o) for n, per, o, _ in seas]
    X, _, s_a, s_m = po.seasonal_features(p.ds_sorted, p.seasonalities, opts)
    if columns != "numpy" and seas:
        X = np.column_stack([fourier_columns(p.ds_sorted, per, o, columns) for _, per, o, _ in seas])
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


def table_seasonal(opts, columns: str = "numpy"):
    """oracle/mc_stream's seasonal term for a table model of options ``opts`` (a pb200_options_v2): the active entries
    of the table mask in table order, their betas packed from column 0.  predict_kernel.cuh seasonal_term evaluates
    numpy's arguments, so the MC consumers are held to ``"numpy"``."""
    ents = [(opts.seasonalities[i].period, opts.seasonalities[i].fourier_order) for i in range(opts.n_seasonalities)]
    names = {opts.seasonalities[i].name.decode() for i in range(opts.n_seasonalities)}
    for (name, period, order), sw, o in zip(BUILTINS, (opts.yearly, opts.weekly, opts.daily),
                                            (opts.yearly_order, opts.weekly_order, opts.daily_order)):
        if sw != 0 and name not in names:
            ents.append((period, o or order))

    def seasonal(ds_ns, mask, beta):
        acc, col = np.zeros(np.asarray(ds_ns).size), 0
        for e, (period, order) in enumerate(ents):
            if (mask >> e) & 1:
                X = fourier_columns(ds_ns, period, order, columns)
                blk = np.zeros(acc.size)
                for i in range(order):
                    blk = blk + X[:, 2 * i] * beta[col + 2 * i] + X[:, 2 * i + 1] * beta[col + 2 * i + 1]
                acc = acc + blk
                col += 2 * order
        return acc
    return seasonal
