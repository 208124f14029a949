"""fbprophet's extra regressors on top of the seasonality-table oracle (DESIGN §19): the standardised regressor columns
appended to the table's Fourier columns, in the order they were added, with their own prior scales and the model's
mode.  Test reference only.

fbprophet's make_all_seasonality_features puts the regressors after the seasonalities; its single zero column appears
only when there is no column at all, so a history with every seasonality off and R regressors has K = R.
"""
import numpy as np

from oracle import prophet_oracle as po

import seasonality_table as st


def prior_scales(opts) -> np.ndarray:
    """[R] prior scale of each regressor of a pb200_options_v3: its own, or holidays_prior_scale when 0."""
    return np.array([opts.regressors[r].prior_scale or opts.holidays_prior_scale for r in range(opts.n_regressors)])


def standardise(reg, scale) -> np.ndarray:
    """[T, R] columns (x - mu) / std of a series' values ``reg`` [R, T] under its ``scale`` [R, 2]."""
    reg = np.asarray(reg, np.float64).reshape(len(scale), -1)
    return ((reg - scale[:, 0][:, None]) / scale[:, 1][:, None]).T


def prepare(ds_ns, y, floor, cap, opts: po.ProphetOptions, builtin, custom, reg, scale, priors, columns="numpy"):
    """st.prepare with the R regressor columns appended: ``reg`` [R, T] the series' values in row order, ``scale``
    [R, 2] its (mu, std), ``priors`` [R] the regressors' prior scales.  Returns (prepared, seasonalities)."""
    p, seas = st.prepare(ds_ns, y, floor, cap, opts, builtin, custom, columns)
    Z = standardise(reg, scale)
    R = Z.shape[1]
    add = np.zeros(R) if opts.seasonality_mode == "multiplicative" else np.ones(R)
    if seas:
        p.X = np.column_stack([p.X, Z])
        p.sigmas = np.concatenate([p.sigmas, priors])
        p.s_a, p.s_m = np.concatenate([p.s_a, add]), np.concatenate([p.s_m, 1.0 - add])
    else:
        p.X, p.sigmas, p.s_a, p.s_m = Z, np.asarray(priors, np.float64), add, 1.0 - add
    p.K = p.X.shape[1]
    return p, seas


def predict_yhat(fr: po.FitResult, seas, ds_ns, floor, cap, opts: po.ProphetOptions, freg, scale) -> np.ndarray:
    """Prophet.predict's yhat of a fitted regressor model at ``ds_ns`` with future values ``freg`` [R, H]."""
    p = fr.prep
    t = (np.asarray(ds_ns, np.int64) - p.start_ns).astype(np.float64) / np.float64(p.t_scale_ns)
    fl = float(floor) if p.logistic else 0.0
    cap_s = np.full(t.size, (float(cap) - fl) / p.y_scale) if p.logistic else np.zeros(t.size)
    trend = po._piecewise_trend(t, cap_s, fr.delta, fr.k, fr.m, p.t_change, p.logistic) * p.y_scale + fl
    blocks = [st.fourier_columns(ds_ns, per, o) for _, per, o, _ in seas]
    X = np.column_stack(blocks + [standardise(freg, scale)])
    term = X @ fr.beta
    if opts.seasonality_mode == "multiplicative":
        return trend * (1 + term)
    return trend + term * p.y_scale


def mc_seasonal(opts, freg, scale):
    """oracle/mc_stream's seasonal term for one model of a regressor model: the table's term (st.table_seasonal) plus
    sum_r beta[K_seas + r] (x_r - mu_r) / std_r, as mc_kernel stages it per point; ``freg`` [R, H] that model's future
    values, ``scale`` [R, 2] its standardisation."""
    table = st.table_seasonal(opts, "numpy")
    ents = [opts.seasonalities[i].fourier_order for i in range(opts.n_seasonalities)]
    names = {opts.seasonalities[i].name.decode() for i in range(opts.n_seasonalities)}
    for (name, _, order), sw, o in zip(st.BUILTINS, (opts.yearly, opts.weekly, opts.daily),
                                       (opts.yearly_order, opts.weekly_order, opts.daily_order)):
        if sw != 0 and name not in names:
            ents.append(o or order)
    Z = standardise(freg, scale)

    def seasonal(ds_ns, mask, beta):
        k = sum(2 * o for e, o in enumerate(ents) if (mask >> e) & 1)
        acc = table(ds_ns, mask, beta)
        reg = np.zeros(acc.size)
        for r in range(Z.shape[1]):
            reg = reg + beta[k + r] * Z[:, r]
        return acc + reg
    return seasonal
