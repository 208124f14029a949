"""newton_kernel.cuh held to the oracles per iteration (the GPU tests run with -m gpu on an H100).

fbprophet 0.5 retries a series whose L-BFGS run ends in a line-search failure with Stan's Newton optimiser.  The kernel
that does it shares nothing with the fit kernels (its own objective, stan_init and set_changepoints, a finite-difference
Hessian over 16 warps, cyclic Jacobi, step halving), so it is checked on its own, after max_iter = 1, 2, 3 and 5
iterations, against both CPU restatements: numpy's stan_newton (LAPACK eigh) and C's po_newton (Jacobi).  Per series:

  * status 60, and iteration and evaluation counts equal to both oracles.  The evaluation count is
    1 + sum over iterations of (1 + 4 P + halvings), so it pins every step-halving decision;
  * changepoint times exact;
  * theta within ten times the two oracles' own disagreement plus 1e-10 of its size (1e-7 on yearly + weekly + daily
    series), the objective the same with a floor of 1e-8 (fit_oracle.newton_bound).  The oracles agree to ~5e-10 in objective, and in theta to ~1e-10 at P = 29
    and ~1e-8 .. 1e-7 on yearly + weekly + daily series, where the Hessian is ill-conditioned along the Laplace prior's
    kinks.

The matrix: both growths and seasonality modes over masks 0..7 on regular and irregular grids, T = 13 and 33 (lanes that
own no point; every changepoint on a lane's first point) and a longer series with one there too, n_changepoints 0 and 1,
P = 64 .. 67 (mask 7 with 27 .. 30 changepoints), y as int32 / float32 / float64, warm start points, and the error path.
"""
import dataclasses
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import fit_oracle as fo  # noqa: E402
import test_kernel_instances as ki  # noqa: E402
import warm_oracle  # noqa: E402
from oracle import c_oracle as co
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

STEPS = (1, 2, 3, 5)
GROWTHS = ("linear", "logistic")
_measured = {}


def _cp_on_lane_start_T(mask=0, lo=100):
    """The first T >= lo of the mask's regular recipe with a changepoint on the first point of a lane's chunk (chunk >= 3)."""
    for T in range(lo, lo + 400):
        s = ki._series(mask, T, True, 5)
        if s is None:
            continue
        chunk = -(-T // 32)
        idx = po.changepoint_indexes(T, po.ProphetOptions())
        if chunk >= 3 and any(i > 0 and i % chunk == 0 for i in idx):
            return T
    raise AssertionError("no such length")


def _recipe_series(mask, seed):
    step, span = ki.RECIPES[mask][:2]
    return ki._series(mask, span // step + 1, True, seed, step)


def batches():
    """name -> (Prophet option overrides, [(ds, y)]): the series of the matrix, grouped by the options they need."""
    out = {}
    s = [_recipe_series(m, 30 + m) for m in (0, 1, 2, 3, 4, 6, 7)]
    s += [ki._series(m, 45, False, 40 + m) for m in (1, 2, 3, 4, 6, 7)]
    s += [ki._series(0, 13, True, 50), ki._series(0, 33, True, 51), ki._series(0, _cp_on_lane_start_T(), True, 52)]
    out["masks"] = ({}, s)
    out["mask5"] = (ki.RECIPES[5][4], [_recipe_series(5, 35), ki._series(5, 45, False, 45)])
    for ncp in (0, 1):
        out[f"ncp{ncp}"] = ({"n_changepoints": ncp}, [_recipe_series(3, 60 + ncp), ki._series(6, 45, False, 62 + ncp),
                                                       ki._series(0, 33, True, 64 + ncp)])
    for ncp in (27, 28, 29, 30):         # P = 64 .. 67
        out[f"p{ncp + 37}"] = ({"n_changepoints": ncp}, [ki._series(7, 801, False, 70 + ncp)])
    return out


def _oracles(b, growth, mode, extra, k):
    """The numpy oracle's FitResult per series and the C oracle's (theta, f, info) rows, both Newton alone for k iterations."""
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, max_iter=k, **extra)
    frs = [po.fit(b.ds[b.offsets[i]:b.offsets[i + 1]], b.y[b.offsets[i]:b.offsets[i + 1]].astype(np.float64), opts=oopts,
                  algorithm="Newton") for i in range(b.n)]
    ncp = extra.get("n_changepoints", 25)
    copts = fo.c_newton_opts(growth, mode, extra, ncp, k)
    th, f, info = co.fit_batch(b.ds, b.y.astype(np.float64), b.offsets, 0.0, 1.1, copts)
    return frs, th, f, info


@pytest.fixture(scope="module", autouse=True)
def _report_measured_ratios():
    yield
    if _measured:
        print("\n[newton steps] largest |GPU - numpy| / (10 |C - numpy| + floor max(1, |numpy|)): "
              + ", ".join(f"{k} {v:.3e}" for k, v in sorted(_measured.items())) + " (bound 1)")


# ---------------------------------------------------------------------------------------------------------------------
# no GPU: the matrix is what it claims, and the two oracles the bound rests on agree per iteration
# ---------------------------------------------------------------------------------------------------------------------
def test_matrix_covers_its_edges():
    bs = batches()
    seen = set()
    for name, (extra, series) in bs.items():
        oopts = po.ProphetOptions(**extra)
        for ds, y in series:
            p = po.prepare(ds, y.astype(np.float64), 0.0, 1.1 * y.max(), oopts)
            mask = ki._oracle_mask(p)
            seen.add(("mask", mask, ki._is_regular(ds)))
            seen.add(("P", p.S + p.K + 3))
            seen.add(("ncp", p.n_changepoints_real))
            chunk = -(-p.T // 32)
            seen.add(("T", p.T))
            if p.n_changepoints_real and any(i > 0 and i % chunk == 0 and chunk >= 3
                                             for i in po.changepoint_indexes(p.T, oopts)):
                seen.add("cp on a lane's first point")
    assert {("mask", m, True) for m in range(8)} <= seen
    assert {("mask", m, False) for m in range(1, 8)} <= seen
    assert {("P", P) for P in (64, 65, 66, 67)} <= seen and any(s[0] == "P" and s[1] < 32 for s in seen if s[0] == "P")
    assert {("ncp", 0), ("ncp", 1), ("T", 13), ("T", 33), "cp on a lane's first point"} <= seen


@pytest.mark.parametrize("k", (1, 3))
def test_numpy_and_c_newton_agree_per_iteration(k):
    """The calibration the GPU bound rests on, on P = 29 (no seasonality), 42 (weekly + daily) and 67 (yearly + weekly +
    daily, 30 changepoints): identical iteration and evaluation counts, objective within 5e-10 and theta within 1e-9 /
    1e-6 relative of each other."""
    cases = [({}, ki._series(0, 97, True, 3)), ({}, ki._series(6, 200, False, 4)),
             ({"n_changepoints": 30}, ki._series(7, 801, False, 100))]
    for extra, s in cases:
        b = ki._ragged([s])
        frs, th, f, info = _oracles(b, "logistic", "multiplicative", extra, k)
        fr, p = frs[0], frs[0].prep
        P = p.S + p.K + 3
        assert P in (29, 42, 67)
        assert (fr.ret, fr.iters, fr.n_evals) == (info[0, 0], info[0, 1], info[0, 2]), (P, fr.iters, fr.n_evals, info[0])
        assert abs(fr.neg_logp - f[0]) <= 5e-10 * max(1.0, abs(fr.neg_logp)), (P, fr.neg_logp, f[0])
        d = np.max(np.abs(fr.theta - th[0, :P])) / max(1.0, np.max(np.abs(fr.theta)))
        assert d <= (1e-9 if P < 64 else 1e-6), (P, d)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", STEPS)
@pytest.mark.parametrize("mode", ki.MODES)
@pytest.mark.parametrize("growth", GROWTHS)
def test_newton_steps_match_both_oracles(gpu_ctx, growth, mode, k):
    for name, (extra, series) in batches().items():
        b = ki._ragged(series)
        opts = batched.make_options(growth=growth, seasonality_mode=mode, max_iter=k, algorithm="Newton", **extra)
        fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
        frs, th, f, info = _oracles(b, growth, mode, extra, k)
        for i in range(b.n):
            fo.assert_newton_row(fb, i, frs[i], th[i], f[i], info[i], _measured, (growth, mode, k, name, i))


@pytest.mark.gpu
@pytest.mark.parametrize("ydt", ("int32", "float32", "float64"))
def test_newton_steps_take_every_y_dtype(gpu_ctx, ydt):
    series = [_recipe_series(m, 80 + m) for m in (0, 3, 6)]
    b = ki._ragged(series)
    y = b.y if ydt == "int32" else (b.y * 1.37 + 0.25).astype(ydt)
    b = dataclasses.replace(b, y=y)
    opts = batched.make_options(max_iter=2, algorithm="Newton")
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    frs, th, f, info = _oracles(b, "logistic", "multiplicative", {}, 2)
    for i in range(b.n):
        fo.assert_newton_row(fb, i, frs[i], th[i], f[i], info[i], _measured, (ydt, i))


def _warm_init(b, fb):
    """Previous models for a warm start: a cold fit's records with delta moved to both signs and some exactly zero."""
    init = dataclasses.replace(fb, params=fb.params.copy())
    rng = np.random.default_rng(5)
    for i in range(b.n):
        S = int(fb.meta_i32[i, 1])
        d = rng.normal(0.0, 0.02, S)
        d[::3] = 0.0
        init.params[i, 3:3 + S] = d
    return init


def _c_objective_newton(b, i, copts, x0, k):
    """numpy's stan_newton on the C oracle's objective (the calibration of a warm start, which has no C driver)."""
    a, e = b.offsets[i], b.offsets[i + 1]
    y = b.y[a:e].astype(np.float64)
    return po.stan_newton(lambda x: co.objective(b.ds[a:e], y, 0.0, 1.1 * y.max(), x, copts), x0,
                          po.ProphetOptions(max_iter=k))


@pytest.mark.gpu
@pytest.mark.parametrize("k", (1, 3))
@pytest.mark.parametrize("growth", GROWTHS)
def test_newton_steps_from_warm_start_points(gpu_ctx, growth, k):
    series = [_recipe_series(m, 90 + m) for m in (0, 3, 6)] + [ki._series(7, 801, False, 97)]
    b = ki._ragged(series)
    mode = "multiplicative"
    cold = batched.fit_batch_host(gpu_ctx, batched.make_options(growth=growth, algorithm="LBFGS"), b.ds, b.y, b.offsets,
                                  0.0, 1.1)
    init = _warm_init(b, cold)
    opts = batched.make_options(growth=growth, max_iter=k, algorithm="Newton")
    fb, _ = batched.fit_batch_warm_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, init=init)
    assert np.all(fb.warm == L.WARM_USED), fb.warm
    codes, x = batched.warm_start(init, fb.meta_i32[:, 1], fb.meta_i32[:, 3], np.ones(b.n, bool))
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, max_iter=k)
    copts = co.options(growth=growth, seasonality_mode=mode)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        S, mask = int(fb.meta_i32[i, 1]), int(fb.meta_i32[i, 3])
        P = S + fo.seasonal_k(mask) + 3
        x0 = x[i, :P]
        assert np.any(x0[2:2 + S] > 0) and np.any(x0[2:2 + S] < 0) and np.any(x0[2:2 + S] == 0)
        fr = warm_oracle.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=oopts, algorithm="Newton", init=x0)
        xc, fc, itc, _, nec = _c_objective_newton(b, i, copts, x0, k)
        fo.assert_newton_row(fb, i, fr, xc, fc, (60, itc, nec), _measured, ("warm", growth, k, i))


@pytest.mark.gpu
def test_newton_error_path_is_a_line_search_failure(gpu_ctx):
    """k = 1e-3 and delta_0 = 1e-3 on a logistic trend: the Hessian's -2e-3 perturbation of delta_0 makes k + delta_0
    exactly 0, the perturbed gradient is not finite, Stan throws and fbprophet drops the series."""
    b = ki._ragged([_recipe_series(3, 33)])
    cold = batched.fit_batch_host(gpu_ctx, batched.make_options(algorithm="LBFGS"), b.ds, b.y, b.offsets, 0.0, 1.1)
    init = dataclasses.replace(cold, params=cold.params.copy())
    init.params[0, 0] = 1e-3
    init.params[0, 3] = 1e-3
    fb, _ = batched.fit_batch_warm_host(gpu_ctx, batched.make_options(algorithm="Newton"), b.ds, b.y, b.offsets, 0.0,
                                        1.1, init=init)
    _, x = batched.warm_start(init, fb.meta_i32[:, 1], fb.meta_i32[:, 3], np.ones(1, bool))
    S = int(fb.meta_i32[0, 1])
    x0 = x[0, :S + fo.seasonal_k(int(fb.meta_i32[0, 3])) + 3]
    with pytest.raises(RuntimeError, match="perturbed gradient"):
        warm_oracle.fit(b.ds, b.y.astype(np.float64), algorithm="Newton", init=x0)
    assert fb.warm[0] == L.WARM_USED
    assert fb.meta_i32[0, 4] == L.ST_LSFAIL and fb.meta_i32[0, 5] == 1, fb.meta_i32[0]
