"""GPU parity tests (run with -m gpu on an H100).  Everything goes through the C ABI
(libprophet_b200.so via ctypes); the numpy oracle is only the checker.

What can and cannot be pinned.  The model arithmetic (objective, gradient, predict) is
checked to ~1e-10 relative.  The FITTED parameters are the end point of Stan's L-BFGS with
its loose relative-gradient stop (1e7 * eps) on a non-smooth objective (Laplace prior): the
trajectory amplifies last-bit differences, so two correct fp64 implementations with different
summation order agree bit-for-bit on many series and drift apart on others.  The oracle
shows the same spread against ITSELF when one input is perturbed by one ulp
(test_fit_discrepancy_is_at_the_algorithms_own_sensitivity), so the stated tolerances for
fitted values are distribution-level: forecast differences relative to y_scale.
Stated tolerances (FP, relative to y_scale unless noted):
  objective value at a given point      1e-10 relative
  gradient at a given point             1e-8  relative to max(1, |g|_inf)
  predict given identical parameters    1e-12
  fitted forecast vs oracle             median <= 2e-3, max <= 3e-2   (config 2/3/4 samples)
  objective at the returned optimum     |f_gpu - f_oracle| / |f|: median <= 5e-4, max <= 5e-3
  MC interval bounds                    within 0.05 sigma_obs*y_scale of the oracle's own 1000-draw bounds (mean)
"""
import os

import numpy as np
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

pytestmark = pytest.mark.gpu

NS15 = 15 * 60 * 10**9


def _cases():
    return [
        ("c3", synth.config3(n=24), batched.make_options(), po.ProphetOptions(), NS15),
        ("c2", synth.config2(n=24), batched.make_options(growth="linear", yearly_seasonality=True),
         po.ProphetOptions(growth="linear", yearly_seasonality=True), 86400 * 10**9),
        ("c2_additive_logistic", synth.config2(n=12),
         batched.make_options(growth="logistic", seasonality_mode="additive", yearly_seasonality=True),
         po.ProphetOptions(growth="logistic", seasonality_mode="additive", yearly_seasonality=True), 86400 * 10**9),
        ("c4", synth.config4(n=48), batched.make_options(), po.ProphetOptions(), NS15),
    ]


def _fixture_batch(gi):
    order = np.lexsort((gi["ds_ns"], gi["dim_id"]))
    dim, ds, y = gi["dim_id"][order], gi["ds_ns"][order], gi["y"][order]
    cut = int(np.searchsorted(dim, 155))
    return synth.RaggedBatch(np.array([751, 751], np.int32), np.array([91, 155], np.int32),
                             np.array([0, cut, dim.size], np.int64), np.ascontiguousarray(ds),
                             np.ascontiguousarray(y.astype(np.int32)))


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
def test_objective_and_gradient_match_oracle(gpu_ctx, case):
    name, b, opts, oopts, _ = case
    lay = L.get_layout(opts)
    rng = np.random.RandomState(11)
    thetas, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        thetas.append(row)
        preps.append((p, th))
    f, g, mi = batched.objective_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, np.array(thetas))
    for i, (p, th) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(th, p)
        assert err == 0 and mi[i, 4] == 0
        assert (mi[i, 0], mi[i, 1]) == (p.T, p.S)
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (name, i, f[i], fo)
        gd = np.max(np.abs(g[i, :th.size] - go)) / max(1.0, np.max(np.abs(go)))
        assert gd <= 1e-8, (name, i, gd)


def test_objective_on_reference_fixture_matches_golden(gpu_ctx, golden_input, golden_oracle):
    """Config #1 input (the reference's only fixture): objective/gradient at the golden points."""
    b = _fixture_batch(golden_input)
    opts = batched.make_options()
    lay = L.get_layout(opts)
    for j in range(4):
        th = np.zeros((2, lay.pstride))
        for i, dim in enumerate((91, 155)):
            pt = golden_oracle[f"d{dim}_points"][j]
            th[i, :pt.size] = pt
        f, g, mi = batched.objective_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
        for i, dim in enumerate((91, 155)):
            fo, go = golden_oracle[f"d{dim}_f"][j], golden_oracle[f"d{dim}_g"][j]
            assert abs(f[i] - fo) <= 1e-10 * abs(fo)
            assert np.max(np.abs(g[i, :go.size] - go)) <= 1e-8 * max(1.0, np.max(np.abs(go)))
            assert mi[i, 3] == 6          # weekly + daily, yearly off (span 722.4 d < 730 d)


def test_fit_reference_fixture(gpu_ctx, golden_input, golden_oracle):
    b = _fixture_batch(golden_input)
    opts = batched.make_options()
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    for i, dim in enumerate((91, 155)):
        k = f"d{dim}_"
        assert fb.meta_i32[i, 4] in (L.ST_RELGRAD, L.ST_RELF, L.ST_ABSX)
        assert fb.meta_f64[i, 0] == float(golden_oracle[k + "y_scale"])
        assert fb.meta_f64[i, 2] == float(golden_oracle[k + "cap"])          # cap in double, prophet_modeler.py:59
        assert np.array_equal(fb.tchange[i], golden_oracle[k + "t_change"])
        fo = float(golden_oracle[k + "neg_logp"])
        assert abs(fb.meta_f64[i, 3] - fo) <= 2e-3 * abs(fo)
        fut = golden_oracle[k + "future_ns"][None, :]
        one = batched.FittedBatch(fb.params[i:i + 1], fb.tchange[i:i + 1], fb.meta_i32[i:i + 1],
                                  fb.meta_i64[i:i + 1], fb.meta_f64[i:i + 1], fb.smax, fb.kmax)
        fc = batched.predict_batch_host(gpu_ctx, opts, one, fut, np.zeros(1), np.array([float(golden_oracle[k + "cap32"])]),
                                        intervals=False)
        rel = np.max(np.abs(fc.yhat[0] - golden_oracle[k + "yhat_future"])) / float(golden_oracle[k + "y_scale"])
        assert rel <= 3e-2, (dim, rel)
        assert np.max(np.abs(fc.yhat_int[0] - golden_oracle[k + "yhat_int"])) <= 3e-2 * float(golden_oracle[k + "y_scale"]) + 1


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
def test_fit_and_forecast_match_oracle_within_stated_tolerance(gpu_ctx, case):
    _check_fit_and_forecast(gpu_ctx, case)


def _check_fit_and_forecast(gpu_ctx, case):
    name, b, opts, oopts, freq = case
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    last = b.ds[b.offsets[1:] - 1]
    fut = batched.make_future(last, 48, freq)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, intervals=False)
    rel, relf, same_path = [], [], 0
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=oopts)
        assert fb.meta_i32[i, 4] >= 0 and fr.ret >= 0
        S, K = fr.prep.S, fr.prep.K
        assert (fb.meta_i32[i, 0], fb.meta_i32[i, 1]) == (fr.prep.T, S)
        assert np.array_equal(fb.tchange[i, :S], fr.prep.t_change)
        relf.append(abs(fb.meta_f64[i, 3] - fr.neg_logp) / abs(fr.neg_logp))
        pr = po.predict(fr, fut[i], 0.0, cap32[i], oopts)
        rel.append(np.max(np.abs(pr["yhat"] - fc.yhat[i])) / fr.prep.y_scale)
        if fb.meta_i32[i, 5] == fr.iters and fb.meta_i32[i, 6] == fr.n_evals:
            # identical optimiser trajectory: parameters agree to rounding amplification only
            same_path += 1
            assert abs(fb.params[i, 0] - fr.k) < 1e-5 and abs(fb.params[i, 1] - fr.m) < 1e-5
            assert np.max(np.abs(fb.params[i, 3:3 + S] - fr.delta)) < 1e-5
            if fr.prep.seasonalities:
                assert np.max(np.abs(fb.params[i, 3 + fb.smax:3 + fb.smax + K] - fr.beta)) < 1e-5
    rel, relf = np.array(rel), np.array(relf)
    msg = (f"{name}: forecast rel diff median {np.median(rel):.2e} max {rel.max():.2e}; objective rel diff median "
           f"{np.median(relf):.2e} max {relf.max():.2e}; identical iteration path on {same_path}/{b.n}")
    print(msg)
    # objective at the returned optimum: both stop on the same loose rule, a few 1e-4 apart at most
    assert np.median(relf) <= 5e-4 and relf.max() <= 5e-3, msg
    assert np.median(rel) <= 2e-3 and rel.max() <= 3e-2, msg
    if name == "c4":
        assert same_path >= b.n // 4, msg     # short series mostly follow the oracle's exact iteration path


def test_fit_discrepancy_is_at_the_algorithms_own_sensitivity(gpu_ctx):
    """GPU-vs-oracle forecast spread is no larger than oracle-vs-oracle when ONE input value is
    moved by one ulp: the difference is the algorithm's conditioning, not an implementation error."""
    b = synth.config3(n=16)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    last = b.ds[b.offsets[1:] - 1]
    fut = batched.make_future(last, 48, NS15)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, intervals=False)
    d_gpu, d_self = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        ds, y = b.ds[a:e], b.y[a:e].astype(np.float64)
        fr = po.fit(ds, y, opts=oopts)
        pr = po.predict(fr, fut[i], 0.0, cap32[i], oopts)
        y2 = y.copy()
        y2[y2.size // 2] = np.nextafter(y2[y2.size // 2], np.inf)
        pr2 = po.predict(po.fit(ds, y2, opts=oopts), fut[i], 0.0, cap32[i], oopts)
        d_gpu.append(np.max(np.abs(pr["yhat"] - fc.yhat[i])) / fr.prep.y_scale)
        d_self.append(np.max(np.abs(pr["yhat"] - pr2["yhat"])) / fr.prep.y_scale)
    assert np.median(d_gpu) <= 5 * np.median(d_self) + 1e-6
    assert np.max(d_gpu) <= 10 * np.max(d_self) + 1e-6


@pytest.mark.parametrize("case", _cases(), ids=lambda c: c[0])
def test_predict_kernel_matches_oracle_given_same_parameters(gpu_ctx, case):
    name, b, opts, oopts, freq = case
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    last = b.ds[b.offsets[1:] - 1]
    fut = batched.make_future(last, 40, freq)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, intervals=False)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        S, K = p.S, p.K
        fr = po.FitResult(prep=p, k=fb.params[i, 0], m=fb.params[i, 1], delta=fb.params[i, 3:3 + S].copy(),
                          sigma_obs=fb.params[i, 2], beta=fb.params[i, 3 + fb.smax:3 + fb.smax + K].copy(),
                          theta=None, neg_logp=0.0, iters=0, n_evals=0, ret=0)
        pr = po.predict(fr, fut[i], 0.0, cap32[i], oopts)
        assert np.max(np.abs(pr["yhat"] - fc.yhat[i])) <= 1e-12 * p.y_scale * max(1.0, np.max(np.abs(pr["yhat"])) / p.y_scale)
        # the int epilogue exactly, on the kernel's own yhat; and the oracle's wherever the two yhat truncate alike
        assert np.array_equal(fc.yhat_int[i], np.maximum(np.trunc(fc.yhat[i]), 0.0).astype(np.int32))
        exp_int = po.scorer_epilogue(pr["yhat"], 0.0)
        same = np.trunc(pr["yhat"]) == np.trunc(fc.yhat[i])
        assert same.sum() >= same.size - 1 and np.array_equal(exp_int[same], fc.yhat_int[i][same])


def test_mc_intervals_statistically_match_oracle(gpu_ctx):
    b = synth.config3(n=4)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    last = b.ds[b.offsets[1:] - 1]
    fut = batched.make_future(last, 96, NS15)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, seed=7, intervals=True)
    fc2 = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, seed=7, intervals=True)
    assert np.array_equal(fc.yhat_lower, fc2.yhat_lower) and np.array_equal(fc.yhat_upper, fc2.yhat_upper)
    assert np.all(fc.yhat_lower < fc.yhat) and np.all(fc.yhat < fc.yhat_upper)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        S, K = p.S, p.K
        fr = po.FitResult(prep=p, k=fb.params[i, 0], m=fb.params[i, 1], delta=fb.params[i, 3:3 + S].copy(),
                          sigma_obs=fb.params[i, 2], beta=fb.params[i, 3 + fb.smax:3 + fb.smax + K].copy(),
                          theta=None, neg_logp=0.0, iters=0, n_evals=0, ret=0)
        pr = po.predict(fr, fut[i], 0.0, cap32[i], oopts)
        un = po.predict_uncertainty(fr, fut[i], pr, np.random.RandomState(3), oopts)
        sd = fr.sigma_obs * p.y_scale
        assert abs(np.mean(fc.yhat_lower[i] - un["yhat_lower"])) <= 0.05 * sd
        assert abs(np.mean(fc.yhat_upper[i] - un["yhat_upper"])) <= 0.05 * sd
        # pointwise: MC standard error of a 10 % quantile from 1000 draws is ~0.055 sd
        assert np.max(np.abs(fc.yhat_lower[i] - un["yhat_lower"])) <= 0.4 * sd
        width_o = np.mean(un["yhat_upper"] - un["yhat_lower"])
        assert abs(np.mean(fc.yhat_upper[i] - fc.yhat_lower[i]) - width_o) <= 0.03 * width_o


def test_scale_equivariance_and_batch_independence(gpu_ctx):
    """Size-independent properties: y -> 2y leaves every scaled quantity bit-identical
    (y_scale absorbs it); a series' result does not depend on what else is in the batch."""
    b = synth.config3(n=64)
    opts = batched.make_options()
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    fb2 = batched.fit_batch_host(gpu_ctx, opts, b.ds, (b.y * 2).astype(np.int32), b.offsets, 0.0, 1.1)
    assert np.array_equal(fb.params, fb2.params)
    assert np.array_equal(fb2.meta_f64[:, 0], 2 * fb.meta_f64[:, 0])
    sub = b.take(10, 20)
    fb3 = batched.fit_batch_host(gpu_ctx, opts, sub.ds, sub.y, sub.offsets, 0.0, 1.1)
    assert np.array_equal(fb3.params, fb.params[10:20]) and np.array_equal(fb3.meta_i32[:, 4:7], fb.meta_i32[10:20, 4:7])
    # f64 / f32 input dtypes give the same fit as int32
    fb4 = batched.fit_batch_host(gpu_ctx, opts, sub.ds, sub.y.astype(np.float64), sub.offsets, 0.0, 1.1)
    assert np.array_equal(fb4.params, fb3.params)


def test_edge_cases_status_codes(gpu_ctx):
    ns = 10**9
    day = 86400 * ns
    ds = np.concatenate([np.arange(1) * day, np.arange(2) * day, np.arange(30) * day, np.arange(30) * day,
                         np.arange(30) * day]).astype(np.int64)
    y = np.concatenate([[5], [3, 4], np.full(30, 7), np.arange(30) + 1, np.zeros(30)]).astype(np.int32)
    offsets = np.array([0, 1, 3, 33, 63, 93], np.int64)
    # logistic (reference default): 1 row -> TOO_FEW; all-zero y -> cap = 0 <= floor -> CAP_LE_FLOOR
    fb = batched.fit_batch_host(gpu_ctx, batched.make_options(), ds, y, offsets, 0.0, 1.1)
    st = fb.meta_i32[:, 4]
    assert st[0] == L.ST_TOO_FEW and st[4] == L.ST_CAP_LE_FLOOR
    assert st[1] >= 0 or st[1] in (L.ST_LSFAIL, L.ST_INIT_ERROR)      # 2 rows: S = 1 dummy changepoint
    assert st[3] >= 0
    # linear growth, constant y: fbprophet's "nothing to fit" shortcut
    fl = batched.fit_batch_host(gpu_ctx, batched.make_options(growth="linear"), ds, y, offsets, 0.0, 1.1)
    assert fl.meta_i32[2, 4] == L.ST_CONST_LINEAR and fl.params[2, 2] == 1e-9
    fr = po.fit(ds[3:33], y[3:33].astype(float), opts=po.ProphetOptions(growth="linear"))
    assert abs(fl.params[2, 0] - fr.k) < 1e-12 and abs(fl.params[2, 1] - fr.m) < 1e-12
    # empty batch
    e = batched.fit_batch_host(gpu_ctx, batched.make_options(), ds[:0], y[:0], np.zeros(1, np.int64), 0.0, 1.1)
    assert e.n == 0
    # unsorted timestamps are rejected per series, not silently fitted
    ds_bad = ds.copy()
    ds_bad[40], ds_bad[41] = ds_bad[41], ds_bad[40]
    fbad = batched.fit_batch_host(gpu_ctx, batched.make_options(), ds_bad, y, offsets, 0.0, 1.1)
    assert fbad.meta_i32[3, 4] == L.ST_BAD_INPUT


def test_long_and_irregular_series(gpu_ctx):
    """No shared-memory length limit (planes live in the L2-resident workspace): a 6000-point series
    with gaps, duplicates and yearly+weekly+daily seasonality (K = 34, the largest class) fits and its
    objective/gradient match the oracle."""
    rng = np.random.RandomState(42)
    step = 3 * 3600 * 10**9
    idx = np.sort(rng.choice(np.arange(9000), 6000, replace=False))
    idx[100:104] = idx[100]                      # duplicate timestamps
    ds = (np.datetime64("2015-01-01T00:00:00", "ns").astype(np.int64) + step * idx).astype(np.int64)
    days = (ds - ds[0]) / (86400 * 10**9)
    y = (500 * (1 + 0.3 * np.sin(2 * np.pi * days / 365.25) + 0.1 * np.sin(2 * np.pi * days / 7) +
                0.1 * np.sin(2 * np.pi * days)) * (1 + 0.2 * days / days.max()) + rng.normal(0, 15, ds.size))
    y = np.maximum(np.rint(y), 1).astype(np.int32)
    offsets = np.array([0, ds.size], np.int64)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    p = po.prepare(ds, y.astype(np.float64), 0.0, float(y.max()) * 1.1, oopts)
    assert (p.K, p.S) == (34, 25)
    lay = L.get_layout(opts)
    th = po.initial_theta(p) + 0.03 * rng.randn(p.S + p.K + 3)
    row = np.zeros((1, lay.pstride))
    row[0, :th.size] = th
    f, g, mi = batched.objective_host(gpu_ctx, opts, ds, y, offsets, 0.0, 1.1, row)
    err, fo, go = po.neg_logp_grad(th, p)
    assert err == 0 and mi[0, 3] == 7
    assert abs(f[0] - fo) <= 1e-10 * abs(fo)
    assert np.max(np.abs(g[0, :th.size] - go)) <= 1e-8 * max(1.0, np.max(np.abs(go)))
    fb = batched.fit_batch_host(gpu_ctx, opts, ds, y, offsets, 0.0, 1.1)
    fr = po.fit(ds, y.astype(np.float64), opts=oopts)
    assert fb.meta_i32[0, 4] >= 0 and abs(fb.meta_f64[0, 3] - fr.neg_logp) <= 5e-3 * abs(fr.neg_logp)


# ---------------------------------------------------------------------------------------
# seasonal-table kernel variants (fit_kernel.cuh point_pass_tab): the production path of a full-size
# batch of regular 10..60-minute series.  Small batches of long series default to 4 warps per series,
# so these tests pin one warp per series (PB200_LC0_MAX, read at pb200_create) to reach the variants,
# and check with pb200_last_fit_variant_counts that they really ran.
# ---------------------------------------------------------------------------------------
def _ctx_with_env(**env):
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


@pytest.fixture(scope="module")
def warp_ctx():
    """One warp per series / the grouped kernel with 8 lanes per series for every batch size (the library would give a
    batch this small 4 warps per series, and the day-table class 16 lanes per series)."""
    c = _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_GROUP=8, PB200_PLAIN_GROUP=1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def warp_ctx_tab32():
    """One warp per series for the day-table class too (point_pass_tab, the round-1 kernel) instead of the
    grouped-lanes kernel of fit_group.cuh."""
    c = _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_GROUP=0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def warp_ctx_g16():
    c = _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_GROUP=16, PB200_PLAIN_GROUP=1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def warp_ctx_no_tab():
    c = _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_NO_TAB=1)
    yield c
    c.close()


def _regrid(b, step_ns, T=None):
    """The series of a synthetic batch on another regular grid (same values, other cadence / length)."""
    T0 = int(b.offsets[1] - b.offsets[0])
    T = T0 if T is None else T
    y = b.y.reshape(b.n, T0)[:, :T]
    grid = b.ds[0] + step_ns * np.arange(T, dtype=np.int64)
    return synth.RaggedBatch(b.series_id, b.dim_id, np.arange(b.n + 1, dtype=np.int64) * T, np.tile(grid, b.n),
                             np.ascontiguousarray(y).reshape(-1))


def _tab_cases():
    c3 = synth.config3(n=16)
    H = 3600 * 10**9
    return [
        ("day_table_15min", c3, 3),                          # config #3 itself: P = 96
        ("day_table_15min_T1400", _regrid(c3, NS15, 1400), 3),   # chunk 44 would collide (44 * 24 = 11 P): widened to 45
        ("day_table_20min", _regrid(c3, 20 * 60 * 10**9), 3),    # P = 72, 20 days (chunk 45 -> 46)
        ("week_table_hourly", _regrid(c3, H), 2),            # P = 168, 60 days
        ("week_table_hourly_T337", _regrid(c3, H, 337), 2),  # two weeks + 1 point: the shortest series with weekly
        ("week_table_2h", _regrid(c3, 2 * H), 2),            # P = 84, 120 days
        ("day_table_30min", _regrid(c3, 30 * 60 * 10**9), 3),    # P = 48: the smallest table of the grouped kernel
        ("rotation_12min", _regrid(synth.config3(n=16, T=1800), 12 * 60 * 10**9), 1),   # P = 120 > 96 phases per day: no table
        ("rotation_25min", _regrid(c3, 25 * 60 * 10**9), 1),   # step divides neither day nor week: no table
    ]


_TAB_MODES = {
    "logistic_multiplicative": ({}, {}),                       # the reference's configuration
    "linear_multiplicative": ({"growth": "linear"}, {"growth": "linear"}),
    "logistic_additive": ({"seasonality_mode": "additive"}, {"seasonality_mode": "additive"}),
}


@pytest.mark.parametrize("mode", ["linear_multiplicative", "logistic_additive"])
@pytest.mark.parametrize("which", ["day_table_15min", "week_table_hourly"])
def test_table_variants_other_growth_and_mode(warp_ctx, warp_ctx_no_tab, which, mode):
    case = [c for c in _tab_cases() if c[0] == which][0]
    _check_table_objective(warp_ctx, warp_ctx_no_tab, case, mode)


@pytest.mark.parametrize("case", _tab_cases(), ids=lambda c: c[0])
def test_table_variants_objective_and_gradient(warp_ctx, warp_ctx_no_tab, case):
    _check_table_objective(warp_ctx, warp_ctx_no_tab, case, "logistic_multiplicative")


def _check_table_objective(warp_ctx, warp_ctx_no_tab, case, mode):
    name, b, variant = case
    opts, oopts = batched.make_options(**_TAB_MODES[mode][0]), po.ProphetOptions(**_TAB_MODES[mode][1])
    lay = L.get_layout(opts)
    rng = np.random.RandomState(5)
    thetas, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        thetas.append(row)
        preps.append((p, th))
    th = np.array(thetas)
    f, g, mi = batched.objective_host(warp_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    counts = warp_ctx.last_fit_variant_counts()
    assert counts[variant, 6] == b.n and counts.sum() == b.n, (name, counts)
    f0, g0, _ = batched.objective_host(warp_ctx_no_tab, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    c0 = warp_ctx_no_tab.last_fit_variant_counts()
    assert c0[1, 6] == b.n, (name, c0)
    for i, (p, t) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0 and mi[i, 3] == 6
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (name, i, f[i], fo)
        gd = np.max(np.abs(g[i, :t.size] - go)) / max(1.0, np.max(np.abs(go)))
        assert gd <= 1e-8, (name, i, gd)
        # table and rotation variants are the same sums in another order
        # (f is a difference of terms of size ~T: 0.5 ss / sigma^2 against T log sigma, so an absolute 1e-10 is 1e-13 of them)
        assert abs(f[i] - f0[i]) <= 1e-10 * max(1.0, abs(fo))
        assert np.max(np.abs(g[i] - g0[i])) <= 1e-9 * max(1.0, np.max(np.abs(go)))


@pytest.mark.parametrize("which", ["day_table_15min", "day_table_15min_T1400", "day_table_20min"])
@pytest.mark.parametrize("kernel", ["tab32", "g16"])
def test_day_table_other_kernels_objective_and_gradient(warp_ctx_tab32, warp_ctx_g16, warp_ctx_no_tab, which, kernel):
    """The day-table class on its two other kernels: 16 lanes per series (PB200_GROUP=16) and the one-warp-per-series
    point_pass_tab (PB200_GROUP=0); the default (8 lanes per series) is what every other test of this section runs."""
    case = [c for c in _tab_cases() if c[0] == which][0]
    _check_table_objective(warp_ctx_tab32 if kernel == "tab32" else warp_ctx_g16, warp_ctx_no_tab, case, "logistic_multiplicative")


@pytest.mark.parametrize("kernel", ["default_small_batch", "grouped_g8", "one_warp_rotation"])
def test_y_dtypes_give_identical_fits(gpu_ctx, warp_ctx, warp_ctx_no_tab, kernel):
    """The C ABI takes y as int32, float32 or float64 (prophet_b200.h y_dtype).  Integer counts are exact in all three, so
    the three calls must give the same bits on every kernel family; and a genuinely fractional float64 y is held to the
    oracle's objective / gradient like the integer fixtures."""
    ctx = {"default_small_batch": gpu_ctx, "grouped_g8": warp_ctx, "one_warp_rotation": warp_ctx_no_tab}[kernel]
    b = synth.config3(n=8)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    outs = []
    for dt in (np.int32, np.float32, np.float64):
        y = b.y.astype(dt)
        assert np.array_equal(y.astype(np.float64), b.y.astype(np.float64))           # exactly representable
        fb = batched.fit_batch_host(ctx, opts, b.ds, y, b.offsets, 0.0, 1.1)
        outs.append(fb)
        assert np.all(fb.meta_i32[:, 4] >= 0)
    for fb in outs[1:]:
        assert np.array_equal(fb.params, outs[0].params) and np.array_equal(fb.meta_i32, outs[0].meta_i32)
        assert np.array_equal(fb.meta_f64, outs[0].meta_f64)
    # fractional float64 values: objective and gradient against the oracle at random points
    rng = np.random.RandomState(2)
    yf = b.y.astype(np.float64) * (1.0 + 1e-3 * rng.rand(b.y.size)) + 0.37
    lay = L.get_layout(opts)
    th, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        p = po.prepare(b.ds[a:e], yf[a:e], 0.0, yf[a:e].max() * 1.1, oopts)
        t = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:t.size] = t
        th.append(row)
        preps.append((p, t))
    f, g, mi = batched.objective_host(ctx, opts, b.ds, yf, b.offsets, 0.0, 1.1, np.array(th))
    for i, (p, t) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (kernel, i, f[i], fo)
        assert np.max(np.abs(g[i, :t.size] - go)) <= 1e-8 * max(1.0, np.max(np.abs(go))), (kernel, i)


@pytest.mark.parametrize("kernel", ["default_small_batch", "grouped_g8"])
def test_explicit_cap_array_and_nonzero_floor(gpu_ctx, warp_ctx, kernel):
    """pb200_fit_* take either cap_multiplier (the reference UDF: cap = max(y) * multiplier, prophet_modeler.py:59) or a cap
    per series; and the reference's floor is a config value, not always 0 (prophet_modeler.py:57-58).  The explicit caps
    max(y) * 1.1 must reproduce the multiplier path bit for bit, and the objective with a non-zero floor must match the oracle."""
    ctx = gpu_ctx if kernel == "default_small_batch" else warp_ctx
    b = synth.config3(n=8)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    floor = 12.5
    caps = np.array([b.y[b.offsets[i]:b.offsets[i + 1]].astype(np.float64).max() * 1.1 for i in range(b.n)])
    f1 = batched.fit_batch_host(ctx, opts, b.ds, b.y, b.offsets, floor, 1.1)
    f2 = batched.fit_batch_host(ctx, opts, b.ds, b.y, b.offsets, floor, 0.0, cap=caps)
    assert np.array_equal(f1.params, f2.params) and np.array_equal(f1.meta_i32, f2.meta_i32)
    assert np.array_equal(f1.meta_f64, f2.meta_f64) and np.array_equal(f1.meta_f64[:, 2], caps)
    assert np.all(f1.meta_f64[:, 1] == floor)
    rng = np.random.RandomState(4)
    lay = L.get_layout(opts)
    th, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        p = po.prepare(b.ds[a:e], b.y[a:e].astype(np.float64), floor, caps[i], oopts)
        t = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:t.size] = t
        th.append(row)
        preps.append((p, t))
    f, g, mi = batched.objective_host(ctx, opts, b.ds, b.y, b.offsets, floor, 1.1, np.array(th))
    for i, (p, t) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (kernel, i, f[i], fo)
        assert np.max(np.abs(g[i, :t.size] - go)) <= 1e-8 * max(1.0, np.max(np.abs(go))), (kernel, i)


def _plain_cases():
    c3 = synth.config3(n=8)
    tiny = synth.config4(n=12, tmin=2, tmax=13)                     # 2 .. 13 points: fewer points than lanes, ncp < 25
    return {
        "config4_ragged": (synth.config4(n=24), {}),
        "tiny_series": (tiny, {}),
        "long_series_seasonality_off": (c3, {"weekly_seasonality": False, "daily_seasonality": False}),
        "one_day_of_15min": (_regrid(c3, NS15, 96), {}),             # span < 2 days: every auto seasonality off
        "short_series": (synth.config4(n=16, tmin=6, tmax=20), {}),
    }


@pytest.mark.parametrize("kernel", ["g8", "g16"])
@pytest.mark.parametrize("growth", ["logistic", "linear"])
@pytest.mark.parametrize("which", list(_plain_cases()))
def test_plain_grouped_class_objective_and_gradient(warp_ctx, warp_ctx_g16, warp_ctx_no_tab, which, growth, kernel):
    """The grouped kernel's class without seasonality (regular grid, seasonality mask 0: reference config #4) against the
    oracle and against the one-warp-per-series kernel, at random points around the initial one."""
    b, kw = _plain_cases()[which]
    ctx = warp_ctx if kernel == "g8" else warp_ctx_g16
    opts, oopts = batched.make_options(growth=growth, **kw), po.ProphetOptions(growth=growth, **kw)
    lay = L.get_layout(opts)
    rng = np.random.RandomState(11)
    thetas, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        assert p.K == 1
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        thetas.append(row)
        preps.append((p, th))
    th = np.array(thetas)
    f, g, mi = batched.objective_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    counts = ctx.last_fit_variant_counts()
    assert counts[3, 0] == b.n and counts.sum() == b.n, (which, counts)
    f0, g0, _ = batched.objective_host(warp_ctx_no_tab, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    assert warp_ctx_no_tab.last_fit_variant_counts()[0, 0] == b.n
    for i, (p, t) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0 and mi[i, 3] == 0
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (which, i, f[i], fo)
        gd = np.max(np.abs(g[i, :t.size] - go)) / max(1.0, np.max(np.abs(go)))
        assert gd <= 1e-8, (which, i, gd)
        assert abs(f[i] - f0[i]) <= 1e-10 * max(1.0, abs(fo))
        assert np.max(np.abs(g[i] - g0[i])) <= 1e-9 * max(1.0, np.max(np.abs(go)))


@pytest.mark.parametrize("which", ["config4_ragged", "short_series"])
def test_plain_grouped_class_fit(warp_ctx, warp_ctx_no_tab, which):
    """Fits of the class: same statuses as the one-warp-per-series kernel wherever both ran the same trajectory, objective at the
    optimum within the algorithm's own sensitivity, deterministic, batch-order independent."""
    b, kw = _plain_cases()[which]
    opts = batched.make_options(**kw)
    fa = batched.fit_batch_host(warp_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    assert warp_ctx.last_fit_variant_counts()[3, 0] == b.n
    fb = batched.fit_batch_host(warp_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    assert np.array_equal(fa.params, fb.params) and np.array_equal(fa.meta_i32, fb.meta_i32)
    f0 = batched.fit_batch_host(warp_ctx_no_tab, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    ok = (fa.meta_i32[:, 4] >= 0) & (f0.meta_i32[:, 4] >= 0)
    assert ok.sum() >= b.n - 1
    rel = np.abs(fa.meta_f64[ok, 3] - f0.meta_f64[ok, 3]) / np.maximum(1.0, np.abs(f0.meta_f64[ok, 3]))
    assert np.median(rel) <= 1e-6 and rel.max() <= 5e-3, rel
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=po.ProphetOptions(**kw))
        if fa.meta_i32[i, 4] >= 0 and fr.ret >= 0:
            assert abs(fa.meta_f64[i, 3] - fr.neg_logp) <= 5e-3 * max(1.0, abs(fr.neg_logp)), (i, fa.meta_f64[i, 3], fr.neg_logp)
    # a series' result does not depend on its neighbours in the warp: reversed batch
    T = np.diff(b.offsets)
    order = np.arange(b.n)[::-1]
    offs = np.zeros(b.n + 1, np.int64)
    np.cumsum(T[order], out=offs[1:])
    ds_r = np.concatenate([b.ds[b.offsets[i]:b.offsets[i + 1]] for i in order])
    y_r = np.concatenate([b.y[b.offsets[i]:b.offsets[i + 1]] for i in order])
    fr_ = batched.fit_batch_host(warp_ctx, opts, ds_r, y_r, offs, 0.0, 1.1)
    assert np.array_equal(fr_.params[::-1], fa.params) and np.array_equal(fr_.meta_i32[::-1, 4:7], fa.meta_i32[:, 4:7])


@pytest.mark.parametrize("which", ["day_table_15min", "week_table_hourly"])
def test_table_variants_fit_and_forecast(warp_ctx, which):
    b, variant = {c[0]: (c[1], c[2]) for c in _tab_cases()}[which]
    freq = NS15 if variant == 3 else 3600 * 10**9
    _check_fit_and_forecast(warp_ctx, (which, b, batched.make_options(), po.ProphetOptions(), freq))
    assert warp_ctx.last_fit_variant_counts()[variant, 6] == b.n
    fb = batched.fit_batch_host(warp_ctx, batched.make_options(), b.ds, b.y, b.offsets, 0.0, 1.1)
    fb2 = batched.fit_batch_host(warp_ctx, batched.make_options(), b.ds, b.y, b.offsets, 0.0, 1.1)
    assert np.array_equal(fb.params, fb2.params) and np.array_equal(fb.meta_i32, fb2.meta_i32)   # deterministic
