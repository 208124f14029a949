"""Forecast quantiles at many levels and their backtest calibration (DESIGN §15) on the GPU (run with -m gpu on an H100).

* the planes at the interval bounds' percentiles are pb200_predict_device's bounds bit for bit (both growths and
  modes, widths, sample counts, tile edges, an in-history frame, 0 / 30 changepoints, rows taken by the sort fallback),
  and the call's pointwise outputs are pb200_predict_device's;
* every plane within 1e-9 * y_scale of quantile_oracle.quantiles on mc_stream's draws, at Q = 1, 9, 32, unsorted and
  repeated levels, 0 and 100, ranks sharing a histogram bin, crowded rows, past the grid-stride loop;
* a model's planes do not depend on the batch; failed models are NaN; argument errors launch nothing;
* cv_quantile_metrics_kernel against quantile_oracle.quantile_metrics, and cross_validation_device(quantiles=...).
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import quantile_oracle as qo  # noqa: E402
from oracle import mc_stream as mcs  # noqa: E402
from test_gpu_backtest import _mixed_batch  # noqa: E402
from test_gpu_scorer import ALL_MASKS, _batch, _future, _model, _prep, _take  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched  # noqa: E402

pytestmark = pytest.mark.gpu

H_NS = 3600 * 10**9
D = 24 * H_NS
Q_TOL = 1e-9          # |plane - restatement| / y_scale
E_ARG, E_UNSUPPORTED = -1, -4
DECILES = [0.1 * k for k in range(1, 10)]
_measured = {"q": 0.0, "m": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviation():
    yield
    print(f"\n[quantiles] max |plane - restatement| / y_scale = {_measured['q']:.3e}; "
          f"max relative deviation of the quantile metrics = {_measured['m']:.3e}")


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _quant_host(ctx, opts, fb, fut, floor, cap, pct, seed, bounds=True):
    """pb200_predict_quantiles_host at raw percentiles (the bounds' own, bit for bit): (yhat, lo, hi, yint, planes)."""
    n, h = fb.n, fut.shape[1]
    pct = np.ascontiguousarray(pct, dtype=np.float64)
    fut = np.ascontiguousarray(fut, dtype=np.int64)
    floor = np.ascontiguousarray(floor, dtype=np.float64)
    cap = np.ascontiguousarray(cap, dtype=np.float64)
    yhat, lo, hi = (np.empty((n, h)) for _ in range(3))
    yint = np.empty((n, h), np.int32)
    planes = np.empty((pct.size, n, h))
    p = lambda a: a.ctypes.data                                       # noqa: E731
    rc = L.load().pb200_predict_quantiles_host(
        ctx.handle, C.byref(opts), p(np.ascontiguousarray(fb.params)), p(np.ascontiguousarray(fb.tchange)),
        p(np.ascontiguousarray(fb.meta_i32)), p(np.ascontiguousarray(fb.meta_i64)), p(np.ascontiguousarray(fb.meta_f64)),
        n, p(fut), h, p(floor), p(cap), seed, p(yhat), p(lo) if bounds else None, p(hi) if bounds else None, p(yint),
        pct.size, p(pct), p(planes))
    L.check(rc, "pb200_predict_quantiles_host")
    return yhat, (lo if bounds else None), (hi if bounds else None), yint, planes


def _identity(ctx, fb, fut, floor, cap, growth, mode, n, w, seed, ncp=25):
    """Planes at mc_stream.percentiles(w) == pb200_predict_host's bounds, and the pointwise outputs, byte for byte."""
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp, interval_width=w,
                                uncertainty_samples=n)
    ref = batched.predict_batch_host(ctx, opts, fb, fut, floor, cap, seed=seed, intervals=True)
    lo_p, hi_p = mcs.percentiles(w)
    for bounds in (True, False):
        yhat, lo, hi, yint, pl = _quant_host(ctx, opts, fb, fut, floor, cap, [lo_p, hi_p], seed, bounds)
        assert pl[0].tobytes() == ref.yhat_lower.tobytes(), (growth, mode, n, w)
        assert pl[1].tobytes() == ref.yhat_upper.tobytes(), (growth, mode, n, w)
        assert yhat.tobytes() == ref.yhat.tobytes() and yint.tobytes() == ref.yhat_int.tobytes()
        if bounds:
            assert lo.tobytes() == ref.yhat_lower.tobytes() and hi.tobytes() == ref.yhat_upper.tobytes()
    return ref


def _models(growth, mode, masks, H, seed=0, ncp=25, in_history=()):
    rng = np.random.RandomState(seed)
    frs, fut = [], []
    for i, mask in enumerate(masks):
        p, _ = _prep(mask, growth, mode, ncp=ncp)
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=i in in_history))
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp)
    fb = _batch(frs, opts)
    fut = np.stack(fut)
    floor = np.zeros(len(frs)) if growth == "linear" else rng.uniform(-5, 5, len(frs))
    cap = np.array([fr.prep.cap_value for fr in frs]) + floor
    return fb, fut, floor, cap


# ---------------------------------------------------------------------------------------------------------------------
# identity with the interval bounds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_planes_at_the_bounds_percentiles_are_the_bounds(gpu_ctx, growth, mode):
    fb, fut, floor, cap = _models(growth, mode, [6, 2, 0, 7], 40, seed=1, in_history=(3,))
    for w in (0.0, 0.5, 0.8, 0.95, 1.0):
        _identity(gpu_ctx, fb, fut, floor, cap, growth, mode, 1000, w, 5)
    for n in (2, 3, 1024):
        _identity(gpu_ctx, fb, fut, floor, cap, growth, mode, n, 0.8, 6)


@pytest.mark.parametrize("H", [1, 15, 16, 17, 672])
def test_identity_at_tile_edges(gpu_ctx, H):
    fb, fut, floor, cap = _models("logistic", "multiplicative", [6, 0], H, seed=2)
    _identity(gpu_ctx, fb, fut, floor, cap, "logistic", "multiplicative", 1000, 0.8, 7)


@pytest.mark.parametrize("ncp", [0, 30])
def test_identity_changepoint_counts(gpu_ctx, ncp):
    fb, fut, floor, cap = _models("linear", "additive", [6, 2, 0], 33, seed=3, ncp=ncp, in_history=(1,))
    _identity(gpu_ctx, fb, fut, floor, cap, "linear", "additive", 1000, 0.8, 8, ncp=ncp)


def _crowded():
    """sigma_obs = 0 just past the history's end: most draws share one value, the target ranks' bin is crowded and the
    rows go through the sort fallback (test_mc_bitonic_fallback_agrees_with_restatement's construction)."""
    p, _ = _prep(0, "linear", "additive")
    rng = np.random.RandomState(4)
    frs = [_model(p, rng, sigma=0.0, delta_scale=1.0) for _ in range(2)]
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    last = int(p.ds_sorted[-1])
    fut = np.stack([last + 20 * 10**9 * np.arange(1, 33, dtype=np.int64)] * 2)
    return fb, fut, np.zeros(2), np.ones(2)


def test_identity_through_the_sort_fallback(gpu_ctx):
    fb, fut, floor, cap = _crowded()
    for w in (0.8, 0.95):
        _identity(gpu_ctx, fb, fut, floor, cap, "linear", "additive", 1000, w, 5)
        crowd = np.concatenate([mcs.crowded_bin(mcs.draws(fb, i, fut[i], 0.0, 1.0, False, False, 1000, 5), w)
                                for i in range(2)])
        assert np.sum(crowd > 64) >= 8, crowd            # the premise: the fallback really runs


# ---------------------------------------------------------------------------------------------------------------------
# against the restatement
# ---------------------------------------------------------------------------------------------------------------------
def _check_planes(ctx, fb, fut, floor, cap, growth, mode, n, levels, seed, ncp=25):
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp, uncertainty_samples=n)
    fc = batched.predict_quantiles_host(ctx, opts, fb, fut, floor, cap, levels, seed=seed)
    assert fc.quantiles.shape == (len(levels), fb.n, fut.shape[1]) and fc.yhat_lower is None
    pct = 100.0 * np.asarray(levels, np.float64)
    for i in range(fb.n):
        if fb.meta_i32[i, 4] < 0:
            assert np.all(np.isnan(fc.quantiles[:, i]))
            continue
        d = mcs.draws(fb, i, fut[i], floor[i], cap[i], growth == "logistic", mode == "multiplicative", n, seed)
        ref = qo.quantiles(d, pct)
        err = np.max(np.abs(fc.quantiles[:, i] - ref)) / fb.meta_f64[i, 0]
        assert err <= Q_TOL, (i, err)
        _measured["q"] = max(_measured["q"], err)
    return fc


@pytest.mark.parametrize("levels", [
    [0.5],
    DECILES,
    [0.01 * k for k in np.random.RandomState(9).permutation(np.linspace(0, 100, 32))],
    [0.9, 0.1, 0.5, 0.5, 0.0, 1.0, 0.1, 0.975, 0.025],
    [0.5, 0.5005, 0.501, 0.502, 0.499],                  # ranks in one histogram bin
])
def test_planes_match_restatement_past_the_grid_stride(gpu_ctx, sms, levels):
    N = sms + 20
    rng = np.random.RandomState(10)
    frs, fut = [], []
    for i in range(N):
        p, _ = _prep(ALL_MASKS[i % len(ALL_MASKS)], "logistic", "multiplicative")
        frs.append(_model(p, rng))
        fut.append(_future(p, 18, in_history=(i % 9 == 4)))
    status = np.where(np.arange(N) % 11 == 7, L.ST_TOO_FEW, 0)
    fb = _batch(frs, batched.make_options(), status)
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    _check_planes(gpu_ctx, fb, fut, np.zeros(N), cap, "logistic", "multiplicative", 1000, levels, 3)


@pytest.mark.parametrize("growth,mode", [("logistic", "additive"), ("linear", "multiplicative")])
@pytest.mark.parametrize("n", [2, 3, 1000, 1024])
def test_planes_match_restatement_sample_counts(gpu_ctx, growth, mode, n):
    fb, fut, floor, cap = _models(growth, mode, [6, 2, 0], 17, seed=11, ncp=30)
    _check_planes(gpu_ctx, fb, fut, floor, cap, growth, mode, n, [0.0, 0.05, 0.5, 0.95, 1.0, 0.3], 4, ncp=30)


def test_planes_match_restatement_on_crowded_rows(gpu_ctx):
    fb, fut, floor, cap = _crowded()
    _check_planes(gpu_ctx, fb, fut, floor, cap, "linear", "additive", 1000, [0.05 * k for k in range(21)] + [0.333], 5)


# ---------------------------------------------------------------------------------------------------------------------
# batch independence, failed models, argument errors
# ---------------------------------------------------------------------------------------------------------------------
def test_planes_independent_of_the_batch(gpu_ctx):
    fb, fut, floor, cap = _models("logistic", "multiplicative", [6, 2, 0, 7, 6, 3], 24, seed=12)
    opts = batched.make_options()
    fb.meta_i32[4, 4] = L.ST_TOO_FEW
    full = batched.predict_quantiles_host(gpu_ctx, opts, fb, fut, floor, cap, DECILES, seed=2, intervals=True)
    assert np.all(np.isnan(full.quantiles[:, 4])) and np.all(np.isnan(full.yhat_lower[4]))
    perm = np.array([3, 0, 5, 1, 4, 2])
    pm = batched.predict_quantiles_host(gpu_ctx, opts, _take(fb, perm), fut[perm], floor[perm], cap[perm], DECILES, seed=2,
                                        intervals=True)
    assert pm.quantiles.tobytes() == full.quantiles[:, perm].tobytes()
    for i in range(6):
        one = batched.predict_quantiles_host(gpu_ctx, opts, _take(fb, [i]), fut[i:i + 1], floor[i:i + 1], cap[i:i + 1],
                                             DECILES, seed=2)
        assert one.quantiles.tobytes() == np.ascontiguousarray(full.quantiles[:, i:i + 1]).tobytes()


def test_device_call_matches_host_call(gpu_ctx):
    import torch
    fb, fut, floor, cap = _models("linear", "additive", [6, 0], 20, seed=13)
    opts = batched.make_options(growth="linear", seasonality_mode="additive")
    h = batched.predict_quantiles_host(gpu_ctx, opts, fb, fut, floor, cap, DECILES, seed=1, intervals=True)
    fd = batched.FittedBatch(*(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                               (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)), fb.smax, fb.kmax)
    d = batched.predict_quantiles_device(gpu_ctx, opts, fd, _cuda(fut), _cuda(floor), _cuda(cap), DECILES, seed=1,
                                         intervals=True)
    for k in ("yhat", "yhat_lower", "yhat_upper", "yhat_int", "quantiles"):
        assert getattr(d, k).cpu().numpy().tobytes() == getattr(h, k).tobytes(), k


def test_argument_errors_launch_nothing(gpu_ctx):
    fb, fut, floor, cap = _models("logistic", "multiplicative", [6], 8, seed=14)
    good = batched.make_options()
    lc = gpu_ctx.launch_count
    cases = [(good, 0, [50.0], E_ARG), (good, 33, [50.0] * 33, E_ARG), (good, 1, [float("nan")], E_ARG),
             (good, 1, [-1e-9], E_ARG), (good, 1, [100.0000001], E_ARG), (good, 2, None, E_ARG),
             (batched.make_options(uncertainty_samples=1), 1, [50.0], E_UNSUPPORTED),
             (batched.make_options(uncertainty_samples=1025), 1, [50.0], E_UNSUPPORTED),
             (batched.make_options(interval_width=1.5), 1, [50.0], E_ARG)]
    n, h = 1, 8
    yhat, lo, hi, planes = np.empty((1, h)), np.empty((1, h)), np.empty((1, h)), np.empty((33, 1, h))
    yint = np.empty((1, h), np.int32)
    p = lambda a: a.ctypes.data                                       # noqa: E731
    base = [gpu_ctx.handle, None, p(fb.params), p(fb.tchange), p(fb.meta_i32), p(fb.meta_i64), p(fb.meta_f64), n,
            p(np.ascontiguousarray(fut)), h, p(floor), p(cap), 0, p(yhat), p(lo), p(hi), p(yint)]
    for opts, nq, pct, code in cases:
        arr = np.ascontiguousarray(pct, dtype=np.float64) if pct is not None else None
        args = list(base)
        args[1] = C.byref(opts)
        rc = L.load().pb200_predict_quantiles_host(*args, nq, p(arr) if arr is not None else None, p(planes))
        assert rc == code, (nq, pct, rc, L.last_error())
    args = list(base)
    args[1] = C.byref(good)
    assert L.load().pb200_predict_quantiles_host(*args, 1, p(np.array([50.0])), None) == E_ARG
    assert gpu_ctx.launch_count == lc
    with pytest.raises(ValueError):
        batched.predict_quantiles_host(gpu_ctx, good, fb, fut, floor, cap, [1.5])
    assert gpu_ctx.launch_count == lc
    batched.predict_quantiles_host(gpu_ctx, good, fb, fut, floor, cap, [0.5])
    assert gpu_ctx.launch_count == lc + 2                   # predict_kernel and the quantile kernel


# ---------------------------------------------------------------------------------------------------------------------
# backtest: cv_quantile_metrics_kernel and cross_validation_device(quantiles=...)
# ---------------------------------------------------------------------------------------------------------------------
def _check_quantile_metrics(got, series, horizon, y, yq, levels, n_series, rw):
    for s in range(n_series):
        r = series == s
        ref = qo.quantile_metrics(horizon[r], y[r], yq[:, r], levels, rw)
        g = got["series"] == s
        for q, lv in enumerate(levels):
            gq = g & (got["level"] == lv) & (np.arange(g.size) % len(levels) == q)
            assert got["horizon"][gq].tolist() == ref[q]["horizon"].tolist(), (s, q)
            for k in ("pinball", "share_below"):
                a, b = got[k][gq], ref[q][k]
                np.testing.assert_allclose(a, b, rtol=1e-12, atol=0)
                if a.size:
                    _measured["m"] = max(_measured["m"], float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300))))


@pytest.mark.parametrize("rw", [0.0, 1e-3, 0.1, 0.35, 1.0])
def test_quantile_metrics_kernel_matches_oracle_past_the_stride_loop(gpu_ctx, sms, rw):
    """Interleaved, unsorted rows of more series than the kernel's grid holds threads (sms * 16 CTAs of 128), ties
    between y and its quantile, one-row series."""
    rng = np.random.RandomState(int(rw * 1000) + 1)
    n_series = sms * 16 * 128 + 37
    counts = rng.randint(1, 9, n_series)
    series = np.repeat(np.arange(n_series), counts)
    rng.shuffle(series)
    R = series.size
    horizon = rng.randint(1, 5, R).astype(np.int64) * H_NS
    y = np.round(rng.normal(0, 3, R), 1)
    levels = [0.1, 0.5, 0.9, 0.5, 0.0, 1.0]
    yq = np.stack([np.round(y + rng.normal(0, 2, R), 1) for _ in levels])
    yq[:, ::7] = y[::7]                                          # ties count as below
    got = batched.quantile_metrics_device(gpu_ctx, _cuda(series), _cuda(horizon), _cuda(y), _cuda(yq), levels, n_series, rw)
    check = rng.choice(n_series, 300, replace=False)
    check = np.concatenate([check, [n_series - 1]])
    keep = np.isin(series, check)
    remap = -np.ones(n_series, np.int64)
    remap[check] = np.arange(check.size)
    sub = {k: v[np.isin(got["series"], check)] for k, v in got.items()}
    sub["series"] = remap[sub["series"]]
    _check_quantile_metrics(sub, remap[series[keep]], horizon[keep], y[keep], yq[:, keep], levels, check.size, rw)


def test_quantile_metrics_argument_errors(gpu_ctx):
    lc = gpu_ctx.launch_count
    z = _cuda(np.zeros(4))
    i = _cuda(np.zeros(4, np.int64))
    for nq, lv, rw in ((0, [0.5], 0.1), (33, [0.5] * 33, 0.1), (1, [1.5], 0.1), (1, [float("nan")], 0.1),
                       (1, [0.5], 1.5), (1, None, 0.1)):
        arr = np.ascontiguousarray(lv, dtype=np.float64) if lv is not None else None
        rc = L.load().pb200_cv_quantile_metrics_device(gpu_ctx.handle, i.data_ptr(), z.data_ptr(), z.data_ptr(), 4, nq,
                                                       arr.ctypes.data if arr is not None else None, i.data_ptr(),
                                                       i.data_ptr(), 1, rw, i.data_ptr(), i.data_ptr(), z.data_ptr(),
                                                       z.data_ptr(), i.data_ptr())
        assert rc == E_ARG, (nq, lv, rw)
    assert gpu_ctx.launch_count == lc


FLOOR, CAPM = 0.0, 1.1
HORIZON, PERIOD, INITIAL = D, D // 2, 3 * D
KEEP = [0, 1, 2, 3, 4, 8, 9, 10, 11]
LEVELS = [0.1, 0.5, 0.9, 0.025, 0.975]


def _cv(ctx, ds, y, off, intervals=True, quantiles=None, keep_fits=False, budget=None):
    opts = batched.make_options(uncertainty_samples=200)
    cap = _cuda(np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])]))
    return batched.cross_validation_device(ctx, opts, _cuda(ds), _cuda(y), off, FLOOR, cap, HORIZON, PERIOD, INITIAL,
                                           intervals=intervals, seed=3, rolling_window=0.1, quantiles=quantiles,
                                           keep_fits=keep_fits, _row_budget=budget)


@pytest.fixture(scope="module", params=[np.float32, np.float64])
def cv_batch(request):
    ds, y, off = _mixed_batch()
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in KEEP]
    o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]).astype(request.param), o2


def _result_bytes(res):
    out = {k: (None if getattr(res, k) is None else getattr(res, k).tobytes())
           for k in ("pair_series", "pair_cutoff", "pair_status", "pair_mask", "row_series", "ds", "cutoff", "y", "yhat",
                     "yhat_lower", "yhat_upper")}
    out.update({"m_" + k: (None if v is None else v.tobytes()) for k, v in res.metrics.items()})
    return out


def test_backtest_quantiles_end_to_end(gpu_ctx, cv_batch):
    ds, y, off = cv_batch
    n_series = off.size - 1
    plain = _cv(gpu_ctx, ds, y, off)
    res = _cv(gpu_ctx, ds, y, off, quantiles=LEVELS, keep_fits=True)
    point = _cv(gpu_ctx, ds, y, off, intervals=False, quantiles=LEVELS)
    assert plain.yhat_q is None and plain.quantile_metrics is None
    assert _result_bytes(res) == _result_bytes(plain)
    assert point.yhat_lower is None and point.yhat_q.tobytes() == res.yhat_q.tobytes()
    assert res.yhat_q.shape == (len(LEVELS), res.ds.size)
    # chunks do not change a row
    small = _cv(gpu_ctx, ds, y, off, quantiles=LEVELS, budget=1)
    assert small.yhat_q.tobytes() == res.yhat_q.tobytes()
    for k, v in res.quantile_metrics.items():
        assert small.quantile_metrics[k].tobytes() == v.tobytes(), k
    # the held-out planes against the restatement at the GPU's parameters
    cap = np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])])
    rng = np.random.RandomState(0)
    for p in rng.choice(res.pair_series.size, 8, replace=False):
        s, c = int(res.pair_series[p]), int(res.pair_cutoff[p])
        rows = (res.row_series == s) & (res.cutoff == c)
        d = mcs.draws(res.fitted, int(p), res.ds[rows], FLOOR, cap[s], True, True, 200, 3)
        ref = qo.quantiles(d, 100.0 * np.asarray(LEVELS))
        err = np.max(np.abs(res.yhat_q[:, rows] - ref)) / float(res.fitted.meta_f64[p, 0])
        assert err <= Q_TOL, (p, err)
        _measured["q"] = max(_measured["q"], err)
    _check_quantile_metrics(res.quantile_metrics, res.row_series, res.ds - res.cutoff, res.y, res.yhat_q, LEVELS,
                            n_series, 0.1)


def test_backtest_quantiles_refuse_aggregate_and_grid(gpu_ctx, cv_batch):
    ds, y, off = cv_batch
    opts = batched.make_options(uncertainty_samples=200)
    cap = _cuda(np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])]))
    for kw in ({"aggregate_ns": D}, {"grid": [(0.05, 10.0)]}):
        with pytest.raises(ValueError):
            batched.cross_validation_device(gpu_ctx, opts, _cuda(ds), _cuda(y), off, FLOOR, cap, HORIZON, PERIOD, INITIAL,
                                            quantiles=LEVELS, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# the jobs on the golden fixture
# ---------------------------------------------------------------------------------------------------------------------
def test_scorer_job_writes_quantile_columns(tmp_path, model_input_dir, gpu_ctx):
    import pyarrow.dataset as pads
    from time_series_spark_b200 import model_record
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    from time_series_spark_b200.jobs.prophet_scorer import ProphetScorer, frequency_to_future
    models = str(tmp_path / "models")
    ProphetModeler.model(None, {"io": {"input": model_input_dir, "models": models}, "model": {"floor": 0, "cap_multiplier": 1.1}})
    fcast = {"periods": 300, "frequency": "15min", "uncertainty_samples": 500, "seed": 3, "intervals": True}
    levels = [0.9, 0.1, 0.5]
    plain = {"io": {"models": models, "forecasts": str(tmp_path / "plain")}, "forecast": dict(fcast)}
    quant = {"io": {"models": models, "forecasts": str(tmp_path / "q")}, "forecast": dict(fcast, quantiles=levels)}
    ProphetScorer.score(None, plain)
    ProphetScorer.score(None, quant)
    a = pads.dataset(plain["io"]["forecasts"], format="csv").to_table().drop_columns(["created_timestamp"])
    b = pads.dataset(quant["io"]["forecasts"], format="csv").to_table().drop_columns(["created_timestamp"])
    cols = ["yhat_q0.9", "yhat_q0.1", "yhat_q0.5"]
    assert b.column_names == a.column_names + cols and a.num_rows == 600
    assert b.select(a.column_names).equals(a)
    mt = pads.dataset(models, format="parquet").to_table()
    fitted, last_ds, info = model_record.decode(mt["model"])
    opts = batched.make_options(growth="logistic" if info["logistic"] else "linear",
                                seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
                                n_changepoints=info["n_changepoints"], uncertainty_samples=500)
    opts.yearly, opts.weekly, opts.daily = info["yearly"], info["weekly"], info["daily"]
    floor = np.asarray(mt["floor"].to_pylist(), np.float32).astype(np.float64)
    cap = np.asarray(mt["cap"].to_pylist(), np.float32).astype(np.float64)
    fc = batched.predict_quantiles_host(gpu_ctx, opts, fitted, frequency_to_future(last_ds, 300, "15min"), floor, cap,
                                        levels, seed=3, intervals=True)
    for q, c in enumerate(cols):
        assert np.array_equal(b[c].to_numpy(), fc.quantiles[q].reshape(-1)), c        # the CSV prints doubles round-trip
    assert np.array_equal(b["yhat_lower"].to_numpy(), fc.yhat_lower.reshape(-1))


QM_COLS = ["series_id", "dim_id", "horizon", "quantile", "pinball_loss", "share_below"]


def _bt_config(tmp_path, inp, **bt):
    return {"io": {"input": inp, "metrics": str(tmp_path / "metrics"), "cv_rows": str(tmp_path / "rows"),
                   "quantile_metrics": str(tmp_path / "qm")},
            "model": {"floor": 0, "cap_multiplier": 1.1},
            "backtest": {"horizon": "30 days", "period": "15 days", "initial": "180 days", "uncertainty_samples": 100, **bt}}


@pytest.mark.parametrize("intervals", [True, False])
def test_backtest_job_on_golden_fixture(tmp_path, model_input_dir, intervals):
    import shutil
    import pyarrow as pa
    import pyarrow.parquet as pq
    from time_series_spark_b200.jobs.prophet_backtest import ProphetBacktester
    ProphetBacktester.run(None, _bt_config(tmp_path, model_input_dir, intervals=intervals))
    base_m, base_r = pq.read_table(str(tmp_path / "metrics")), pq.read_table(str(tmp_path / "rows"))
    for d in ("metrics", "rows"):
        shutil.rmtree(str(tmp_path / d))
    ProphetBacktester.run(None, _bt_config(tmp_path, model_input_dir, intervals=intervals, quantiles=LEVELS))
    m, r = pq.read_table(str(tmp_path / "metrics")), pq.read_table(str(tmp_path / "rows"))
    qcols = ["yhat_q" + repr(float(q)) for q in LEVELS]
    assert m.equals(base_m)
    assert r.column_names == base_r.column_names + qcols and r.select(base_r.column_names).equals(base_r)
    qm = pq.read_table(str(tmp_path / "qm"))
    assert qm.schema.names == QM_COLS and qm.schema.field("horizon").type == pa.duration("ns") and qm.num_rows > 0
    rows, got = r.to_pandas(), qm.to_pandas()
    for (sid, dim), g in rows.groupby(["series_id", "dim_id"]):
        h = (g.ds.values.astype(np.int64) - g.cutoff.values.astype(np.int64))
        yq = np.stack([g[c].values for c in qcols])
        ref = qo.quantile_metrics(h, g.y.values.astype(np.float64), yq, LEVELS, 0.1)
        gg = got[(got.series_id == sid) & (got.dim_id == dim)]
        for q, lv in enumerate(LEVELS):
            s = gg[gg["quantile"] == lv]
            assert s.horizon.values.astype(np.int64).tolist() == ref[q]["horizon"].tolist()
            np.testing.assert_allclose(s.pinball_loss.values, ref[q]["pinball"], rtol=1e-12, atol=0)
            np.testing.assert_allclose(s.share_below.values, ref[q]["share_below"], rtol=1e-12, atol=0)


def test_backtest_job_empty_shard_schema(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq
    from time_series_spark_b200.jobs import prophet_backtest as pb
    tbl = pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32()),
                    "ds": pa.array([], pa.timestamp("ns")), "y": pa.array([], pa.int32())})
    job = pb.ProphetBacktester(_bt_config(tmp_path, None, quantiles=[0.5, 0.9]))
    metrics, rows = job.backtest(tbl)
    assert rows.column_names[-2:] == ["yhat_q0.5", "yhat_q0.9"] and rows.num_rows == 0
    assert job.quantile_metrics.schema.names == QM_COLS and job.quantile_metrics.num_rows == 0
    job.persist(metrics, rows)
    assert pq.read_table(str(tmp_path / "qm")).schema.names == QM_COLS
