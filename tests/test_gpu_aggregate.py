"""Forecast totals over time windows (DESIGN §13) on the GPU (run with -m gpu on an H100).

* mc_sum_kernel against tests/window_oracle.window_sums at the GPU's parameters: every window bound within
  1e-9 * y_scale * n_points; yhat_sum the ordered sum of the kernel's own yhat exactly and within
  1e-12 * y_scale * n_points of the oracle's; quantity_sum, n_points, window_start, n_windows exact;
* with one point per window the bounds are the bits of pb200_predict_*'s yhat_lower / yhat_upper, and the pointwise
  outputs of the call are those of pb200_predict_* in any case;
* a model's window rows do not depend on its place in the batch or on wmax;
* failed models, empty batches and frames, argument errors (nothing launched), too few slots;
* the scorer job with forecast.aggregate on the golden fixture.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pyarrow.dataset as pads
import pytest

import window_oracle as wo
from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
from test_gpu_scorer import ALL_MASKS, _batch, _future, _model, _prep, _take
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, model_record

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H_NS = 3600 * 10**9
DAY = 24 * H_NS
MIN15 = 15 * 60 * 10**9
INT64_MIN = -2**63
SUM_TOL = 1e-9       # |kernel - restatement| / (y_scale * n_points)
PRED_TOL = 1e-12     # |yhat_sum - ordered sum of the oracle's yhat| / (y_scale * n_points * max(1, |yhat| / y_scale))
_measured = {"sum": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviation():
    yield
    print(f"\n[aggregate] max |mc_sum_kernel - restatement| / (y_scale * n_points) = {_measured['sum']:.3e}")


def _check_empty_slots(ws, i, nw):
    assert np.all(ws.start[i, nw:] == INT64_MIN) and np.all(ws.points[i, nw:] == 0)
    assert np.all(ws.quantity_sum[i, nw:] == INT64_MIN)
    assert np.all(np.isnan(ws.yhat_sum[i, nw:])) and np.all(np.isnan(ws.lower[i, nw:])) and np.all(np.isnan(ws.upper[i, nw:]))


def _check_sums(gpu_ctx, frs, fb, fut, floor, cap, growth, mode, n, width, seed, width_ns, origin_ns, ncp=25, oopts=None):
    """Run the kernel, restate every model's windows, compare; returns the result and the restated draws."""
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp, interval_width=width,
                                uncertainty_samples=n)
    fc, ws = batched.predict_sums_host(gpu_ctx, opts, fb, fut, floor, cap, width_ns, origin_ns, seed=seed)
    out = []
    for i in range(fb.n):
        if fb.meta_i32[i, 4] < 0:
            assert ws.n_windows[i] == 0
            _check_empty_slots(ws, i, 0)
            out.append(None)
            continue
        d = mcs.draws(fb, i, fut[i], floor[i], cap[i], growth == "logistic", mode == "multiplicative", n, seed)
        start, pts, lo, hi = wo.window_sums(d, fut[i], width_ns, origin_ns, width)
        nw = start.size
        assert ws.n_windows[i] == nw, (i, ws.n_windows[i], nw)
        assert np.array_equal(ws.start[i, :nw], start) and np.array_equal(ws.points[i, :nw], pts)
        _check_empty_slots(ws, i, nw)
        ys = fb.meta_f64[i, 0]
        err = max(np.max(np.abs(ws.lower[i, :nw] - lo) / pts), np.max(np.abs(ws.upper[i, :nw] - hi) / pts)) / ys
        assert err <= SUM_TOL, (i, n, width, seed, err)
        _measured["sum"] = max(_measured["sum"], err)
        first, _ = wo.window_runs(fut[i], width_ns, origin_ns)
        ref = po.predict(frs[i], fut[i], floor[i], cap[i], oopts)["yhat"] if oopts is not None else None
        for j in range(nw):
            s, r = 0.0, 0.0
            for h in range(first[j], first[j + 1]):
                s = s + fc.yhat[i, h]
                if ref is not None:
                    r = r + ref[h]
            assert ws.yhat_sum[i, j] == s
            if ref is not None:
                big = max(1.0, np.max(np.abs(ref[first[j]:first[j + 1]])) / ys)
                assert abs(s - r) <= PRED_TOL * ys * pts[j] * big, (i, j, s, r)
            assert ws.quantity_sum[i, j] == int(fc.yhat_int[i, first[j]:first[j + 1]].astype(np.int64).sum())
        out.append(d)
    return fc, ws, out


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_sums_match_restatement_many_models(gpu_ctx, growth, mode):
    """200 models (more than the grid), all eight masks, 30 changepoints: histories at 15 minutes ... one week per
    point with different last dates, so daily windows hold 96 ... 1 points, models of one call have 1 ... 60 windows
    with partial first and last ones, and a weekly grid leaves windows without a point; every fifth model is forecast
    inside its history (Tmax <= 1), failed rows interleaved."""
    rng = np.random.RandomState(1)
    H, N = 60, 200
    frs, fut = [], []
    for i in range(N):
        p, oopts = _prep(ALL_MASKS[i % len(ALL_MASKS)], growth, mode, ncp=30)
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=(i % 5 == 3)) + (i % 3) * 5 * H_NS)     # ragged: 0 / 5 / 10 hours later
    status = np.where(np.arange(N) % 7 == 5, L.ST_TOO_FEW, 0)
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=30)
    fb = _batch(frs, opts, status)
    fut = np.stack(fut)
    floor = np.zeros(N) if growth == "linear" else rng.uniform(-5, 5, N)
    cap = np.array([fr.prep.cap_value for fr in frs]) + floor
    _, ws, _ = _check_sums(gpu_ctx, frs, fb, fut, floor, cap, growth, mode, 1000, 0.8, 7, DAY, 0, ncp=30, oopts=oopts)
    counts = set(ws.n_windows[status == 0].tolist())
    assert min(counts) <= 3 and max(counts) >= 60 and len(counts) >= 4, counts


def test_sums_match_restatement_sample_counts_and_widths(gpu_ctx):
    """n_samples 2 ... 1024 x interval widths 0, 0.8, 1 with the dummy changepoint of n_changepoints = 0, 8-hour
    windows from an origin that is not midnight."""
    rng = np.random.RandomState(2)
    frs, fut = [], []
    for mask in (6, 2, 0):
        p, _ = _prep(mask, "logistic", "multiplicative", ncp=0)
        frs.append(_model(p, rng))
        fut.append(_future(p, 40))
    fb = _batch(frs, batched.make_options(n_changepoints=0))
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    for n in (2, 100, 1000, 1024):
        for w in (0.0, 0.8, 1.0):
            _check_sums(gpu_ctx, frs, fb, fut, np.zeros(3), cap, "logistic", "multiplicative", n, w, 3, 8 * H_NS,
                        5 * H_NS + 1, ncp=0)


@pytest.mark.parametrize("H", [1, 15, 16, 17, 672])
def test_sums_match_restatement_horizons(gpu_ctx, H):
    """Frames shorter and longer than the 512-point staging tile, odd and even, one of them inside the history."""
    rng = np.random.RandomState(3)
    frs, fut = [], []
    for mask, inside in ((6, False), (0, False), (6, True), (2, False)):
        p, _ = _prep(mask, "linear", "additive")
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=inside))
    fut = np.stack(fut)
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    _check_sums(gpu_ctx, frs, fb, fut, np.zeros(4), np.ones(4), "linear", "additive", 1000, 0.8, 11, DAY, 0)


@pytest.mark.parametrize("count", [1, 15, 16, 17, 33])
def test_sums_match_restatement_window_counts(gpu_ctx, count):
    """Window counts on both sides of the 16-row staging area: an hourly frame from midnight in 4-hour windows, and the
    same frame shifted by an hour (one window more, partial edges)."""
    rng = np.random.RandomState(4)
    p, _ = _prep(6, "logistic", "additive")
    frs = [_model(p, rng), _model(p, rng)]
    base = _future(p, 4 * count)
    assert base[0] % (4 * H_NS) == 0
    fut = np.stack([base, base + H_NS])
    fb = _batch(frs, batched.make_options(growth="logistic", seasonality_mode="additive"))
    cap = np.array([fr.prep.cap_value for fr in frs])
    _, ws, _ = _check_sums(gpu_ctx, frs, fb, fut, np.zeros(2), cap, "logistic", "additive", 1000, 0.8, 5, 4 * H_NS, 0)
    assert ws.n_windows.tolist() == [count, count + 1]
    assert np.all(ws.points[0, :count] == 4) and ws.points[1, 0] == 3 and ws.points[1, count] == 1


def test_sums_bitonic_fallback_agrees_with_restatement(gpu_ctx):
    """sigma_obs = 0 just past the history's end: most draws have met no simulated changepoint and share one value, so do
    their window sums, the histogram bin of the target ranks holds far more than 64 of them and the selection falls back
    to the full sort."""
    p, _ = _prep(0, "linear", "additive")
    rng = np.random.RandomState(4)
    frs = [_model(p, rng, sigma=0.0, delta_scale=1.0) for _ in range(2)]
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    last = int(p.ds_sorted[-1])
    fut = np.stack([last + 20 * 10**9 * np.arange(1, 35, dtype=np.int64)] * 2)
    for w in (0.8, 0.95):
        _, _, ds = _check_sums(gpu_ctx, frs, fb, fut, np.zeros(2), np.ones(2), "linear", "additive", 1000, w, 5,
                               40 * 10**9, last)
        crowd = []
        for i, d in enumerate(ds):
            first, _ = wo.window_runs(fut[i], 40 * 10**9, last)
            sums = np.array([np.add.reduce(d[first[j]:first[j + 1]], axis=0) for j in range(first.size - 1)])
            crowd.append(mcs.crowded_bin(sums, w))
        assert np.sum(np.concatenate(crowd) > 64) >= 8, crowd      # the premise: the fallback really runs


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("linear", "additive")])
def test_one_point_windows_are_the_pointwise_intervals(gpu_ctx, growth, mode):
    """With the grid step as the width every window holds one point: lower / upper are the bits of pb200_predict_*'s
    yhat_lower / yhat_upper, yhat_sum those of yhat, quantity_sum is yhat_int; and the pointwise outputs of the sums
    call are pb200_predict_*'s."""
    rng = np.random.RandomState(6)
    H = 672
    frs, fut = [], []
    for k in range(6):
        p, _ = _prep(0, growth, mode)
        frs.append(_model(p, rng))
        fut.append(_future(p, H) + k * DAY)
    opts = batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=1000)
    fb = _batch(frs, opts)
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    ref = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(6), cap, seed=9, intervals=True)
    fc, ws = batched.predict_sums_host(gpu_ctx, opts, fb, fut, np.zeros(6), cap, MIN15, 0, seed=9, intervals=True)
    assert ws.start.shape == (6, H) and np.all(ws.n_windows == H) and np.all(ws.points == 1)
    assert np.array_equal(ws.start, fut)
    assert np.array_equal(ws.lower, ref.yhat_lower) and np.array_equal(ws.upper, ref.yhat_upper)
    assert np.array_equal(ws.yhat_sum, ref.yhat) and np.array_equal(ws.quantity_sum, ref.yhat_int.astype(np.int64))
    for a, b in ((fc.yhat, ref.yhat), (fc.yhat_int, ref.yhat_int), (fc.yhat_lower, ref.yhat_lower),
                 (fc.yhat_upper, ref.yhat_upper)):
        assert np.array_equal(a, b)
    # without the pointwise intervals the call returns none, and the same sums
    fc2, ws2 = batched.predict_sums_host(gpu_ctx, opts, fb, fut, np.zeros(6), cap, MIN15, 0, seed=9)
    assert fc2.yhat_lower is None and np.array_equal(fc2.yhat, ref.yhat) and np.array_equal(ws2.lower, ws.lower)


def test_device_call_equals_host_call(gpu_ctx):
    import torch
    rng = np.random.RandomState(7)
    frs, fut = [], []
    for k in range(5):
        p, _ = _prep([6, 0][k % 2], "linear", "multiplicative")
        frs.append(_model(p, rng))
        fut.append(_future(p, 200))
    opts = batched.make_options(growth="linear", seasonality_mode="multiplicative", uncertainty_samples=300)
    fb = _batch(frs, opts)
    fut = np.stack(fut)
    fc, ws = batched.predict_sums_host(gpu_ctx, opts, fb, fut, np.zeros(5), np.ones(5), DAY, 0, seed=4, intervals=True)
    dev = torch.device("cuda", gpu_ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    dfb = batched.FittedBatch(t(fb.params), t(fb.tchange), t(fb.meta_i32), t(fb.meta_i64), t(fb.meta_f64), fb.smax, fb.kmax)
    dfc, dws = batched.predict_sums_device(gpu_ctx, opts, dfb, t(fut), t(np.zeros(5)), t(np.ones(5)), DAY, 0, seed=4,
                                           intervals=True)
    for name in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        assert np.array_equal(getattr(dws, name).cpu().numpy(), getattr(ws, name), equal_nan=name in ("yhat_sum", "lower", "upper")), name
    assert np.array_equal(dfc.yhat.cpu().numpy(), fc.yhat) and np.array_equal(dfc.yhat_lower.cpu().numpy(), fc.yhat_lower)


def test_window_rows_do_not_depend_on_batch_position_or_slots(gpu_ctx):
    rng = np.random.RandomState(8)
    N = 150
    frs, fut = [], []
    for i in range(N):
        p, _ = _prep([6, 2, 0][i % 3], "logistic", "multiplicative")
        frs.append(_model(p, rng))
        fut.append(_future(p, 48))                 # hourly: 2 days, daily: 48 days, 15 minutes: half a day
    opts = batched.make_options(uncertainty_samples=1000)
    fb = _batch(frs, opts)
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    _, full = batched.predict_sums_host(gpu_ctx, opts, fb, fut, np.zeros(N), cap, DAY, 0, seed=21)
    assert full.start.shape[1] == 48
    fields = ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper")

    def same(sub, idx):
        w = sub.start.shape[1]
        for f in fields:
            a, b = getattr(sub, f), getattr(full, f)[idx]
            assert np.array_equal(a, b if a.ndim == 1 else b[:, :w], equal_nan=True), f
        assert np.all(full.n_windows[idx] <= w)

    idx = np.concatenate([np.arange(120, 140), np.arange(37, 102)[::-1]])
    _, sub = batched.predict_sums_host(gpu_ctx, opts, _take(fb, idx), fut[idx], np.zeros(idx.size), cap[idx], DAY, 0, seed=21)
    same(sub, idx)
    # an hourly model alone: 2 or 3 slots instead of 48
    _, one = batched.predict_sums_host(gpu_ctx, opts, _take(fb, [75]), fut[[75]], np.zeros(1), cap[[75]], DAY, 0, seed=21)
    assert one.start.shape[1] <= 3
    same(one, np.array([75]))
    _, other = batched.predict_sums_host(gpu_ctx, opts, _take(fb, [75]), fut[[75]], np.zeros(1), cap[[75]], DAY, 0, seed=22)
    assert not np.array_equal(other.lower, one.lower) and np.array_equal(other.yhat_sum, one.yhat_sum)


def _raw(gpu_ctx, opts, fb, fut, wmax, width_ns=DAY, origin_ns=0, n=None, h=None, null=None):
    """pb200_predict_sums_host with every argument in the caller's hand; returns (rc, outputs)."""
    n = fb.n if n is None else n
    h = fut.shape[1] if h is None else h
    slots = max(1, fb.n * max(wmax, 1))
    o = dict(nw=np.full(max(fb.n, 1), -7, np.int32), start=np.full(slots, -7, np.int64), pts=np.full(slots, -7, np.int32),
             ys=np.full(slots, -7.0), qs=np.full(slots, -7, np.int64), lo=np.full(slots, -7.0), hi=np.full(slots, -7.0),
             yhat=np.full(fut.size + 1, -7.0), yint=np.full(fut.size + 1, -7, np.int32))
    ptr = lambda k: None if null == k else o[k].ctypes.data_as(C.c_void_p)      # noqa: E731
    arr = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)          # noqa: E731
    floor, cap = np.zeros(max(fb.n, 1)), np.ones(max(fb.n, 1))
    rc = L.load().pb200_predict_sums_host(
        gpu_ctx.handle, C.byref(opts), arr(fb.params), arr(fb.tchange), arr(fb.meta_i32), arr(fb.meta_i64),
        arr(fb.meta_f64), n, arr(fut), h, arr(floor), arr(cap), 0, ptr("yhat"), None, None, ptr("yint"), width_ns,
        origin_ns, wmax, ptr("nw"), ptr("start"), ptr("pts"), ptr("ys"), ptr("qs"), ptr("lo"), ptr("hi"))
    return rc, o


def _small(growth="linear", mode="additive", n=3, H=48):
    rng = np.random.RandomState(9)
    p, _ = _prep(6, growth, mode)
    frs = [_model(p, rng) for _ in range(n)]
    fb = _batch(frs, batched.make_options(growth=growth, seasonality_mode=mode))
    return fb, np.stack([_future(p, H)] * n)


def test_argument_errors_launch_nothing(gpu_ctx):
    fb, fut = _small()
    ok = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=100)
    E_ARG, E_UNSUPPORTED = -1, -4
    cases = []
    for ns in (0, 1, 1025):
        cases.append((batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=ns), {}, E_UNSUPPORTED))
    for w in (-0.1, 1.5, float("nan")):
        cases.append((batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=100,
                                           interval_width=w), {}, E_ARG))
    cases += [(ok, dict(width_ns=0), E_ARG), (ok, dict(width_ns=-DAY), E_ARG), (ok, dict(wmax=0), E_ARG),
              (ok, dict(wmax=-3), E_ARG), (ok, dict(n=-1), E_ARG), (ok, dict(h=-1), E_ARG)]
    cases += [(ok, dict(null=k), E_ARG) for k in ("nw", "start", "pts", "ys", "qs", "lo", "hi", "yhat", "yint")]
    before = gpu_ctx.launch_count
    for opts, kw, code in cases:
        kw = dict(dict(wmax=4), **kw)
        rc, o = _raw(gpu_ctx, opts, fb, fut, **kw)
        assert rc == code, (kw, opts.uncertainty_samples, opts.interval_width, rc, L.last_error())
        assert all(np.all(v == -7) for v in o.values()), kw
    assert gpu_ctx.launch_count == before
    rc, o = _raw(gpu_ctx, ok, fb, fut, 4)
    assert rc == 0 and gpu_ctx.launch_count == before + 2         # predict_kernel and mc_sum_kernel, no pointwise intervals
    assert np.all(o["nw"] == 2)                                   # 48 hourly points from midnight
    with pytest.raises(ValueError, match="width_ns"):
        batched.predict_sums_host(gpu_ctx, ok, fb, fut, np.zeros(3), np.ones(3), 0)


def test_too_few_slots_report_the_true_count(gpu_ctx):
    fb, fut = _small(H=100)          # hourly from midnight: 5 daily windows
    opts = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=100)
    rc, full = _raw(gpu_ctx, opts, fb, fut, 8)
    rc2, cut = _raw(gpu_ctx, opts, fb, fut, 2)
    assert rc == 0 and rc2 == 0
    assert np.all(full["nw"] == 5) and np.all(cut["nw"] == 5)
    for k in ("start", "pts", "ys", "qs", "lo", "hi"):
        assert np.array_equal(cut[k].reshape(3, 2), full[k].reshape(3, 8)[:, :2]), k
    assert np.all(full["pts"].reshape(3, 8)[:, 5:] == 0) and np.all(np.isnan(full["lo"].reshape(3, 8)[:, 5:]))


def test_failed_models_and_empty_inputs(gpu_ctx):
    fb, fut = _small(n=4)
    fb.meta_i32[[1, 3], 4] = L.ST_TOO_FEW
    opts = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=100)
    fc, ws = batched.predict_sums_host(gpu_ctx, opts, fb, fut, np.zeros(4), np.ones(4), DAY, 0)
    assert ws.n_windows.tolist() == [2, 0, 2, 0]
    for i in (1, 3):
        _check_empty_slots(ws, i, 0)
        assert np.all(np.isnan(fc.yhat[i]))
    assert np.all(np.isfinite(ws.lower[[0, 2]])) and np.all(ws.lower[[0, 2]] < ws.upper[[0, 2]])
    # no model: nothing to do; no point: every model has no window
    before = gpu_ctx.launch_count
    fc0, ws0 = batched.predict_sums_host(gpu_ctx, opts, _take(fb, []), fut[:0], np.zeros(0), np.ones(0), DAY, 0)
    assert ws0.n_windows.shape == (0,) and ws0.start.shape == (0, 1) and gpu_ctx.launch_count == before
    fch, wsh = batched.predict_sums_host(gpu_ctx, opts, fb, fut[:, :0], np.zeros(4), np.ones(4), DAY, 0)
    assert fch.yhat.shape == (4, 0) and wsh.n_windows.tolist() == [0, 0, 0, 0] and wsh.start.shape == (4, 1)
    for i in range(4):
        _check_empty_slots(wsh, i, 0)


def _run_scorer(cfg, tmp_path, name):
    import yaml
    path = tmp_path / f"{name}.yaml"
    path.write_text(yaml.safe_dump(cfg))
    r = subprocess.run([sys.executable, "-m", "time_series_spark_b200.scorer_driver", str(path)], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-2000:])


def test_scorer_job_writes_window_totals(tmp_path, model_input_dir, gpu_ctx):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    from time_series_spark_b200.jobs.prophet_scorer import frequency_to_future
    models = str(tmp_path / "models")
    ProphetModeler.model(None, {"io": {"input": model_input_dir, "models": models}, "model": {"floor": 0, "cap_multiplier": 1.1}})
    fcast = {"periods": 300, "frequency": "15min", "uncertainty_samples": 500, "seed": 3}
    plain = {"io": {"models": models, "forecasts": str(tmp_path / "plain")}, "forecast": dict(fcast)}
    agg = {"io": {"models": models, "forecasts": str(tmp_path / "fc"), "aggregates": str(tmp_path / "agg")},
           "forecast": dict(fcast, aggregate="1D")}
    _run_scorer(plain, tmp_path, "plain")
    _run_scorer(agg, tmp_path, "agg")
    a = pads.dataset(plain["io"]["forecasts"], format="csv").to_table().drop_columns(["created_timestamp"])
    b = pads.dataset(agg["io"]["forecasts"], format="csv").to_table().drop_columns(["created_timestamp"])
    assert a.num_rows == 600 and a.equals(b)
    strip = lambda d: [ln.split(",", 1)[1] for ln in open(os.path.join(d, "part-00000.csv")).read().splitlines()[1:]]   # noqa: E731
    assert strip(plain["io"]["forecasts"]) == strip(agg["io"]["forecasts"])
    t = pads.dataset(agg["io"]["aggregates"], format="csv").to_table()
    assert t.column_names == ["created_timestamp", "series_id", "dim_id", "window_start", "window_points",
                              "forecast_quantity", "yhat", "yhat_lower", "yhat_upper"]
    got = t.to_pandas()
    rows = b.to_pandas()
    # the windows are the forecast_date groups of the forecast rows, their quantities those rows' totals
    grp = rows.groupby(["series_id", "dim_id", "forecast_date"], sort=False)["forecast_quantity"].agg(["sum", "size"]).reset_index()
    assert len(got) == len(grp) and len(got) >= 6
    assert [str(x)[:10] for x in got["window_start"]] == [str(x) for x in grp["forecast_date"]]
    assert got["forecast_quantity"].tolist() == grp["sum"].tolist() and got["window_points"].tolist() == grp["size"].tolist()
    assert got["dim_id"].tolist() == grp["dim_id"].tolist()
    # and the rows are predict_sums_host's on the decoded models
    mt = pads.dataset(models, format="parquet").to_table()
    fitted, last_ds, info = model_record.decode(mt["model"])
    opts = batched.make_options(growth="logistic" if info["logistic"] else "linear",
                                seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
                                n_changepoints=info["n_changepoints"], uncertainty_samples=500)
    opts.yearly, opts.weekly, opts.daily = info["yearly"], info["weekly"], info["daily"]
    floor = np.asarray(mt["floor"].to_pylist(), np.float32).astype(np.float64)
    cap = np.asarray(mt["cap"].to_pylist(), np.float32).astype(np.float64)
    _, ws = batched.predict_sums_host(gpu_ctx, opts, fitted, frequency_to_future(last_ds, 300, "15min"), floor, cap, DAY, 0, seed=3)
    keep = np.arange(ws.start.shape[1])[None, :] < ws.n_windows[:, None]
    assert np.array_equal(np.repeat(np.asarray(mt["dim_id"].to_pylist()), ws.n_windows), got["dim_id"].to_numpy())
    assert np.array_equal(ws.quantity_sum[keep], got["forecast_quantity"].to_numpy())
    for col, v in (("yhat", ws.yhat_sum), ("yhat_lower", ws.lower), ("yhat_upper", ws.upper)):
        assert np.array_equal(v[keep], got[col].to_numpy()), col             # the CSV prints doubles round-trip
    assert np.all(got["yhat_lower"] < got["yhat_upper"])
