"""Forecast totals per calendar period (DESIGN §17) on the GPU (run with -m gpu on an H100).

* mc_sum_kernel's calendar instance against tests/period_oracle.period_sums at the GPU's parameters: every period bound
  within 1e-9 * y_scale * n_points; yhat_sum the ordered sum of the call's own yhat exactly and within
  1e-12 * y_scale * n_points of the oracle's; quantity_sum, n_points, window_start (the period start) and n_windows
  exact -- both growths and modes, rules M, Q, Q-NOV, Y, Y-JUN, frames at 15 minutes, hours, days, weeks and month starts
  and an irregular grid, across Feb 29 2024, 2100-02-28, year ends and 1969-12 -> 1970-01;
* identities, bit for bit: the pointwise outputs are pb200_predict_*'s; a frame inside one period is the fixed-width
  call with one window over it; the job's W-SUN is its 7D from 1970-01-05;
* sample counts, widths, too few slots, failed models, empty frames, argument errors (nothing launched);
* a model's rows do not depend on its place in the batch; the device call is the host call;
* the scorer job with forecast.aggregate_period on the golden fixture.
"""
import ctypes as C

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.dataset as pads
import pytest

import period_oracle as pdo
from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
from test_gpu_aggregate import _check_empty_slots, _run_scorer
from test_gpu_scorer import _MASK_HIST, _batch, _model, _prep, _take
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

pytestmark = pytest.mark.gpu

H_NS = 3600 * 10**9
DAY = 24 * H_NS
MIN15 = 15 * 60 * 10**9
SUM_TOL = 1e-9
PRED_TOL = 1e-12
RULES = ("M", "Q", "Q-NOV", "Y", "Y-JUN")
_measured = {"sum": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviation():
    yield
    print(f"\n[period sums] max |mc_sum_kernel<CAL> - restatement| / (y_scale * n_points) = {_measured['sum']:.3e}")


def _ns(s):
    return int(pd.Timestamp(s).value)


def _irregular():
    rng = np.random.RandomState(5)
    gaps = rng.randint(1, 40, size=300).astype(np.int64) * (H_NS // 4) + rng.randint(0, 10**9, size=300)
    ds = _ns("2023-12-20") + np.cumsum(gaps)
    ds[40] = _ns("2024-01-01")                       # exactly 00:00 on the 1st
    return np.sort(ds)


# (frame, mask) -- the frames the matrix runs
FRAMES = [
    (_ns("2024-02-27") + MIN15 * np.arange(700, dtype=np.int64), 0),          # 15 minutes over Feb 29 2024, two tiles
    (_ns("2099-12-25") + H_NS * np.arange(600, dtype=np.int64), 6),           # hourly over a year end
    (_ns("2099-11-01") + DAY * np.arange(150, dtype=np.int64), 2),            # daily over 2100-02-28 -> 2100-03-01
    (_ns("1969-11-20") + DAY * np.arange(90, dtype=np.int64), 3),             # daily over 1969-12 -> 1970-01
    (_ns("2023-10-02") + 7 * DAY * np.arange(120, dtype=np.int64), 1),        # pd.offsets.Week(): 28 months, > 16 periods
    (pd.date_range("2020-01-01", periods=40, freq="MS").values.astype("datetime64[ns]").astype(np.int64), 7),   # month starts: 00:00 on the 1st
    (_irregular(), 4),
]


def _models(growth, mode, frames, rng, ncp=25):
    """One model per (frame, mask), its history ending one history step before the frame's first point."""
    frs, oo = [], []
    for fut, mask in frames:
        step, T, _ = _MASK_HIST[mask]
        start = pd.Timestamp(int(fut[0]) - step * T).isoformat()
        p, oopts = _prep(mask, growth, mode, ncp=ncp, start=start)
        frs.append(_model(p, rng))
        oo.append(oopts)
    return frs, oo


def _pad(frames):
    """Frames of unequal length as one [N, H] batch: each row padded by repeating its last point."""
    H = max(f.size for f in frames)
    return np.stack([np.concatenate([f, np.full(H - f.size, f[-1])]) for f in frames])


def _check_period(gpu_ctx, fb, fut, floor, cap, growth, mode, n, width, seed, alias, frs=None, oopts=None, draws=None):
    """Run the calendar call, restate every model's periods, compare; returns (ForecastBatch, WindowSums, draws)."""
    opts = batched.make_options(growth=growth, seasonality_mode=mode, interval_width=width, uncertainty_samples=n)
    _, months, shift = batched.period_rule(alias)
    fc, ws = batched.predict_period_sums_host(gpu_ctx, opts, fb, fut, floor, cap, months, shift, seed=seed)
    draws = draws if draws is not None else {}
    for i in range(fb.n):
        if fb.meta_i32[i, 4] < 0:
            assert ws.n_windows[i] == 0
            _check_empty_slots(ws, i, 0)
            continue
        if i not in draws:
            draws[i] = mcs.draws(fb, i, fut[i], floor[i], cap[i], growth == "logistic", mode == "multiplicative", n, seed)
        start, pts, lo, hi = pdo.period_sums(draws[i], fut[i], alias, width)
        nw = start.size
        assert ws.n_windows[i] == nw, (i, alias, ws.n_windows[i], nw)
        assert np.array_equal(ws.start[i, :nw], start) and np.array_equal(ws.points[i, :nw], pts), (i, alias)
        _check_empty_slots(ws, i, nw)
        ys = fb.meta_f64[i, 0]
        err = max(np.max(np.abs(ws.lower[i, :nw] - lo) / pts), np.max(np.abs(ws.upper[i, :nw] - hi) / pts)) / ys
        assert err <= SUM_TOL, (i, alias, n, width, err)
        _measured["sum"] = max(_measured["sum"], err)
        first, _ = pdo.period_runs(fut[i], alias)
        ref = po.predict(frs[i], fut[i], floor[i], cap[i], oopts[i])["yhat"] if oopts is not None else None
        for j in range(nw):
            s, r = 0.0, 0.0
            for h in range(first[j], first[j + 1]):
                s = s + fc.yhat[i, h]
                if ref is not None:
                    r = r + ref[h]
            assert ws.yhat_sum[i, j] == s, (i, j)
            if ref is not None:
                big = max(1.0, np.max(np.abs(ref[first[j]:first[j + 1]])) / ys)
                assert abs(s - r) <= PRED_TOL * ys * pts[j] * big, (i, j, s, r)
            assert ws.quantity_sum[i, j] == int(fc.yhat_int[i, first[j]:first[j + 1]].astype(np.int64).sum())
    return fc, ws, draws


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_period_sums_match_restatement(gpu_ctx, growth, mode):
    """Every frame of FRAMES (padded to one batch by repeating each frame's last point, which adds points to its last
    period) under each rule of RULES, with a failed model between them."""
    rng = np.random.RandomState(1)
    frs, oo = _models(growth, mode, FRAMES, rng)
    frs.insert(3, frs[0])
    oo.insert(3, oo[0])
    status = np.zeros(len(frs), np.int64)
    status[3] = L.ST_TOO_FEW
    fb = _batch(frs, batched.make_options(growth=growth, seasonality_mode=mode), status)
    frames = [f for f, _ in FRAMES]
    frames.insert(3, frames[0])
    fut = _pad(frames)
    N = fut.shape[0]
    floor = np.zeros(N) if growth == "linear" else rng.uniform(-5, 5, N)
    cap = np.array([fr.prep.cap_value for fr in frs]) + floor
    draws = {}
    counts = {}
    for alias in RULES:
        _, ws, draws = _check_period(gpu_ctx, fb, fut, floor, cap, growth, mode, 1000, 0.8, 7, alias, frs, oo, draws)
        counts[alias] = ws.n_windows.tolist()
    assert counts["M"][5] == 28 and counts["M"][6] == 40          # weekly frame, month starts: more than 16 periods
    assert counts["Y"][4] == 2 and counts["Y"][2] == 2             # the 1969 / 1970 frame spans a year end, as the 2099 one


def test_period_sums_sample_counts_and_widths(gpu_ctx):
    """2, 1000 and 1024 draws x interval widths 0, 0.8 and 1 on the daily frames of FRAMES, under Q-NOV."""
    rng = np.random.RandomState(2)
    frames = [FRAMES[2], FRAMES[3]]
    frs, _ = _models("logistic", "multiplicative", frames, rng)
    fb = _batch(frs, batched.make_options())
    fut = _pad([f for f, _ in frames])
    cap = np.array([fr.prep.cap_value for fr in frs])
    for n in (2, 1000, 1024):
        draws = {}
        for w in (0.0, 0.8, 1.0):
            _, _, draws = _check_period(gpu_ctx, fb, fut, np.zeros(2), cap, "logistic", "multiplicative", n, w, 3, "Q-NOV",
                                        draws=draws)


def _hourly(n=4, first="2024-01-20", H=24 * 60, growth="linear", mode="additive", seed=9):
    rng = np.random.RandomState(seed)
    fut = _ns(first) + H_NS * np.arange(H, dtype=np.int64)
    frs, _ = _models(growth, mode, [(fut, 6)] * n, rng)
    fb = _batch(frs, batched.make_options(growth=growth, seasonality_mode=mode))
    return fb, np.stack([fut] * n), np.array([fr.prep.cap_value for fr in frs])


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("linear", "additive")])
def test_pointwise_outputs_are_predicts_and_one_period_is_one_fixed_window(gpu_ctx, growth, mode):
    """The call's yhat / yhat_int / bounds are pb200_predict_*'s; over a frame inside March 2024 the month's row is the
    fixed-width call's single window from 2024-03-01, bit for bit."""
    fb, fut, cap = _hourly(growth=growth, mode=mode)
    n = fb.n
    opts = batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=1000)
    ref = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(n), cap, seed=4, intervals=True)
    fc, ws = batched.predict_period_sums_host(gpu_ctx, opts, fb, fut, np.zeros(n), cap, 1, 0, seed=4, intervals=True)
    for a, b in ((fc.yhat, ref.yhat), (fc.yhat_int, ref.yhat_int), (fc.yhat_lower, ref.yhat_lower),
                 (fc.yhat_upper, ref.yhat_upper)):
        assert np.array_equal(a, b)
    assert ws.n_windows.tolist() == [3] * n                         # Jan, Feb, Mar
    march = fut[:, (fut[0] >= _ns("2024-03-01"))][:, 1:]           # inside March, not on its first instant
    _, one = batched.predict_period_sums_host(gpu_ctx, opts, fb, march, np.zeros(n), cap, 1, 0, seed=4)
    _, fixed = batched.predict_sums_host(gpu_ctx, opts, fb, march, np.zeros(n), cap, 31 * DAY, _ns("2024-03-01"), seed=4)
    assert one.start.shape == fixed.start.shape == (n, 1) and np.all(one.n_windows == 1)
    for f in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        assert np.array_equal(getattr(one, f), getattr(fixed, f)), f
    assert np.all(one.start == _ns("2024-03-01"))


def test_period_rows_do_not_depend_on_batch_position(gpu_ctx):
    rng = np.random.RandomState(8)
    frames = [FRAMES[k % len(FRAMES)] for k in range(60)]
    frs, _ = _models("logistic", "multiplicative", frames, rng)
    fb = _batch(frs, batched.make_options())
    fut = _pad([f for f, _ in frames])
    cap = np.array([fr.prep.cap_value for fr in frs])
    opts = batched.make_options(uncertainty_samples=1000)
    _, full = batched.predict_period_sums_host(gpu_ctx, opts, fb, fut, np.zeros(60), cap, 3, 1, seed=21)
    idx = np.concatenate([np.arange(40, 55), np.arange(3, 30)[::-1]])
    _, sub = batched.predict_period_sums_host(gpu_ctx, opts, _take(fb, idx), fut[idx], np.zeros(idx.size), cap[idx], 3, 1,
                                              seed=21)
    w = sub.start.shape[1]
    for f in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        a, b = getattr(sub, f), getattr(full, f)[idx]
        assert np.array_equal(a, b if a.ndim == 1 else b[:, :w], equal_nan=True), f


def test_device_call_equals_host_call(gpu_ctx):
    import torch
    fb, fut, cap = _hourly(n=5, H=1500)
    opts = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=300)
    fc, ws = batched.predict_period_sums_host(gpu_ctx, opts, fb, fut, np.zeros(5), cap, 12, 6, seed=4, intervals=True)
    dev = torch.device("cuda", gpu_ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    dfb = batched.FittedBatch(t(fb.params), t(fb.tchange), t(fb.meta_i32), t(fb.meta_i64), t(fb.meta_f64), fb.smax, fb.kmax)
    dfc, dws = batched.predict_period_sums_device(gpu_ctx, opts, dfb, t(fut), t(np.zeros(5)), t(cap), 12, 6, seed=4,
                                                  intervals=True)
    for name in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        assert np.array_equal(getattr(dws, name).cpu().numpy(), getattr(ws, name), equal_nan=True), name
    assert np.array_equal(dfc.yhat.cpu().numpy(), fc.yhat) and np.array_equal(dfc.yhat_lower.cpu().numpy(), fc.yhat_lower)


def _raw(gpu_ctx, opts, fb, fut, wmax, months=1, shift=0, h=None, null=None):
    """pb200_predict_period_sums_host with every argument in the caller's hand; returns (rc, outputs)."""
    h = fut.shape[1] if h is None else h
    slots = max(1, fb.n * max(wmax, 1))
    o = dict(nw=np.full(fb.n, -7, np.int32), start=np.full(slots, -7, np.int64), pts=np.full(slots, -7, np.int32),
             ys=np.full(slots, -7.0), qs=np.full(slots, -7, np.int64), lo=np.full(slots, -7.0), hi=np.full(slots, -7.0),
             yhat=np.full(fut.size + 1, -7.0), yint=np.full(fut.size + 1, -7, np.int32))
    ptr = lambda k: None if null == k else o[k].ctypes.data_as(C.c_void_p)      # noqa: E731
    arr = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)          # noqa: E731
    floor, cap = np.zeros(fb.n), np.ones(fb.n)
    rc = L.load().pb200_predict_period_sums_host(
        gpu_ctx.handle, C.byref(opts), arr(fb.params), arr(fb.tchange), arr(fb.meta_i32), arr(fb.meta_i64),
        arr(fb.meta_f64), fb.n, arr(fut), h, arr(floor), arr(cap), 0, ptr("yhat"), None, None, ptr("yint"), months, shift,
        wmax, ptr("nw"), ptr("start"), ptr("pts"), ptr("ys"), ptr("qs"), ptr("lo"), ptr("hi"))
    return rc, o


def test_argument_errors_too_few_slots_failed_models_and_empty_frames(gpu_ctx):
    fb, fut, cap = _hourly(n=3)                                   # 2024-01-20 .. 2024-03-19: three months
    ok = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=100)
    E_ARG, E_UNSUPPORTED = -1, -4
    cases = [(batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=ns), {}, E_UNSUPPORTED)
             for ns in (0, 1, 1025)]
    cases += [(ok, dict(months=m, shift=s), E_ARG) for m, s in ((0, 0), (2, 0), (3, 3), (12, 12), (1, -1), (6, 0))]
    cases += [(ok, dict(wmax=0), E_ARG)] + [(ok, dict(null=k), E_ARG) for k in ("nw", "start", "lo", "hi", "yhat")]
    before = gpu_ctx.launch_count
    for opts, kw, code in cases:
        rc, o = _raw(gpu_ctx, opts, fb, fut, **dict(dict(wmax=4), **kw))
        assert rc == code, (kw, rc, L.last_error())
        assert all(np.all(v == -7) for v in o.values()), kw
    assert gpu_ctx.launch_count == before
    # too few slots: the true count, the first wmax periods
    rc, full = _raw(gpu_ctx, ok, fb, fut, 5)
    rc2, cut = _raw(gpu_ctx, ok, fb, fut, 2)
    assert rc == 0 and rc2 == 0 and np.all(full["nw"] == 3) and np.all(cut["nw"] == 3)
    for k in ("start", "pts", "ys", "qs", "lo", "hi"):
        assert np.array_equal(cut[k].reshape(3, 2), full[k].reshape(3, 5)[:, :2]), k
    assert full["start"].reshape(3, 5)[0, :3].tolist() == [_ns("2024-01-01"), _ns("2024-02-01"), _ns("2024-03-01")]
    # failed models; no point at all
    fb.meta_i32[1, 4] = L.ST_TOO_FEW
    fc, ws = batched.predict_period_sums_host(gpu_ctx, ok, fb, fut, np.zeros(3), cap, 1, 0)
    assert ws.n_windows.tolist() == [3, 0, 3] and np.all(np.isnan(fc.yhat[1]))
    _check_empty_slots(ws, 1, 0)
    fch, wsh = batched.predict_period_sums_host(gpu_ctx, ok, fb, fut[:, :0], np.zeros(3), cap, 3, 0)
    assert fch.yhat.shape == (3, 0) and wsh.n_windows.tolist() == [0, 0, 0] and wsh.start.shape == (3, 1)
    for i in range(3):
        _check_empty_slots(wsh, i, 0)
    # a first period start before the int64-ns minimum is refused before anything runs
    early = np.stack([_ns("1678-01-15") + DAY * np.arange(3, dtype=np.int64)] * 3)
    before = gpu_ctx.launch_count
    with pytest.raises(ValueError, match="1677-09-21"):
        batched.predict_period_sums_host(gpu_ctx, ok, fb, early, np.zeros(3), cap, 12, 11)
    assert gpu_ctx.launch_count == before


def test_scorer_job_writes_period_totals(tmp_path, model_input_dir, gpu_ctx):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    from time_series_spark_b200.jobs.prophet_scorer import AGGREGATE_SCHEMA, forecast_time_series
    models = str(tmp_path / "models")
    ProphetModeler.model(None, {"io": {"input": model_input_dir, "models": models}, "model": {"floor": 0, "cap_multiplier": 1.1}})
    fcast = {"periods": 2208, "frequency": "1h", "uncertainty_samples": 500, "seed": 3}

    def run(name, **kw):
        cfg = {"io": {"models": models, "forecasts": str(tmp_path / f"fc_{name}"), "aggregates": str(tmp_path / name)},
               "forecast": dict(fcast, **kw)}
        _run_scorer(cfg, tmp_path, name)
        return (pads.dataset(cfg["io"]["forecasts"], format="csv").to_table().to_pandas(),
                pads.dataset(cfg["io"]["aggregates"], format="csv").to_table().drop_columns(["created_timestamp"]))

    rows, month = run("month", aggregate_period="M")
    assert month.column_names == ["series_id", "dim_id", "window_start", "window_points", "forecast_quantity", "yhat",
                                  "yhat_lower", "yhat_upper"]
    got = month.to_pandas()
    # each row is the sum of the forecast rows of its calendar month
    rows["month"] = pd.to_datetime(rows["forecast_date"]).dt.to_period("M").dt.start_time
    grp = rows.groupby(["series_id", "dim_id", "month"], sort=False)["forecast_quantity"].agg(["sum", "size"]).reset_index()
    assert len(got) == len(grp) and len(got) >= 8
    assert pd.to_datetime(got["window_start"]).dt.tz_localize(None).tolist() == grp["month"].tolist()
    assert got["forecast_quantity"].tolist() == grp["sum"].tolist() and got["window_points"].tolist() == grp["size"].tolist()
    assert np.all(got["yhat_lower"] < got["yhat_upper"])
    # W-SUN is 7D from Monday 1970-01-05
    _, week = run("week", aggregate_period="W-SUN")
    _, fixed = run("fixed", aggregate="7D", aggregate_origin="1970-01-05")
    assert week.num_rows > 0 and week.equals(fixed)
    # an empty shard hands back the same columns
    op = forecast_time_series({"io": {"aggregates": "a"}, "forecast": dict(fcast, aggregate_period="Q")})
    op.apply_batched(pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32())}),
                     ["series_id", "dim_id"])
    assert op.aggregates.schema == AGGREGATE_SCHEMA and op.aggregates.num_rows == 0
