"""Backtest window totals (DESIGN §14) on the GPU (run with -m gpu on an H100).

* cv_window_kernel against tests/window_backtest_oracle.window_rows: n_windows, starts and points exact, y / yhat sums bit
  for bit, for int32 / float32 / float64 y, on an irregular batch with more than sms * 32 entries;
* pb200_predict_sums_anchored_device against tests/window_oracle.window_sums (origin c + 1, the pair's unpadded frame)
  within 1e-9 * y_scale * n_points; its pointwise outputs, its plain-origin case, its one-point windows and a padded
  entry against the existing entry points, bit for bit; both growths and both seasonality modes; failed models;
* cross_validation_device(aggregate_ns=...) against the oracle's window rows and performance_metrics, the unchanged
  outputs with and without the key, batch and chunk independence, and the job on the golden fixture.
"""
import os
import sys

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import backtest_oracle as bo  # noqa: E402
import window_backtest_oracle as wbo  # noqa: E402
import window_oracle as wo  # noqa: E402
from oracle import mc_stream as mcs  # noqa: E402
from test_gpu_backtest import _mixed_batch  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched  # noqa: E402

pytestmark = pytest.mark.gpu

H = 3600 * 10**9
D = 24 * H
MIN15 = 15 * 60 * 10**9
INT64_MIN = -2**63
HORIZON, PERIOD, INITIAL = D, D // 2, 3 * D
FLOOR, CAPM = 0.0, 1.1
SUM_TOL = 1e-9
_measured = {"sum": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviation():
    yield
    print(f"\n[backtest windows] max |window bound - restatement| / (y_scale * n_points) = {_measured['sum']:.3e}")


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---------------------------------------------------------------------------------------------------------------------
# cv_window_kernel
# ---------------------------------------------------------------------------------------------------------------------
def _irregular_batch(rng, n_series, dtype):
    """Hourly-grid series with 1-3 hour steps and one gap of 7-40 hours each (longer than every width below but the
    day), 300-500 rows, start times off the hour; y of the given type with -0.0, subnormals and large values."""
    parts = []
    t0 = 1_600_000_000 * 10**9 + 7 * MIN15
    for s in range(n_series):
        n = int(rng.randint(300, 500))
        steps = rng.randint(1, 4, n).astype(np.int64) * H
        steps[int(rng.randint(60, n - 60))] += int(rng.randint(7, 41)) * H
        ds = t0 + (s % 4) * MIN15 + np.cumsum(steps)
        if dtype == np.int32:
            y = rng.randint(-2**31, 2**31 - 1, n, dtype=np.int64).astype(np.int32)
        else:
            y = rng.normal(0, 50, n).astype(dtype)
            y[::17] = -0.0
            y[5::23] = np.finfo(dtype).smallest_subnormal * rng.randint(1, 9)
            y[7::29] = (1e30 if dtype == np.float32 else 1e300) * rng.choice([-1, 1])
        parts.append((ds, y))
    off = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), off


@pytest.mark.parametrize("dtype", [np.int32, np.float32, np.float64])
def test_window_kernel_matches_oracle_past_the_stride_loop(gpu_ctx, sms, dtype):
    import torch
    rng = np.random.RandomState({np.int32: 1, np.float32: 2, np.float64: 3}[dtype])
    ds, y, off = _irregular_batch(rng, 70, dtype)
    H_, P_, I_ = D, 6 * H, 2 * D
    plan = batched.cv_plan_device(gpu_ctx, batched.make_options(), _cuda(ds), off, H_, P_, I_)
    assert not plan.err.any()
    n = plan.n_pairs
    assert n > sms * 32, (n, sms)
    pairs = rng.permutation(n).astype(np.int64)                     # gathered order: any order of the plan's pairs
    he, we, cut = plan.hist_end.cpu().numpy(), plan.win_end.cpu().numpy(), plan.cutoff.cpu().numpy()
    wl = (we - he)[pairs]
    hmax = int(wl.max())
    yhat = rng.normal(0, 50, (n, hmax))
    yhat[:, ::11] = -0.0
    yhat[np.arange(hmax)[None, :] >= wl[:, None]] = np.nan          # the frame's padding is never read
    dy = _cuda(y)
    for W in (H, 6 * H, D):                                          # the grid step, a divisor, the horizon
        got = batched.cv_windows_device(gpu_ctx, _cuda(ds), dy, plan, _cuda(pairs), _cuda(yhat), W)
        got = {k: v.cpu().numpy() for k, v in got.items()}
        wmax = got["start"].shape[1]
        short = 0
        for k in range(n):
            p = pairs[k]
            rows = slice(he[p], we[p])
            ref = wbo.window_rows(ds[rows], np.full(we[p] - he[p], cut[p]), y[rows].astype(np.float64), yhat[k, :wl[k]], W)
            nw = ref["horizon"].size
            assert got["n_windows"][k] == nw, (W, k)
            assert got["start"][k, :nw].tolist() == (cut[p] + ref["horizon"] - W).tolist()
            assert got["points"][k, :nw].tolist() == ref["points"].tolist()
            assert got["y_sum"][k, :nw].tobytes() == ref["y"].tobytes(), (W, k)
            assert got["yhat_sum"][k, :nw].tobytes() == ref["yhat"].tobytes(), (W, k)
            assert np.all(got["start"][k, nw:] == INT64_MIN) and np.all(got["points"][k, nw:] == 0)
            assert np.all(np.isnan(got["y_sum"][k, nw:])) and np.all(np.isnan(got["yhat_sum"][k, nw:]))
            short += nw < D // W
        assert wmax == hmax and (short > 0 or W == D)              # gaps leave windows empty
    # a count above wmax: the true count, the first wmax slots (through the C entry point: the Python wrapper refuses)
    n_w = torch.zeros(n, dtype=torch.int32, device="cuda")
    outs = [torch.empty((n, 2), dtype=t, device="cuda") for t in (torch.int64, torch.int32, torch.float64, torch.float64)]
    yh = _cuda(yhat)
    dp = _cuda(pairs)
    L.check(L.load().pb200_cv_windows_device(gpu_ctx.handle, _cuda(ds).data_ptr(), dy.data_ptr(), batched._y_dtype(dy),
                                             plan.cutoff.data_ptr(), plan.hist_end.data_ptr(), plan.win_end.data_ptr(),
                                             dp.data_ptr(), n, yh.data_ptr(), hmax, H, 2, n_w.data_ptr(),
                                             *(o.data_ptr() for o in outs)), "pb200_cv_windows_device")
    gpu_ctx.synchronize()
    full = batched.cv_windows_device(gpu_ctx, _cuda(ds), dy, plan, dp, yh, H)
    assert n_w.cpu().numpy().tolist() == full["n_windows"].cpu().numpy().tolist()
    for o, k in zip(outs, ("start", "points", "y_sum", "yhat_sum")):
        assert o.cpu().numpy().tobytes() == full[k][:, :2].contiguous().cpu().numpy().tobytes(), k


def test_window_kernel_argument_errors(gpu_ctx):
    """Bad sizes, widths, y types and null pointers are PB200_E_ARG (-1) before anything is launched."""
    lib = L.load()
    # ctx, ds, y, y_dtype, cutoff, hist_end, win_end, pairs, n, yhat, hmax, width_ns, wmax, five outputs
    base = [gpu_ctx.handle, 1, 1, 0, 1, 1, 1, 1, 4, 1, 8, H, 8, 1, 1, 1, 1, 1]
    before = gpu_ctx.launch_count
    for i, bad in ((11, 0), (11, -H), (12, 0), (10, 0), (3, 3), (8, -1), (9, None), (17, None)):
        args = list(base)
        args[i] = bad
        assert lib.pb200_cv_windows_device(*args) == -1, (i, bad)
    args = list(base)
    args[8] = 0                                                      # nothing to do
    assert lib.pb200_cv_windows_device(*args) == 0
    assert gpu_ctx.launch_count == before


# ---------------------------------------------------------------------------------------------------------------------
# pb200_predict_sums_anchored_device
# ---------------------------------------------------------------------------------------------------------------------
def _small_batch():
    """Two config #3 series (15-minute grid, 96 held-out rows per pair) and two irregular hourly series with a gap
    longer than the horizon (padded frames, windows emptied by the gap): the first 2 + last 2 of _mixed_batch."""
    ds, y, off = _mixed_batch()
    keep = [0, 1, 10, 11]
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in keep]
    o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), o2


def _frames(ds, off, res):
    """Per plan pair: the held-out frame padded to hmax by its last timestamp (cv_gather's), its length, the cutoff."""
    he, we = [], []
    for p in range(res.pair_series.size):
        s = int(res.pair_series[p])
        a, b = off[s], off[s + 1]
        he.append(a + int(np.searchsorted(ds[a:b], res.pair_cutoff[p], side="right")))
        we.append(a + int(np.searchsorted(ds[a:b], res.pair_cutoff[p] + HORIZON, side="right")))
    he, we = np.array(he), np.array(we)
    wl = we - he
    hmax = int(wl.max())
    idx = he[:, None] + np.minimum(np.arange(hmax)[None, :], wl[:, None] - 1)
    return ds[idx], wl, res.pair_cutoff.astype(np.int64)


def _device_fits(f):
    return batched.FittedBatch(*(_cuda(getattr(f, k)) for k in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")),
                               f.smax, f.kmax)


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_anchored_sums(gpu_ctx, growth, mode):
    import torch
    ds, y, off = _small_batch()
    opts = batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=200)
    capv = np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])])
    res = batched.cross_validation_device(gpu_ctx, opts, _cuda(ds), _cuda(y), off, FLOOR, _cuda(capv), HORIZON, PERIOD,
                                          INITIAL, keep_fits=True)
    assert (res.pair_status >= 0).all()
    fut_h, wl, cut = _frames(ds, off, res)
    P, hmax = fut_h.shape
    assert (wl < hmax).any() and (wl == hmax).any()
    fb = _device_fits(res.fitted)
    fut = _cuda(fut_h)
    floor = torch.full((P,), FLOOR, dtype=torch.float64, device="cuda")
    cap = _cuda(capv[res.pair_series])
    seed, W = 5, 6 * H
    fc, ws = batched.predict_sums_anchored_device(gpu_ctx, opts, fb, fut, floor, cap, W, _cuda(cut + 1),
                                                  _cuda(wl.astype(np.int32)), seed=seed, intervals=True)
    # pointwise outputs: pb200_predict_device's on the same frame
    ref = batched.predict_batch_device(gpu_ctx, opts, fb, fut, floor, cap, seed=seed, intervals=True)
    for k in ("yhat", "yhat_lower", "yhat_upper", "yhat_int"):
        assert getattr(fc, k).cpu().numpy().tobytes() == getattr(ref, k).cpu().numpy().tobytes(), k
    wsh = {k: getattr(ws, k).cpu().numpy() for k in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower",
                                                     "upper")}
    # yhat_sum and the slots: cv_window_kernel's over the same yhat frame
    plan = batched.cv_plan_device(gpu_ctx, opts, _cuda(ds), off, HORIZON, PERIOD, INITIAL)
    cw = batched.cv_windows_device(gpu_ctx, _cuda(ds), _cuda(y), plan, _cuda(np.arange(P, dtype=np.int64)), fc.yhat, W)
    cw = {k: v.cpu().numpy() for k, v in cw.items()}
    assert wsh["n_windows"].tolist() == cw["n_windows"].tolist()
    for p in range(P):
        nw = int(cw["n_windows"][p])
        assert wsh["start"][p, :nw].tolist() == (cw["start"][p, :nw] + 1).tolist()      # origin c + 1 against c
        assert wsh["points"][p, :nw].tolist() == cw["points"][p, :nw].tolist()
        assert wsh["yhat_sum"][p, :nw].tobytes() == cw["yhat_sum"][p, :nw].tobytes()
    # bounds: the restatement on the pair's unpadded frame, origin c + 1
    logi, mult = growth == "logistic", mode == "multiplicative"
    picks = sorted(set(np.flatnonzero(wl < hmax)[:3].tolist() + np.flatnonzero(wl == hmax)[:2].tolist()))
    for p in picks:
        fr = fut_h[p, :wl[p]]
        d = mcs.draws(res.fitted, p, fr, FLOOR, capv[res.pair_series[p]], logi, mult, opts.uncertainty_samples, seed)
        start, pts, lo, hi = wo.window_sums(d, fr, W, int(cut[p]) + 1, opts.interval_width)
        nw = start.size
        assert wsh["n_windows"][p] == nw
        assert wsh["start"][p, :nw].tolist() == start.tolist() and wsh["points"][p, :nw].tolist() == pts.tolist()
        ys = float(res.fitted.meta_f64[p, 0])
        err = max(np.max(np.abs(wsh["lower"][p, :nw] - lo) / pts), np.max(np.abs(wsh["upper"][p, :nw] - hi) / pts)) / ys
        assert err <= SUM_TOL, (p, err)
        _measured["sum"] = max(_measured["sum"], err)
    # a padded entry: the same windows as the model alone on its unpadded frame
    p = int(np.flatnonzero(wl < hmax)[0])
    one = batched.FittedBatch(*(x[p:p + 1] for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)),
                              fb.smax, fb.kmax)
    _, w1 = batched.predict_sums_device(gpu_ctx, opts, one, fut[p:p + 1, :wl[p]].contiguous(), floor[:1], cap[p:p + 1],
                                        W, origin_ns=int(cut[p]) + 1, seed=seed)
    nw = int(w1.n_windows[0])
    assert nw == wsh["n_windows"][p]
    for k in ("start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        assert getattr(w1, k)[0, :nw].cpu().numpy().tobytes() == wsh[k][p, :nw].tobytes(), k
    # one origin for all and full frames: pb200_predict_sums_device, byte for byte
    o = int(cut.min()) - 3 * MIN15
    fc2, ws2 = batched.predict_sums_device(gpu_ctx, opts, fb, fut, floor, cap, W, origin_ns=o, seed=seed, intervals=True)
    fc3, ws3 = batched.predict_sums_anchored_device(gpu_ctx, opts, fb, fut, floor, cap, W, _cuda(np.full(P, o)),
                                                    _cuda(np.full(P, hmax, np.int32)), seed=seed, intervals=True,
                                                    wmax=int(ws2.start.shape[1]))
    for k in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        assert getattr(ws2, k).cpu().numpy().tobytes() == getattr(ws3, k).cpu().numpy().tobytes(), k
    for k in ("yhat", "yhat_lower", "yhat_upper", "yhat_int"):
        assert getattr(fc2, k).cpu().numpy().tobytes() == getattr(fc3, k).cpu().numpy().tobytes(), k
    # windows of one point (every step here is >= 15 minutes): the pointwise bounds, bit for bit
    _, w15 = batched.predict_sums_anchored_device(gpu_ctx, opts, fb, fut, floor, cap, MIN15, _cuda(cut + 1),
                                                  _cuda(wl.astype(np.int32)), seed=seed)
    lo_p, hi_p = fc.yhat_lower.cpu().numpy(), fc.yhat_upper.cpu().numpy()
    assert w15.n_windows.cpu().numpy().tolist() == wl.tolist()
    w15l, w15u = w15.lower.cpu().numpy(), w15.upper.cpu().numpy()
    for p in range(P):
        assert w15l[p, :wl[p]].tobytes() == lo_p[p, :wl[p]].tobytes()
        assert w15u[p, :wl[p]].tobytes() == hi_p[p, :wl[p]].tobytes()
    # failed models have no window; the others keep their bits
    bad = np.arange(P) % 5 == 2
    fbad = _device_fits(res.fitted)
    fbad.meta_i32[_cuda(np.flatnonzero(bad)), 4] = L.ST_TOO_FEW
    _, wb = batched.predict_sums_anchored_device(gpu_ctx, opts, fbad, fut, floor, cap, W, _cuda(cut + 1),
                                                 _cuda(wl.astype(np.int32)), seed=seed, intervals=True,
                                                 wmax=int(ws.start.shape[1]))
    nb = wb.n_windows.cpu().numpy()
    assert np.all(nb[bad] == 0) and np.array_equal(nb[~bad], wsh["n_windows"][~bad])
    assert np.all(np.isnan(wb.lower.cpu().numpy()[bad]))
    for k in ("start", "points", "yhat_sum", "quantity_sum", "lower", "upper"):
        assert getattr(wb, k).cpu().numpy()[~bad].tobytes() == wsh[k][~bad].tobytes(), k


def test_anchored_sums_argument_errors(gpu_ctx):
    import torch
    ds, y, off = _small_batch()
    opts = batched.make_options(uncertainty_samples=100)
    capv = np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])])
    res = batched.cross_validation_device(gpu_ctx, batched.make_options(), _cuda(ds), _cuda(y), off, FLOOR, _cuda(capv),
                                          HORIZON, PERIOD, INITIAL, keep_fits=True)
    fut_h, wl, cut = _frames(ds, off, res)
    fb = _device_fits(res.fitted)
    P = fut_h.shape[0]
    floor = torch.zeros(P, dtype=torch.float64, device="cuda")
    cap = _cuda(capv[res.pair_series])
    before = gpu_ctx.launch_count
    with pytest.raises(L.Pb200Error, match="null pointer"):
        batched.L.check(L.load().pb200_predict_sums_anchored_device(
            gpu_ctx.handle, batched.C.byref(opts), fb.params.data_ptr(), fb.tchange.data_ptr(), fb.meta_i32.data_ptr(),
            fb.meta_i64.data_ptr(), fb.meta_f64.data_ptr(), P, _cuda(fut_h).data_ptr(), fut_h.shape[1], floor.data_ptr(),
            cap.data_ptr(), 0, 1, None, None, 1, H, None, None, 4, 1, 1, 1, 1, 1, 1, 1), "anchored")
    with pytest.raises(ValueError, match="width_ns"):
        batched.predict_sums_anchored_device(gpu_ctx, opts, fb, _cuda(fut_h), floor, cap, 0, _cuda(cut + 1),
                                             _cuda(wl.astype(np.int32)))
    assert gpu_ctx.launch_count == before


# ---------------------------------------------------------------------------------------------------------------------
# cross_validation_device(aggregate_ns=...) and the job
# ---------------------------------------------------------------------------------------------------------------------
KEEP = [0, 1, 2, 3, 4, 8, 9, 10, 11]      # config #3 and irregular series: classes below the fit's dispatch thresholds


@pytest.fixture(scope="module")
def cv_batch():
    ds, y, off = _mixed_batch()
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in KEEP]
    o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), o2


def _cv(ctx, ds, y, off, intervals=True, budget=None, W=None):
    opts = batched.make_options(uncertainty_samples=200 if intervals else 0)
    cap = _cuda(np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])]))
    return batched.cross_validation_device(ctx, opts, _cuda(ds), _cuda(y), off, FLOOR, cap, HORIZON, PERIOD, INITIAL,
                                           intervals=intervals, seed=3, rolling_window=0.1, _row_budget=budget,
                                           aggregate_ns=W)


@pytest.fixture(scope="module")
def cv_runs(gpu_ctx, cv_batch):
    ds, y, off = cv_batch
    return {"plain": _cv(gpu_ctx, ds, y, off), "6h": _cv(gpu_ctx, ds, y, off, W=6 * H),
            "1D": _cv(gpu_ctx, ds, y, off, W=D), "point_6h": _cv(gpu_ctx, ds, y, off, intervals=False, W=6 * H),
            "point": _cv(gpu_ctx, ds, y, off, intervals=False)}


def _result_bytes(res):
    out = {}
    for k in ("pair_series", "pair_cutoff", "pair_status", "pair_mask", "row_series", "ds", "cutoff", "y", "yhat",
              "yhat_lower", "yhat_upper"):
        v = getattr(res, k)
        out[k] = None if v is None else v.tobytes()
    for k, v in res.metrics.items():
        out["m_" + k] = None if v is None else v.tobytes()
    return out


def test_existing_outputs_unchanged_by_the_key(cv_runs):
    assert cv_runs["plain"].windows is None and cv_runs["point"].windows is None
    assert _result_bytes(cv_runs["6h"]) == _result_bytes(cv_runs["plain"])
    assert _result_bytes(cv_runs["1D"]) == _result_bytes(cv_runs["plain"])
    assert _result_bytes(cv_runs["point_6h"]) == _result_bytes(cv_runs["point"])


@pytest.mark.parametrize("run,W", [("6h", 6 * H), ("1D", D), ("point_6h", 6 * H)])
def test_window_rows_and_metrics_match_oracle(cv_runs, cv_batch, run, W):
    res = cv_runs[run]
    w = res.windows
    iv = run != "point_6h"
    assert w.width_ns == W and (w.yhat_lower is not None) == iv and (w.metrics["coverage"] is not None) == iv
    n_series = cv_batch[2].size - 1
    for s in range(n_series):
        r = res.row_series == s
        ref = wbo.window_rows(res.ds[r], res.cutoff[r], res.y[r], res.yhat[r], W)
        g = w.series == s
        assert w.cutoff[g].tolist() == ref["cutoff"].tolist()
        assert w.horizon[g].tolist() == ref["horizon"].tolist()
        assert w.points[g].tolist() == ref["points"].tolist()
        assert w.y[g].tobytes() == ref["y"].tobytes() and w.yhat[g].tobytes() == ref["yhat"].tobytes()
        want = bo.performance_metrics(w.horizon[g], w.y[g], w.yhat[g], w.yhat_lower[g] if iv else None,
                                      w.yhat_upper[g] if iv else None, 0.1)
        m = w.metrics
        gm = m["series"] == s
        assert m["horizon"][gm].tolist() == want["horizon"].tolist()
        if iv:
            assert m["coverage"][gm].tolist() == want["coverage"].tolist()
            assert np.all(w.yhat_lower[g] <= w.yhat_upper[g])
        for k in ("mse", "rmse", "mae", "mape"):
            np.testing.assert_allclose(m[k][gm], want[k], rtol=1e-12, atol=0, equal_nan=True)
    # every held-out row is in exactly one window of its pair
    assert int(w.points.sum()) == res.ds.size
    assert set(np.unique(w.horizon).tolist()) <= set(range(W, HORIZON + 1, W))


def test_window_bounds_match_restatement(cv_runs, cv_batch, gpu_ctx):
    """The window bounds of a few pairs of the end-to-end run against window_sums on the draws of the pair's fit (refit
    here with keep_fits: the same bits, as the fits do not depend on the call's other outputs)."""
    ds, y, off = cv_batch
    res = cv_runs["6h"]
    opts = batched.make_options(uncertainty_samples=200)
    cap = np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])])
    fits = batched.cross_validation_device(gpu_ctx, opts, _cuda(ds), _cuda(y), off, FLOOR, _cuda(cap), HORIZON, PERIOD,
                                           INITIAL, keep_fits=True).fitted
    w = res.windows
    rng = np.random.RandomState(0)
    for p in rng.choice(res.pair_series.size, 6, replace=False):
        s, c = int(res.pair_series[p]), int(res.pair_cutoff[p])
        rows = (res.row_series == s) & (res.cutoff == c)
        fr = res.ds[rows]
        d = mcs.draws(fits, int(p), fr, FLOOR, cap[s], True, True, opts.uncertainty_samples, 3)
        _, pts, lo, hi = wo.window_sums(d, fr, 6 * H, c + 1, opts.interval_width)
        g = (w.series == s) & (w.cutoff == c)
        assert w.points[g].tolist() == pts.tolist()
        ys = float(fits.meta_f64[p, 0])
        err = max(np.max(np.abs(w.yhat_lower[g] - lo) / pts), np.max(np.abs(w.yhat_upper[g] - hi) / pts)) / ys
        assert err <= SUM_TOL, (p, err)
        _measured["sum"] = max(_measured["sum"], err)


def _window_view(res, s):
    w = res.windows
    g = w.series == s
    gm = w.metrics["series"] == s
    out = {k: getattr(w, k)[g].tobytes() for k in ("cutoff", "horizon", "points", "y", "yhat", "yhat_lower", "yhat_upper")}
    out.update({"m_" + k: w.metrics[k][gm].tobytes() for k in ("horizon", "mse", "rmse", "mae", "mape", "coverage")})
    return out


def test_windows_independent_of_batch_and_chunks(gpu_ctx, cv_batch, cv_runs):
    ds, y, off = cv_batch
    full = cv_runs["6h"]
    tiny = _cv(gpu_ctx, ds, y, off, budget=1, W=6 * H)
    pick = [7, 2, 8, 5, 0]
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in pick]
    o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    sub = _cv(gpu_ctx, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), o2, W=6 * H)
    for s in range(off.size - 1):
        a, b = _window_view(full, s), _window_view(tiny, s)
        assert [k for k in a if a[k] != b[k]] == [], f"series {s}, chunked"
    for j, s in enumerate(pick):
        a, b = _window_view(full, s), _window_view(sub, j)
        assert [k for k in a if a[k] != b[k]] == [], f"series {s}, sub-batch position {j}"


def _config(tmp_path, inp, rows=True, **bt):
    cfg = {"io": {"input": inp, "metrics": str(tmp_path / "metrics"), "window_metrics": str(tmp_path / "wm")},
           "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": {"horizon": "30 days", "period": "15 days", "initial": "180 days", **bt}}
    if rows:
        cfg["io"]["cv_rows"] = str(tmp_path / "rows")
        cfg["io"]["window_rows"] = str(tmp_path / "wr")
    return cfg


WM_COLS = ["series_id", "dim_id", "horizon", "mse", "rmse", "mae", "mape"]
WR_COLS = ["series_id", "dim_id", "cutoff", "horizon", "window_points", "y", "yhat"]


@pytest.mark.parametrize("intervals", [True, False])
def test_job_on_golden_fixture(tmp_path, model_input_dir, intervals):
    import shutil
    from time_series_spark_b200.jobs.prophet_backtest import ProphetBacktester
    bt = dict(intervals=intervals, uncertainty_samples=100) if intervals else {}
    m0, r0 = ProphetBacktester.run(None, _config(tmp_path, model_input_dir, **bt))
    base_m, base_r = pq.read_table(str(tmp_path / "metrics")), pq.read_table(str(tmp_path / "rows"))
    for d in ("metrics", "rows"):
        shutil.rmtree(str(tmp_path / d))
    m1, r1 = ProphetBacktester.run(None, _config(tmp_path, model_input_dir, aggregate="10 days", **bt))
    # the existing outputs are what they are without the key
    assert pq.read_table(str(tmp_path / "metrics")).equals(base_m) and pq.read_table(str(tmp_path / "rows")).equals(base_r)
    wm, wr = pq.read_table(str(tmp_path / "wm")), pq.read_table(str(tmp_path / "wr"))
    extra = ["coverage"] if intervals else []
    assert wm.schema.names == WM_COLS + extra and wm.schema.field("horizon").type == pa.duration("ns")
    assert wr.schema.names == WR_COLS + (["yhat_lower", "yhat_upper"] if intervals else [])
    assert wr.schema.field("cutoff").type == pa.timestamp("ns") and wr.schema.field("window_points").type == pa.int32()
    assert wr["y"].type == pa.float64()
    assert wm.num_rows > 0 and wr.num_rows > 0
    assert set(wm["horizon"].cast(pa.int64()).to_pylist()) <= {10 * D, 20 * D, 30 * D}
    # each (dim_id, cutoff): the windows hold the held-out rows, and their y sums are the rows' in order
    rows = base_r.to_pandas()
    for (dim, cut), g in wr.to_pandas().groupby(["dim_id", "cutoff"]):
        src = rows[(rows.dim_id == dim) & (rows.cutoff == cut)]
        assert int(g.window_points.sum()) == len(src)
        ref = wbo.window_rows(src.ds.values.astype(np.int64), src.cutoff.values.astype(np.int64),
                             src.y.values.astype(np.float64), src.yhat.values, 10 * D)
        assert g.y.values.tobytes() == ref["y"].tobytes() and g.yhat.values.tobytes() == ref["yhat"].tobytes()
    if intervals:
        c = wm["coverage"].to_numpy()
        assert np.all((c >= 0) & (c <= 1))


@pytest.mark.parametrize("intervals", [True, False])
def test_job_empty_shard_schema(tmp_path, intervals):
    from time_series_spark_b200.jobs import prophet_backtest as pb
    tbl = pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32()),
                    "ds": pa.array([], pa.timestamp("ns")), "y": pa.array([], pa.int32())})
    cfg = {"io": {"metrics": str(tmp_path / "m"), "window_metrics": str(tmp_path / "wm"), "window_rows": str(tmp_path / "wr")},
           "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": {"horizon": "1 days", "aggregate": "8h", "intervals": intervals}}
    job = pb.ProphetBacktester(cfg)
    metrics, _ = job.backtest(tbl)
    wm, wr = job.window_outputs
    extra = ["coverage"] if intervals else []
    assert wm.num_rows == 0 and wm.schema.names == WM_COLS + extra
    assert wr.num_rows == 0 and wr.schema.names == WR_COLS + (["yhat_lower", "yhat_upper"] if intervals else [])
    assert wm.schema.field("horizon").type == pa.duration("ns") and wr.schema.field("horizon").type == pa.duration("ns")
    job.persist(metrics, None)
    assert pq.read_table(str(tmp_path / "wm")).schema.names == wm.schema.names


def test_job_failed_fit_rule_covers_the_windows(capsys):
    import copy
    import torch
    from time_series_spark_b200 import synth
    from time_series_spark_b200.jobs import prophet_backtest as pb
    from time_series_spark_b200.jobs.prophet_modeler import get_context
    b = synth.config3(n=4)
    ctx = get_context()
    cap = torch.tensor([float(b.y[a:e].max()) * 1.1 for a, e in zip(b.offsets[:-1], b.offsets[1:])], dtype=torch.float64).cuda()
    res = batched.cross_validation_device(ctx, batched.make_options(), torch.from_numpy(b.ds).cuda(),
                                          torch.from_numpy(b.y.astype(np.int32)).cuda(), b.offsets, 0.0, cap, D, D // 2,
                                          3 * D, rolling_window=0.1, aggregate_ns=8 * H)
    res2 = copy.deepcopy(res)
    res2.pair_status[np.flatnonzero(res2.pair_series == 1)[3]] = -1
    sid, did = np.arange(b.n) + 100, np.full(b.n, 3)
    m_ok, r_ok = pb.assemble_window_outputs(sid, did, res)
    m_bad, r_bad = pb.assemble_window_outputs(sid, did, res2)
    assert 101 in m_ok["series_id"].to_pylist() and 101 not in m_bad["series_id"].to_pylist()
    assert 101 not in r_bad["series_id"].to_pylist()
    assert r_bad.num_rows == r_ok.num_rows - r_ok["series_id"].to_pylist().count(101)
    # 22 cutoffs x 3 windows of 32 rows per series
    assert r_ok.num_rows == b.n * 22 * 3 and set(r_ok["window_points"].to_pylist()) == {32}
