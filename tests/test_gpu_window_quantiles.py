"""Quantiles of window and calendar-period totals (DESIGN §21) on the GPU (run with -m gpu on an H100).

* identities, byte for byte, for both growths and modes on fixed, anchored and calendar windows: the planes at the
  bounds' percentiles are lower / upper; every pre-existing output is the call's without levels; one-point windows are
  pb200_predict_quantiles_*'s pointwise planes;
* every plane within 1e-9 * y_scale * n_points of window_quantile_oracle on mc_stream's draws (the tolerance of the
  window bounds, §13 / §17), at Q = 1, 9, 32, unsorted and repeated levels, 0 and 100, n_samples 2, 3, 1000, 1024,
  crowded rows, more windows than wmax, a batch larger than the SM count;
* failed models are NaN, a model's planes do not depend on its place in the batch, refusals launch nothing;
* the backtest's CvWindows.yhat_q and quantile_metrics, the backtest job, the scorer job on one and two ranks.
"""
import ctypes as C

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import quantile_oracle as qo
import window_oracle as wo
import window_quantile_oracle as wqo
from oracle import mc_stream as mcs
from test_gpu_backtest_windows import _frames
from test_gpu_quantiles import _check_quantile_metrics, _crowded, _quant_host
from test_gpu_quantiles import _result_bytes as _cv_bytes
from test_gpu_backtest import _mixed_batch
from test_gpu_scorer import ALL_MASKS, _batch, _future, _model, _prep, _take
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

pytestmark = pytest.mark.gpu

H_NS = 3600 * 10**9
DAY = 24 * H_NS
SUM_TOL = 1e-9        # |plane - restatement| / (y_scale * n_points)
E_ARG, E_UNSUPPORTED = -1, -4
DECILES = [0.1 * k for k in range(1, 10)]
GROWTH_MODES = [("logistic", "multiplicative"), ("logistic", "additive"), ("linear", "multiplicative"),
                ("linear", "additive")]
_measured = {"q": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviation():
    yield
    print(f"\n[window quantiles] max |plane - restatement| / (y_scale * n_points) = {_measured['q']:.3e}")


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _dev_fits(fb):
    return batched.FittedBatch(*(_cuda(getattr(fb, k)) for k in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")),
                               fb.smax, fb.kmax)


# the window rules: (kind, rule arguments), the anchored rule's origins / frame lengths made per batch by _rule_args
RULES = {"fixed": ("fixed", DAY, 5 * H_NS), "anchored": ("anchored", DAY), "period": ("period", 1, 0)}


def _rule_args(rule, fut, flen=None):
    """The C arguments between yhat_int and wmax, the device arrays they point at, and per model the (origin, frame
    length) its windows are taken from."""
    n, h = fut.shape
    if rule[0] == "fixed":
        return (rule[1], rule[2]), (), [(rule[2], h)] * n
    if rule[0] == "period":
        return (rule[1], rule[2]), (), [(None, h)] * n
    origins = fut[:, 0] - np.arange(n, dtype=np.int64) * 3 * H_NS - 1       # a different origin per model
    flen = np.full(n, h, np.int32) if flen is None else np.asarray(flen, np.int32)
    o, f = _cuda(origins), _cuda(flen)
    return (rule[1], o.data_ptr(), f.data_ptr()), (o, f), list(zip(origins.tolist(), flen.tolist()))


def _raw(ctx, opts, fb, fut, floor, cap, rule, wmax, pct, seed, bounds=True, flen=None, planes=True):
    """The device entry point of ``rule`` at raw percentiles ``pct`` (None: the sums twin without levels).  Returns
    (rc, outputs as numpy, per-model (origin, frame length))."""
    import torch
    n, h = fut.shape
    fd, futd, fld, capd = _dev_fits(fb), _cuda(fut), _cuda(floor), _cuda(cap)
    f64 = lambda *s: torch.empty(s, dtype=torch.float64, device="cuda")     # noqa: E731
    out = {"yhat": f64(n, h), "lo": f64(n, h), "hi": f64(n, h), "yint": torch.empty((n, h), dtype=torch.int32, device="cuda"),
           "n_windows": torch.zeros(n, dtype=torch.int32, device="cuda"),
           "start": torch.empty((n, wmax), dtype=torch.int64, device="cuda"),
           "points": torch.empty((n, wmax), dtype=torch.int32, device="cuda"), "yhat_sum": f64(n, wmax),
           "quantity_sum": torch.empty((n, wmax), dtype=torch.int64, device="cuda"), "lower": f64(n, wmax),
           "upper": f64(n, wmax)}
    rargs, keep, anchors = _rule_args(rule, fut, flen)
    name = {"fixed": "pb200_predict_sums", "period": "pb200_predict_period_sums",
            "anchored": "pb200_predict_sums_anchored"}[rule[0]]
    p = lambda t: t.data_ptr()                                               # noqa: E731
    args = [ctx.handle, C.byref(opts), *(p(getattr(fd, k)) for k in ("params", "tchange", "meta_i32", "meta_i64",
                                                                     "meta_f64")),
            n, p(futd), h, p(fld), p(capd), seed, p(out["yhat"]), p(out["lo"]) if bounds else None,
            p(out["hi"]) if bounds else None, p(out["yint"]), *rargs, wmax,
            *(p(out[k]) for k in ("n_windows", "start", "points", "yhat_sum", "quantity_sum", "lower", "upper"))]
    if pct is not None:
        pct = np.ascontiguousarray(pct, dtype=np.float64)
        out["planes"] = f64(pct.size, n, wmax)
        name += "_quantiles"
        args += [pct.size, pct.ctypes.data, p(out["planes"]) if planes else None]
    torch.cuda.synchronize()
    rc = getattr(L.load(), name + "_device")(*args)
    ctx.synchronize()
    del keep                                   # the anchored rule's device arrays lived until here
    res = {k: v.cpu().numpy() for k, v in out.items()}
    if not bounds:
        res["lo"] = res["hi"] = None
    return rc, res, anchors


def _runs(fut_i, rule, anchor):
    """(first index of each window run, frame length walked) of one model's frame under ``rule``."""
    origin, flen = anchor
    fr = fut_i[:flen]
    if rule[0] == "period":
        from period_oracle import period_runs
        first, _ = period_runs(fr, "M")
    else:
        first, _ = wo.window_runs(fr, rule[1], origin)
    return first, fr


def _check_reference(res, fb, fut, floor, cap, growth, mode, n, pct, seed, rule, anchors, wmax):
    """Every written plane against the restatement; NaN past n_windows and for failed models."""
    for i in range(fb.n):
        pl = res["planes"][:, i]
        if fb.meta_i32[i, 4] < 0:
            assert res["n_windows"][i] == 0 and np.all(np.isnan(pl))
            continue
        first, fr = _runs(fut[i], rule, anchors[i])
        nw = first.size - 1
        assert res["n_windows"][i] == nw
        assert np.all(np.isnan(pl[:, min(nw, wmax):]))
        d = mcs.draws(fb, i, fut[i], floor[i], cap[i], growth == "logistic", mode == "multiplicative", n, seed)[:fr.size]
        ref = qo.quantiles(wqo.run_sums(d, first), pct)[:, :wmax]
        k = ref.shape[1]
        pts = np.diff(first)[:k]
        err = np.max(np.abs(pl[:, :k] - ref) / pts) / fb.meta_f64[i, 0]
        assert err <= SUM_TOL, (i, err)
        _measured["q"] = max(_measured["q"], err)


def _daily_models(growth, mode, masks, H, seed=0, status=None):
    """Models whose frames cross several days and months: hourly (6, 4), daily (3, 2) and 12-hourly (7) cadences."""
    rng = np.random.RandomState(seed)
    frs, fut = [], []
    for i, mask in enumerate(masks):
        p, _ = _prep(mask, growth, mode)
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=(i % 7 == 5)))
    opts = batched.make_options(growth=growth, seasonality_mode=mode)
    fb = _batch(frs, opts, status)
    floor = np.zeros(len(frs)) if growth == "linear" else rng.uniform(-5, 5, len(frs))
    cap = np.array([fr.prep.cap_value for fr in frs]) + floor
    return fb, np.stack(fut), floor, cap


def _wmax(fut, rule, anchors):
    return max(_runs(fut[i], rule, anchors[i])[0].size - 1 for i in range(fut.shape[0]))


# ---------------------------------------------------------------------------------------------------------------------
# identities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("growth,mode", GROWTH_MODES)
def test_identities_with_the_sums_call(gpu_ctx, growth, mode, rule):
    r = RULES[rule]
    fb, fut, floor, cap = _daily_models(growth, mode, [6, 2, 7, 3, 4, 3], 100, seed=1)
    flen = [100, 37, 1, 100, 64, 90]
    for n, w in ((1000, 0.8), (3, 0.95), (1024, 0.5)):
        opts = batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=n, interval_width=w)
        anchors = _rule_args(r, fut, flen)[2]
        wmax = _wmax(fut, r, anchors) + 2
        lo_p, hi_p = mcs.percentiles(w)
        pct = [hi_p, 50.0, lo_p, 0.0, 100.0, lo_p]
        for bounds in (True, False):
            rc0, plain, _ = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, wmax, None, 7, bounds, flen)
            rc1, got, _ = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, wmax, pct, 7, bounds, flen)
            assert rc0 == 0 and rc1 == 0, L.last_error()
            for k, v in plain.items():
                assert (v is None and got[k] is None) or v.tobytes() == got[k].tobytes(), (k, n, w, bounds)
            assert got["planes"][2].tobytes() == plain["lower"].tobytes() == got["planes"][5].tobytes()
            assert got["planes"][0].tobytes() == plain["upper"].tobytes()
            for i in range(fb.n):
                nw = got["n_windows"][i]
                assert np.all(np.isnan(got["planes"][:, i, nw:]))
                assert np.all(got["planes"][3, i, :nw] <= got["planes"][1, i, :nw])
                assert np.all(got["planes"][1, i, :nw] <= got["planes"][4, i, :nw])


def _one_point_frames(rule, growth, mode):
    """Frames whose windows hold one point each: the grid step as the width, or month starts under months."""
    rng = np.random.RandomState(6)
    frs, fut = [], []
    for k in range(5):
        mask = 6 if rule != "period" else 3
        p, _ = _prep(mask, growth, mode)
        frs.append(_model(p, rng))
        if rule == "period":
            last = pd.Timestamp(int(p.ds_sorted[-1]))
            ms = pd.date_range(last + pd.Timedelta(days=1 + 40 * k), periods=30, freq="MS")
            fut.append(ms.values.astype("datetime64[ns]").astype(np.int64))
        else:
            fut.append(_future(p, 300) + k * 3 * H_NS)
    opts = batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=1000)
    fb = _batch(frs, opts)
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    return fb, fut, np.zeros(5), cap, opts


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("growth,mode", GROWTH_MODES)
def test_one_point_windows_are_the_pointwise_planes(gpu_ctx, growth, mode, rule):
    fb, fut, floor, cap, opts = _one_point_frames(rule, growth, mode)
    r = {"fixed": ("fixed", H_NS, 0), "anchored": ("anchored", H_NS), "period": ("period", 1, 0)}[rule]
    pct = [2.5, 97.5, 50.0, 0.0, 100.0, 10.0, 90.0, 33.3]
    h = fut.shape[1]
    rc, got, _ = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, h, pct, 9)
    assert rc == 0 and np.all(got["n_windows"] == h) and np.all(got["points"] == 1)
    _, _, _, _, planes = _quant_host(gpu_ctx, opts, fb, fut, floor, cap, pct, 9)
    assert got["planes"].tobytes() == planes.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# against the restatement
# ---------------------------------------------------------------------------------------------------------------------
LEVEL_SETS = {
    "Q1": [50.0],
    "Q9": [100.0 * q for q in DECILES],
    "Q32": list(np.random.RandomState(9).permutation(np.linspace(0, 100, 32))),
    "unsorted": [90.0, 10.0, 50.0, 50.0, 0.0, 100.0, 10.0, 97.5, 2.5],
}


@pytest.mark.parametrize("rule", list(RULES))
@pytest.mark.parametrize("levels", list(LEVEL_SETS))
def test_planes_match_restatement(gpu_ctx, levels, rule):
    r = RULES[rule]
    status = np.array([0, 0, L.ST_TOO_FEW, 0, 0, 0])
    fb, fut, floor, cap = _daily_models("logistic", "multiplicative", [6, 2, 7, 3, 4, 6], 80, seed=2, status=status)
    opts = batched.make_options(uncertainty_samples=1000)
    anchors = _rule_args(r, fut)[2]
    wmax = _wmax(fut, r, anchors)
    pct = LEVEL_SETS[levels]
    rc, got, anchors = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, wmax, pct, 3)
    assert rc == 0
    _check_reference(got, fb, fut, floor, cap, "logistic", "multiplicative", 1000, pct, 3, r, anchors, wmax)


@pytest.mark.parametrize("growth,mode", [("logistic", "additive"), ("linear", "multiplicative")])
@pytest.mark.parametrize("n", [2, 3, 1000, 1024])
def test_planes_match_restatement_sample_counts(gpu_ctx, growth, mode, n):
    fb, fut, floor, cap = _daily_models(growth, mode, [6, 2, 0], 60, seed=11)
    opts = batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=n)
    pct = [0.0, 5.0, 50.0, 95.0, 100.0, 30.0]
    for rule in ("fixed", "period"):
        r = RULES[rule]
        anchors = _rule_args(r, fut)[2]
        wmax = _wmax(fut, r, anchors)
        rc, got, anchors = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, wmax, pct, 4)
        assert rc == 0
        _check_reference(got, fb, fut, floor, cap, growth, mode, n, pct, 4, r, anchors, wmax)


def test_planes_match_restatement_on_crowded_rows(gpu_ctx):
    """sigma_obs = 0 just past the history: most draws of a two-point window's total are equal, so the target ranks'
    histogram bin is crowded and the selection sorts the row."""
    fb, fut, floor, cap = _crowded()
    opts = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=1000)
    r = ("fixed", 40 * 10**9, 0)
    pct = [5.0 * k for k in range(21)] + [33.3]
    anchors = _rule_args(r, fut)[2]
    wmax = _wmax(fut, r, anchors)
    rc, got, anchors = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, wmax, pct, 5)
    assert rc == 0
    _check_reference(got, fb, fut, floor, cap, "linear", "additive", 1000, pct, 5, r, anchors, wmax)
    first, _ = _runs(fut[0], r, anchors[0])
    sums = wqo.run_sums(mcs.draws(fb, 0, fut[0], 0.0, 1.0, False, False, 1000, 5), first)
    assert np.sum(mcs.crowded_bin(sums, 0.8) > 64) >= 8                      # the premise: the sort path runs


@pytest.mark.parametrize("rule", ["fixed", "anchored"])
def test_more_windows_than_slots(gpu_ctx, rule):
    """wmax below the windows' count: the true count is reported and the first wmax windows are written."""
    fb, fut, floor, cap = _daily_models("linear", "additive", [6, 4], 240, seed=12)
    opts = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=500)
    r = ("fixed", 6 * H_NS, 0) if rule == "fixed" else ("anchored", 6 * H_NS)
    pct = [10.0, 50.0, 90.0]
    rc, got, anchors = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, 5, pct, 6)
    assert rc == 0 and np.all(got["n_windows"] >= 40)
    _check_reference(got, fb, fut, floor, cap, "linear", "additive", 500, pct, 6, r, anchors, 5)


def test_batch_larger_than_the_sm_count(gpu_ctx, sms):
    N = sms + 20
    masks = [ALL_MASKS[i % len(ALL_MASKS)] for i in range(N)]
    status = np.where(np.arange(N) % 11 == 7, L.ST_TOO_FEW, 0)
    fb, fut, floor, cap = _daily_models("logistic", "multiplicative", masks, 30, seed=10, status=status)
    opts = batched.make_options(uncertainty_samples=1000)
    r = RULES["fixed"]
    pct = [100.0 * q for q in DECILES]
    anchors = _rule_args(r, fut)[2]
    wmax = _wmax(fut, r, anchors)
    rc, got, anchors = _raw(gpu_ctx, opts, fb, fut, floor, cap, r, wmax, pct, 3)
    assert rc == 0
    _check_reference(got, fb, fut, floor, cap, "logistic", "multiplicative", 1000, pct, 3, r, anchors, wmax)


# ---------------------------------------------------------------------------------------------------------------------
# failed models, batch position, host / device, refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_planes_independent_of_the_batch(gpu_ctx):
    fb, fut, floor, cap = _daily_models("logistic", "multiplicative", [6, 2, 0, 7, 6, 3], 72, seed=12)
    fb.meta_i32[4, 4] = L.ST_TOO_FEW
    opts = batched.make_options()
    for call, rule in ((batched.predict_sums_host, (DAY, 0)), (batched.predict_period_sums_host, (1, 0))):
        full, ws = call(gpu_ctx, opts, fb, fut, floor, cap, *rule, seed=2, levels=DECILES)
        assert isinstance(ws, batched.WindowQuantiles) and ws.quantiles.shape == (9, 6, ws.start.shape[1])
        assert np.all(np.isnan(ws.quantiles[:, 4])) and ws.n_windows[4] == 0
        perm = np.array([3, 0, 5, 1, 4, 2])
        _, wp = call(gpu_ctx, opts, _take(fb, perm), fut[perm], floor[perm], cap[perm], *rule, seed=2, levels=DECILES)
        k = min(wp.start.shape[1], ws.start.shape[1])
        assert wp.quantiles[:, :, :k].tobytes() == np.ascontiguousarray(ws.quantiles[:, perm, :k]).tobytes()
        for i in range(6):
            _, w1 = call(gpu_ctx, opts, _take(fb, [i]), fut[i:i + 1], floor[i:i + 1], cap[i:i + 1], *rule, seed=2,
                         levels=DECILES)
            nw = int(ws.n_windows[i])
            assert w1.quantiles[:, 0, :nw].tobytes() == np.ascontiguousarray(ws.quantiles[:, i, :nw]).tobytes()


def test_device_calls_match_host_calls(gpu_ctx):
    fb, fut, floor, cap = _daily_models("linear", "additive", [6, 0, 2], 50, seed=13)
    opts = batched.make_options(growth="linear", seasonality_mode="additive")
    fd = _dev_fits(fb)
    for host, dev, rule in ((batched.predict_sums_host, batched.predict_sums_device, (DAY, 0)),
                            (batched.predict_period_sums_host, batched.predict_period_sums_device, (3, 2))):
        fh, wh = host(gpu_ctx, opts, fb, fut, floor, cap, *rule, seed=1, intervals=True, levels=[0.9, 0.1, 0.5])
        fdv, wd = dev(gpu_ctx, opts, fd, _cuda(fut), _cuda(floor), _cuda(cap), *rule, seed=1, intervals=True,
                      levels=[0.9, 0.1, 0.5])
        assert list(wh.levels) == [0.9, 0.1, 0.5]
        for f in batched.fields(batched.WindowQuantiles):
            if f.name != "levels":
                assert getattr(wd, f.name).cpu().numpy().tobytes() == getattr(wh, f.name).tobytes(), f.name
        for k in ("yhat", "yhat_lower", "yhat_upper", "yhat_int"):
            assert getattr(fdv, k).cpu().numpy().tobytes() == getattr(fh, k).tobytes(), k
        _, plain = host(gpu_ctx, opts, fb, fut, floor, cap, *rule, seed=1, intervals=True)
        assert type(plain) is batched.WindowSums
        for f in batched.fields(batched.WindowSums):
            assert getattr(plain, f.name).tobytes() == getattr(wh, f.name).tobytes(), f.name


def test_refusals_launch_nothing(gpu_ctx):
    fb, fut, floor, cap = _daily_models("logistic", "multiplicative", [6, 2], 24, seed=14)
    good = batched.make_options()
    reg = batched.make_regressor_options(regressors=[{"name": "promo"}])
    lc = gpu_ctx.launch_count
    cases = [(good, [], E_ARG), (good, [50.0] * 33, E_ARG), (good, [float("nan")], E_ARG), (good, [-1e-9], E_ARG),
             (good, [100.0000001], E_ARG), (batched.make_options(uncertainty_samples=1), [50.0], E_UNSUPPORTED),
             (batched.make_options(uncertainty_samples=1025), [50.0], E_UNSUPPORTED),
             (batched.make_options(interval_width=1.5), [50.0], E_ARG), (reg, [50.0], E_UNSUPPORTED)]
    for rule in RULES.values():
        for opts, pct, code in cases:
            rc, _, _ = _raw(gpu_ctx, opts, fb, fut, floor, cap, rule, 4, pct, 0)
            assert rc == code, (rule, pct, rc, L.last_error())
        rc, _, _ = _raw(gpu_ctx, good, fb, fut, floor, cap, rule, 4, [50.0], 0, planes=False)
        assert rc == E_ARG, L.last_error()
    # a null percentile pointer, on the host entry points too
    n, h = fb.n, fut.shape[1]
    p = lambda a: a.ctypes.data                                               # noqa: E731
    outs = [np.empty((n, h)), np.empty((n, h)), np.empty((n, h)), np.empty((n, h), np.int32)]
    wouts = [np.zeros(n, np.int32), np.empty((n, 4), np.int64), np.empty((n, 4), np.int32), np.empty((n, 4)),
             np.empty((n, 4), np.int64), np.empty((n, 4)), np.empty((n, 4))]
    base = [gpu_ctx.handle, C.byref(good), *(p(np.ascontiguousarray(getattr(fb, k))) for k in
                                             ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")),
            n, p(np.ascontiguousarray(fut)), h, p(floor), p(cap), 0, *map(p, outs)]
    planes = np.empty((1, n, 4))
    lib = L.load()
    assert lib.pb200_predict_sums_quantiles_host(*base, DAY, 0, 4, *map(p, wouts), 1, None, p(planes)) == E_ARG
    assert lib.pb200_predict_period_sums_quantiles_host(*base, 1, 0, 4, *map(p, wouts), 1, None, p(planes)) == E_ARG
    assert lib.pb200_predict_period_sums_quantiles_host(*base, 2, 0, 4, *map(p, wouts), 1, p(np.array([50.0])),
                                                        p(planes)) == E_ARG
    assert gpu_ctx.launch_count == lc
    with pytest.raises(ValueError):
        batched.predict_sums_host(gpu_ctx, good, fb, fut, floor, cap, DAY, levels=[1.5])
    assert gpu_ctx.launch_count == lc
    batched.predict_sums_host(gpu_ctx, good, fb, fut, floor, cap, DAY, levels=[0.5])
    assert gpu_ctx.launch_count == lc + 2                   # predict_kernel and mc_sum_kernel


# ---------------------------------------------------------------------------------------------------------------------
# backtest: cross_validation_device(aggregate_ns=W, window_quantiles=...) and the job
# ---------------------------------------------------------------------------------------------------------------------
FLOOR, CAPM = 0.0, 1.1
HORIZON, PERIOD, INITIAL = DAY, DAY // 2, 3 * DAY
KEEP = [0, 1, 2, 3, 4, 8, 9, 10, 11]
LEVELS = [0.1, 0.5, 0.9, 0.025, 0.975]
W = 6 * H_NS


@pytest.fixture(scope="module", params=[np.float32, np.float64])
def cv_batch(request):
    ds, y, off = _mixed_batch()
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in KEEP]
    o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]).astype(request.param), o2


def _cv(ctx, ds, y, off, window_quantiles=None, keep_fits=False, budget=None):
    opts = batched.make_options(uncertainty_samples=200)
    cap = _cuda(np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])]))
    return batched.cross_validation_device(ctx, opts, _cuda(ds), _cuda(y), off, FLOOR, cap, HORIZON, PERIOD, INITIAL,
                                           intervals=True, seed=3, rolling_window=0.1, aggregate_ns=W,
                                           window_quantiles=window_quantiles, keep_fits=keep_fits, _row_budget=budget)


def _windows_bytes(w):
    out = {k: getattr(w, k).tobytes() for k in ("series", "cutoff", "horizon", "points", "y", "yhat", "yhat_lower",
                                                 "yhat_upper")}
    out.update({"m_" + k: v.tobytes() for k, v in w.metrics.items()})
    return out


def test_backtest_window_quantiles(gpu_ctx, cv_batch):
    import torch
    ds, y, off = cv_batch
    plain = _cv(gpu_ctx, ds, y, off)
    res = _cv(gpu_ctx, ds, y, off, LEVELS, keep_fits=True)
    assert plain.windows.yhat_q is None and plain.windows.quantile_metrics is None
    assert _cv_bytes(res) == _cv_bytes(plain) and _windows_bytes(res.windows) == _windows_bytes(plain.windows)
    w = res.windows
    assert w.yhat_q.shape == (len(LEVELS), w.series.size)
    # chunks do not change a row
    small = _cv(gpu_ctx, ds, y, off, LEVELS, budget=1)
    assert small.windows.yhat_q.tobytes() == w.yhat_q.tobytes()
    for k, v in w.quantile_metrics.items():
        assert small.windows.quantile_metrics[k].tobytes() == v.tobytes(), k
    # yhat_q is the anchored call's planes over each pair's held-out frame
    fut_h, wl, cut = _frames(ds, off, res)
    capv = np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])])
    P = fut_h.shape[0]
    opts = batched.make_options(uncertainty_samples=200)
    _, ws = batched.predict_sums_anchored_device(gpu_ctx, opts, _dev_fits(res.fitted), _cuda(fut_h),
                                                 torch.full((P,), FLOOR, dtype=torch.float64, device="cuda"),
                                                 _cuda(capv[res.pair_series]), W, _cuda(cut + 1),
                                                 _cuda(wl.astype(np.int32)), seed=3, intervals=True, levels=LEVELS)
    q = ws.quantiles.cpu().numpy()
    seen = 0
    for p in range(P):
        g = (w.series == res.pair_series[p]) & (w.cutoff == res.pair_cutoff[p])
        k = int(g.sum())
        seen += k
        assert np.ascontiguousarray(w.yhat_q[:, g]).tobytes() == np.ascontiguousarray(q[:, p, :k]).tobytes(), p
    assert seen == w.series.size
    # a few pairs against the restatement
    rng = np.random.RandomState(0)
    for p in rng.choice(np.flatnonzero(res.pair_status >= 0), 6, replace=False):
        s, c = int(res.pair_series[p]), int(res.pair_cutoff[p])
        rows = (res.row_series == s) & (res.cutoff == c)
        fr = res.ds[rows]
        d = mcs.draws(res.fitted, int(p), fr, FLOOR, capv[s], True, True, 200, 3)
        ref = wqo.window_quantiles(d, fr, W, c + 1, 100.0 * np.asarray(LEVELS))
        g = (w.series == s) & (w.cutoff == c)
        first, _ = wo.window_runs(fr, W, c + 1)
        err = np.max(np.abs(w.yhat_q[:, g] - ref) / np.diff(first)) / float(res.fitted.meta_f64[p, 0])
        assert err <= SUM_TOL, (p, err)
        _measured["q"] = max(_measured["q"], err)
    # the calibration by horizon (j + 1) W over the window rows
    _check_quantile_metrics(w.quantile_metrics, w.series, w.horizon, w.y, w.yhat_q, LEVELS, off.size - 1, 0.1)


def _bt_config(tmp_path, inp, **bt):
    return {"io": {"input": inp, "metrics": str(tmp_path / "metrics"), "cv_rows": str(tmp_path / "rows"),
                   "window_metrics": str(tmp_path / "wm"), "window_rows": str(tmp_path / "wr"),
                   "window_quantile_metrics": str(tmp_path / "wq")},
            "model": {"floor": 0, "cap_multiplier": 1.1},
            "backtest": {"horizon": "30 days", "period": "15 days", "initial": "180 days", "aggregate": "10 days",
                         "intervals": True, "uncertainty_samples": 100, **bt}}


def test_backtest_job_on_golden_fixture(tmp_path, model_input_dir):
    import shutil
    from time_series_spark_b200.jobs.prophet_backtest import QUANTILE_METRICS_SCHEMA, ProphetBacktester
    ProphetBacktester.run(None, _bt_config(tmp_path, model_input_dir))
    base = {k: pq.read_table(str(tmp_path / k)) for k in ("metrics", "rows", "wm", "wr")}
    assert not (tmp_path / "wq").exists()
    for k in base:
        shutil.rmtree(str(tmp_path / k))
    levels = [0.9, 0.1, 0.5]
    ProphetBacktester.run(None, _bt_config(tmp_path, model_input_dir, aggregate_quantiles=levels))
    for k in ("metrics", "rows", "wm"):
        assert pq.read_table(str(tmp_path / k)).equals(base[k]), k
    wr = pq.read_table(str(tmp_path / "wr"))
    assert wr.column_names == base["wr"].column_names + ["yhat_q0.9", "yhat_q0.1", "yhat_q0.5"]
    assert wr.select(base["wr"].column_names).equals(base["wr"])
    wq = pq.read_table(str(tmp_path / "wq"))
    assert wq.schema.equals(QUANTILE_METRICS_SCHEMA) and wq.num_rows > 0
    assert set(wq["horizon"].cast(pa.int64()).to_pylist()) <= {10 * DAY, 20 * DAY, 30 * DAY}
    assert set(wq["quantile"].to_pylist()) == set(levels)
    sb = wq["share_below"].to_numpy()
    assert np.all((sb >= 0) & (sb <= 1)) and np.all(wq["pinball_loss"].to_numpy() >= 0)
    lo, hi = wr["yhat_q0.1"].to_numpy(), wr["yhat_q0.9"].to_numpy()
    assert np.all(lo <= wr["yhat_q0.5"].to_numpy()) and np.all(wr["yhat_q0.5"].to_numpy() <= hi)


def test_backtest_job_empty_shard(tmp_path):
    from time_series_spark_b200.jobs import prophet_backtest as pb
    tbl = pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32()),
                    "ds": pa.array([], pa.timestamp("ns")), "y": pa.array([], pa.int32())})
    cfg = {"io": {"metrics": str(tmp_path / "m"), "window_metrics": str(tmp_path / "wm"), "window_rows": str(tmp_path / "wr"),
                  "window_quantile_metrics": str(tmp_path / "wq")},
           "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": {"horizon": "1 days", "aggregate": "8h", "intervals": True, "aggregate_quantiles": [0.5, 0.05]}}
    job = pb.ProphetBacktester(cfg)
    metrics, _ = job.backtest(tbl)
    _, wr = job.window_outputs
    assert wr.num_rows == 0 and wr.column_names[-2:] == ["yhat_q0.5", "yhat_q0.05"]
    assert job.window_quantile_metrics.num_rows == 0
    assert job.window_quantile_metrics.schema.equals(pb.QUANTILE_METRICS_SCHEMA)
    job.persist(metrics, None)
    assert pq.read_table(str(tmp_path / "wq")).schema.names == pb.QUANTILE_METRICS_SCHEMA.names


# ---------------------------------------------------------------------------------------------------------------------
# the scorer job on the golden fixture, one and two ranks
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fc", [dict(aggregate="1D"), dict(aggregate_period="M")])
def test_scorer_aggregate_quantiles(tmp_path, model_input_dir, gpu_ctx, monkeypatch, fc):
    import pyarrow.dataset as pads
    from time_series_spark_b200 import model_record
    from time_series_spark_b200.jobs import prophet_scorer as ps
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    models = str(tmp_path / "models")
    ProphetModeler.model(None, {"io": {"input": model_input_dir, "models": models}, "model": {"floor": 0, "cap_multiplier": 1.1}})
    mt = pads.dataset(models, format="parquet").to_table()
    levels = [0.95, 0.5, 0.05]
    fcast = {"periods": 3000, "frequency": "15min", "uncertainty_samples": 500, "seed": 3, **fc}
    keys = ["series_id", "dim_id"]
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    op0 = ps.forecast_time_series({"io": {"aggregates": "a"}, "forecast": dict(fcast)})
    f0 = op0.apply_batched(mt, keys)
    op = ps.forecast_time_series({"io": {"aggregates": "a"}, "forecast": dict(fcast, aggregate_quantiles=levels)})
    f1 = op.apply_batched(mt, keys)
    assert f1.equals(f0)
    cols = ["yhat_q0.95", "yhat_q0.5", "yhat_q0.05"]
    agg = op.aggregates
    assert agg.schema.equals(ps.aggregate_schema(levels)) and agg.select(op0.aggregates.column_names).equals(op0.aggregates)
    assert agg.num_rows >= 2 * mt.num_rows
    # the columns are batched's planes over the decoded models
    fitted, last_ds, info = model_record.decode(mt["model"])
    opts = batched.make_options(growth="logistic" if info["logistic"] else "linear",
                                seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
                                n_changepoints=info["n_changepoints"], uncertainty_samples=500)
    opts.yearly, opts.weekly, opts.daily = info["yearly"], info["weekly"], info["daily"]
    floor = np.asarray(mt["floor"].to_pylist(), np.float32).astype(np.float64)
    cap = np.asarray(mt["cap"].to_pylist(), np.float32).astype(np.float64)
    fut = ps.frequency_to_future(last_ds, 3000, "15min")
    if "aggregate" in fc:
        _, ws = batched.predict_sums_host(gpu_ctx, opts, fitted, fut, floor, cap, DAY, 0, seed=3, levels=levels)
    else:
        _, ws = batched.predict_period_sums_host(gpu_ctx, opts, fitted, fut, floor, cap, 1, 0, seed=3, levels=levels)
    keep = np.arange(ws.start.shape[1])[None, :] < ws.n_windows[:, None]
    for j, c in enumerate(cols):
        assert np.array_equal(ws.quantiles[j][keep], agg[c].to_numpy()), c
    assert np.all(agg["yhat_q0.05"].to_numpy() <= agg["yhat_q0.95"].to_numpy())
    # rank 1 of 2 writes the rows of its models
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "1")
    op.apply_batched(mt, keys)
    part = op.aggregates.to_pandas()
    full = agg.to_pandas()
    assert 0 < len(part) < len(full)
    ref = full[full["series_id"].isin(part["series_id"].unique()) & full["dim_id"].isin(part["dim_id"].unique())]
    assert ref.reset_index(drop=True).equals(part.reset_index(drop=True))
