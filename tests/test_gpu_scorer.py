"""The scorer's kernels held to exact references (run with -m gpu on an H100).

* mc_kernel against oracle/mc_stream.py, the numpy restatement of its own stream and sampler: every bound within
  1e-9 * y_scale (what is left is last-bit differences of libm functions and FMA contraction);
* a model's intervals are a function of the model and the seed, not of its place in the batch or the shard;
* predict_kernel against prophet_oracle.predict given identical parameters, within 1e-12 * y_scale, at every segment of
  the trend, far from 1970, past the 64 x 1024-point tile cap, with mixed seasonality masks in one batch;
* the int epilogue exactly: yhat_int == clamp(trunc(yhat), floor), saturated to int32, on the kernel's own yhat.

Models are built by hand as fitted-record arrays on the history of a prophet_oracle.Prepared, so that sigma_obs, the
slope changes and the masks can be chosen.
"""
import functools

import numpy as np
import pyarrow as pa
import pytest

from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, model_record
from time_series_spark_b200.jobs.prophet_scorer import forecast_time_series

pytestmark = pytest.mark.gpu

H_NS = 3600 * 10**9
DAY = 24 * H_NS
MIN15 = 15 * 60 * 10**9
INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
MC_TOL = 1e-9        # |kernel - restatement| / y_scale
PRED_TOL = 1e-12     # |kernel - oracle| / (y_scale * max(1, |yhat| / y_scale))
_measured = {"mc": 0.0, "predict": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviations():
    yield
    print(f"\n[scorer] max |mc_kernel - restatement| / y_scale = {_measured['mc']:.3e}; "
          f"max |predict_kernel - oracle| under the stated rule = {_measured['predict']:.3e}")


# history shapes whose seasonalities give each mask: (step, points, weekly_seasonality switch)
_MASK_HIST = {7: (12 * H_NS, 1600, "auto"),   # 800 days at 12 h: yearly + weekly + daily
              6: (H_NS, 720, "auto"),         # 30 days hourly: weekly + daily
              5: (12 * H_NS, 1600, False),    # 800 days at 12 h without weekly: yearly + daily
              4: (H_NS, 240, "auto"),         # 10 days hourly: daily
              3: (DAY, 801, "auto"),          # 800 days daily: yearly + weekly
              2: (DAY, 60, "auto"),           # 60 days daily: weekly
              1: (7 * DAY, 115, "auto"),      # 798 days weekly: yearly
              0: (MIN15, 96, "auto")}         # one day: none
ALL_MASKS = (7, 6, 5, 4, 3, 2, 1, 0)


@functools.lru_cache(maxsize=None)
def _prep(mask, growth, mode, ncp=25, start="2021-03-01", cpr=0.8):
    step, T, weekly = _MASK_HIST[mask]
    ds = np.datetime64(start, "ns").astype(np.int64) + step * np.arange(T, dtype=np.int64)
    y = 100.0 + 20.0 * np.sin(np.arange(T) / 7.0) + np.arange(T) % 5
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, n_changepoints=ncp, changepoint_range=cpr,
                              weekly_seasonality=weekly)
    p = po.prepare(ds, y, 0.0, 1.1 * y.max(), oopts)
    assert sum(mcs._MASK_BIT[s.name] for s in p.seasonalities) == mask
    return p, oopts


def _model(p, rng, sigma=0.03, delta_scale=0.3):
    logistic = p.logistic
    delta = delta_scale * rng.laplace(size=p.S) if p.n_changepoints_real else np.zeros(p.S)
    beta = 0.05 * rng.randn(p.K) if p.seasonalities else np.zeros(p.K)
    k, m = (rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)) if logistic else (rng.uniform(-0.5, 0.5), rng.uniform(0.3, 0.7))
    return po.FitResult(prep=p, k=k, m=m, delta=delta, sigma_obs=sigma, beta=beta, theta=None, neg_logp=0.0, iters=0,
                        n_evals=0, ret=0)


def _batch(frs, opts, status=None):
    lay = L.get_layout(opts)
    recs = [mcs.record(fr.prep, fr.k, fr.m, fr.sigma_obs, fr.delta, fr.beta, lay.smax, lay.kmax) for fr in frs]
    ns = mcs.stack(recs, lay.smax, lay.kmax)
    if status is not None:
        ns.meta_i32[:, 4] = status
    return batched.FittedBatch(ns.params, ns.tchange, ns.meta_i32, ns.meta_i64, ns.meta_f64, lay.smax, lay.kmax)


def _take(fb, idx):
    return batched.FittedBatch(*(np.ascontiguousarray(a[idx]) for a in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64,
                                                                         fb.meta_f64)), fb.smax, fb.kmax)


def _future(p, H, in_history=False):
    """H timestamps after the history at its own cadence, or its last H timestamps (t <= 1)."""
    step = int(p.ds_sorted[1] - p.ds_sorted[0])
    if in_history:
        assert H <= p.T
        return np.ascontiguousarray(p.ds_sorted[-H:])
    return int(p.ds_sorted[-1]) + step * np.arange(1, H + 1, dtype=np.int64)


def _check_mc(gpu_ctx, fb, fut, floor, cap, growth, mode, n, width, seed, ncp=25):
    """Run the kernel, restate every model, compare the bounds; returns the kernel's result and the restated draws."""
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp, interval_width=width,
                                uncertainty_samples=n)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, floor, cap, seed=seed, intervals=True)
    worst = 0.0
    out = []
    for i in range(fb.n):
        if fb.meta_i32[i, 4] < 0:
            assert np.all(np.isnan(fc.yhat_lower[i])) and np.all(np.isnan(fc.yhat_upper[i]))
            out.append(None)
            continue
        d = mcs.draws(fb, i, fut[i], floor[i], cap[i], growth == "logistic", mode == "multiplicative", n, seed)
        lo, hi = mcs.bounds(d, width)
        ys = fb.meta_f64[i, 0]
        err = max(np.max(np.abs(fc.yhat_lower[i] - lo)), np.max(np.abs(fc.yhat_upper[i] - hi))) / ys
        assert err <= MC_TOL, (i, n, width, seed, err)
        worst = max(worst, err)
        out.append(d)
    _measured["mc"] = max(_measured["mc"], worst)
    return fc, out


# ---------------------------------------------------------------------------------------------------------------
# interval_width / uncertainty_samples are refused before anything is launched
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width", [-0.1, 1.5, 95.0, float("nan")])
def test_out_of_range_interval_width_is_refused(gpu_ctx, width):
    p, _ = _prep(0, "linear", "additive")
    fb = _batch([_model(p, np.random.RandomState(0))], batched.make_options(growth="linear", seasonality_mode="additive"))
    fut = _future(p, 16)[None, :]
    opts = batched.make_options(growth="linear", seasonality_mode="additive", interval_width=width)
    with pytest.raises(L.Pb200Error, match="interval_width"):
        batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(1), np.ones(1), intervals=True)
    # no interval asked for: the width is not used, the forecast goes through
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(1), np.ones(1), intervals=False)
    assert np.all(np.isfinite(fc.yhat))


@pytest.mark.parametrize("n", [1, 1025])
def test_unsupported_sample_count_is_refused(gpu_ctx, n):
    p, _ = _prep(0, "linear", "additive")
    fb = _batch([_model(p, np.random.RandomState(0))], batched.make_options(growth="linear", seasonality_mode="additive"))
    opts = batched.make_options(growth="linear", seasonality_mode="additive", uncertainty_samples=n)
    with pytest.raises(L.Pb200Error, match="uncertainty_samples"):
        batched.predict_batch_host(gpu_ctx, opts, fb, _future(p, 16)[None, :], np.zeros(1), np.ones(1), intervals=True)


# ---------------------------------------------------------------------------------------------------------------
# mc_kernel against the restatement
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [7, (1 << 63) | (0xABCD << 32) | 12345])
@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_mc_matches_restatement_many_models(gpu_ctx, growth, mode, seed):
    """300 models (more than the grid: every CTA loops over models), all eight masks mixed, 30 changepoints, every
    fifth model forecast inside its history (Tmax <= 1: no simulated changepoint), failed rows interleaved; a horizon of
    17 points (one full 16-point tile and a tail of one)."""
    rng = np.random.RandomState(1)
    H, N = 17, 300
    frs, fut = [], []
    for i in range(N):
        p, _ = _prep(ALL_MASKS[i % len(ALL_MASKS)], growth, mode, ncp=30)
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=(i % 5 == 3)))
    status = np.where(np.arange(N) % 7 == 5, L.ST_TOO_FEW, 0)
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=30)
    fb = _batch(frs, opts, status)
    assert fb.smax == 30 and fb.kmax == 34 and N > 132
    fut = np.stack(fut)
    floor = np.zeros(N) if growth == "linear" else rng.uniform(-5, 5, N)
    cap = np.array([fr.prep.cap_value for fr in frs])
    if growth == "logistic":     # the floor enters the logistic trend: keep cap above it
        cap = cap + floor
    _check_mc(gpu_ctx, fb, fut, floor, cap, growth, mode, 1000, 0.8, seed, ncp=30)


def test_mc_matches_restatement_sample_counts_and_widths(gpu_ctx):
    """n_samples 2 ... 1024 (odd and even, below and at the 1024-draw row) x interval widths 0 ... 1, with the dummy
    changepoint of n_changepoints = 0 (rate 1, lambda 1e-8)."""
    rng = np.random.RandomState(2)
    frs, fut = [], []
    for mask in (6, 2, 0):
        p, _ = _prep(mask, "logistic", "multiplicative", ncp=0)
        assert p.S == 1 and p.n_changepoints_real == 0
        frs.append(_model(p, rng))
        fut.append(_future(p, 16) if mask else _future(p, 400)[::25])
    fb = _batch(frs, batched.make_options(n_changepoints=0))
    assert fb.smax == 1
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    for n in (2, 33, 512, 513, 1000, 1024):
        for w in (0.0, 0.5, 0.8, 0.95, 1.0):
            _check_mc(gpu_ctx, fb, fut, np.zeros(3), cap, "logistic", "multiplicative", n, w, 3, ncp=0)


@pytest.mark.parametrize("H", [1, 15, 16, 17, 97, 672])
def test_mc_matches_restatement_horizons(gpu_ctx, H):
    rng = np.random.RandomState(3)
    frs, fut = [], []
    for mask, inside in ((6, False), (2, False), (7, True), (0, False)):
        p, _ = _prep(mask, "linear", "additive")
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=inside))
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    _check_mc(gpu_ctx, fb, np.stack(fut), np.zeros(4), np.ones(4), "linear", "additive", 1000, 0.8, 11)


def test_mc_bitonic_fallback_agrees_with_restatement(gpu_ctx):
    """Points just past the history's end with sigma_obs = 0: most draws have met no simulated changepoint yet and
    share one value exactly, so the histogram bin of the target ranks holds far more than 64 draws and the kernel
    selects by its full bitonic sort.  Both selection paths must give the restatement's percentiles."""
    p, _ = _prep(0, "linear", "additive")
    rng = np.random.RandomState(4)
    frs = [_model(p, rng, sigma=0.0, delta_scale=1.0) for _ in range(2)]
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    last = int(p.ds_sorted[-1])
    fut = np.stack([last + 20 * 10**9 * np.arange(1, 33, dtype=np.int64)] * 2)
    for w in (0.8, 0.95):
        _, ds = _check_mc(gpu_ctx, fb, fut, np.zeros(2), np.ones(2), "linear", "additive", 1000, w, 5)
        crowd = np.concatenate([mcs.crowded_bin(d, w) for d in ds])
        assert np.sum(crowd > 64) >= 8, crowd            # the premise: the fallback really runs at these points


# ---------------------------------------------------------------------------------------------------------------
# a model's intervals do not depend on its place in the batch
# ---------------------------------------------------------------------------------------------------------------
def _mixed_batch(N, growth="logistic", mode="multiplicative", H=24, seed=8):
    rng = np.random.RandomState(seed)
    frs, fut = [], []
    for i in range(N):
        p, _ = _prep([6, 2, 0][i % 3], growth, mode)
        frs.append(_model(p, rng))
        fut.append(_future(p, H))
    opts = batched.make_options(growth=growth, seasonality_mode=mode)
    return frs, _batch(frs, opts), np.stack(fut), opts


def test_mc_intervals_do_not_depend_on_batch_position(gpu_ctx):
    frs, fb, fut, opts = _mixed_batch(150)
    cap = np.array([fr.prep.cap_value for fr in frs])
    full = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(fb.n), cap, seed=21, intervals=True)
    # reversed rows 37..101, placed after other models: no model keeps its index
    idx = np.concatenate([np.arange(120, 140), np.arange(37, 102)[::-1]])
    sub = batched.predict_batch_host(gpu_ctx, opts, _take(fb, idx), fut[idx], np.zeros(idx.size), cap[idx], seed=21,
                                     intervals=True)
    assert np.array_equal(sub.yhat_lower, full.yhat_lower[idx]) and np.array_equal(sub.yhat_upper, full.yhat_upper[idx])
    assert np.array_equal(sub.yhat, full.yhat[idx])
    # a model alone gets the same intervals as in the batch; another seed gives other ones
    one = batched.predict_batch_host(gpu_ctx, opts, _take(fb, [77]), fut[[77]], np.zeros(1), cap[[77]], seed=21)
    assert np.array_equal(one.yhat_lower[0], full.yhat_lower[77])
    other = batched.predict_batch_host(gpu_ctx, opts, _take(fb, [77]), fut[[77]], np.zeros(1), cap[[77]], seed=22)
    assert not np.array_equal(other.yhat_lower[0], full.yhat_lower[77])


def test_scorer_rank_rows_match_single_rank_run(gpu_ctx, monkeypatch):
    """Under torchrun the scorer slices the model rows per rank: rank 1 of 2 must write exactly the rows (intervals
    included) that a single-rank run writes for its series."""
    frs, fb, fut, opts = _mixed_batch(40, H=8, seed=9)
    n = fb.n
    last = np.array([int(fr.prep.ds_sorted[-1]) for fr in frs], np.int64)
    tbl = pa.table({"series_id": pa.array(np.arange(n, dtype=np.int32)), "dim_id": pa.array(np.ones(n, np.int32)),
                    "floor": pa.array(np.zeros(n, np.float32)),
                    "cap": pa.array(np.array([fr.prep.cap_value for fr in frs], np.float32)),
                    "model": model_record.encode(fb, last, opts)})
    op = forecast_time_series({"forecast": {"periods": 8, "frequency": "h", "intervals": True, "seed": 5}})
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    full = op.apply_batched(tbl, ["series_id", "dim_id"]).to_pandas()
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "1")
    part = op.apply_batched(tbl, ["series_id", "dim_id"]).to_pandas()
    assert 0 < len(part) < len(full) and part["series_id"].min() > 0
    ref = full[full["series_id"].isin(part["series_id"].unique())].reset_index(drop=True)
    assert ref.equals(part.reset_index(drop=True))


# ---------------------------------------------------------------------------------------------------------------
# predict_kernel against the oracle given identical parameters
# ---------------------------------------------------------------------------------------------------------------
def _check_predict(gpu_ctx, frs, fut, opts, oopts, floor, cap):
    fb = _batch(frs, opts)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, floor, cap, intervals=False)
    worst = 0.0
    for i, fr in enumerate(frs):
        pr = po.predict(fr, fut[i], floor[i], cap[i], oopts)
        ys = fr.prep.y_scale
        err = np.max(np.abs(pr["yhat"] - fc.yhat[i])) / (ys * max(1.0, np.max(np.abs(pr["yhat"])) / ys))
        assert err <= PRED_TOL, (i, err)
        worst = max(worst, err)
        assert np.array_equal(fc.yhat_int[i], _epilogue(fc.yhat[i], floor[i]))
    _measured["predict"] = max(_measured["predict"], worst)
    return fc


def _epilogue(yhat, floor):
    """prophet_scorer.py:73-84 on the kernel's own yhat: truncate toward zero, values below the floor -> floor, then int32
    saturation.  Saturation is this library's choice; the reference's int64 -> Spark IntegerType path would wrap."""
    yt = np.trunc(yhat)
    yt = np.where(yt < floor, floor, yt)
    return np.clip(yt, INT32_MIN, INT32_MAX).astype(np.int64)


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_predict_matches_oracle_every_segment_and_era(gpu_ctx, growth, mode):
    """One batch with all eight masks (K = 34 / 14 / 28 / 8 / 26 / 6 / 20 / 0 packed into 34 columns: every block of beta
    at every offset a missing block leaves); histories in 1959, 2021 and 2250; timestamps across the whole history
    (every trend segment, the first point before the first changepoint included) and past its end."""
    rng = np.random.RandomState(5)
    frs, fut = [], []
    for start in ("1959-06-01", "2021-03-01", "2250-01-01"):
        for mask in ALL_MASKS:
            p, oopts = _prep(mask, growth, mode, start=start)
            frs.append(_model(p, rng))
            inside = p.ds_sorted[np.linspace(0, p.T - 1, 64).round().astype(int)]
            assert p.t_change[0] > 0                   # the first point (t = 0) lies before the first changepoint
            fut.append(np.concatenate([inside, _future(p, 32)]))
    opts = batched.make_options(growth=growth, seasonality_mode=mode)
    cap = np.array([fr.prep.cap_value for fr in frs])
    fc = _check_predict(gpu_ctx, frs, np.stack(fut), opts, oopts, np.zeros(len(frs)), cap)
    assert np.all(np.isfinite(fc.yhat))


@pytest.mark.parametrize("ncp,cpr", [(0, 0.8), (1, 0.8), (30, 1.0)])
@pytest.mark.parametrize("growth", ["logistic", "linear"])
def test_predict_matches_oracle_changepoint_counts(gpu_ctx, growth, ncp, cpr):
    rng = np.random.RandomState(6)
    frs, fut = [], []
    for mask in (6, 2, 0):
        p, oopts = _prep(mask, growth, "multiplicative", ncp=ncp, cpr=cpr)
        assert p.n_changepoints_real == ncp
        frs.append(_model(p, rng, delta_scale=0.5))
        fut.append(np.concatenate([p.ds_sorted[np.linspace(0, p.T - 1, 40).round().astype(int)], _future(p, 24)]))
    opts = batched.make_options(growth=growth, n_changepoints=ncp, changepoint_range=cpr)
    _check_predict(gpu_ctx, frs, np.stack(fut), opts, oopts, np.zeros(3), np.array([f.prep.cap_value for f in frs]))


def test_predict_long_horizon_beyond_tile_cap(gpu_ctx):
    """66 000 points per model: more than 64 CTAs x 1024 points, so the kernel's grid-stride loop covers the rest."""
    rng = np.random.RandomState(7)
    p, oopts = _prep(6, "linear", "multiplicative")
    frs = [_model(p, rng), _model(p, rng)]
    H = 66_000
    assert H > 64 * 1024
    fut = np.stack([int(p.ds_sorted[-1]) + MIN15 * np.arange(1, H + 1, dtype=np.int64)] * 2)
    _check_predict(gpu_ctx, frs, fut, batched.make_options(growth="linear"), oopts, np.zeros(2), np.ones(2))


def test_int_epilogue_exact(gpu_ctx):
    """yhat_int == clamp(trunc(yhat), floor) with int32 saturation, on a falling linear additive trend from +5 to -5
    (so -0.7 -> 0 and -3.2 -> -3 under floor -5), floors 0, -2, -5 and 3, a model whose |yhat| passes 2^31, and a failed
    row (NaN / INT32_MIN)."""
    p, _ = _prep(0, "linear", "additive")
    opts = batched.make_options(growth="linear", seasonality_mode="additive")
    fr = po.FitResult(prep=p, k=-1.0, m=0.5, delta=np.zeros(p.S), sigma_obs=0.01, beta=np.zeros(p.K), theta=None,
                      neg_logp=0.0, iters=0, n_evals=0, ret=0)
    fb = _batch([fr] * 7, opts, status=np.array([0, 0, 0, 0, 0, 0, L.ST_TOO_FEW]))
    fb.meta_f64[:, 0] = [10.0, 10.0, 10.0, 10.0, 1e10, 1e10, 10.0]
    H = 1440
    fut = np.stack([int(p.ds_sorted[0]) + 60 * 10**9 * np.arange(H, dtype=np.int64)] * 7)   # t from 0 to ~1
    floor = np.array([0.0, -2.0, -5.0, 3.0, 0.0, -1e12, 0.0])
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, floor, np.ones(7), intervals=False)
    for i in range(6):
        assert np.array_equal(fc.yhat_int[i], _epilogue(fc.yhat[i], floor[i])), i
        t = (fut[i] - p.start_ns) / p.t_scale_ns
        assert np.max(np.abs(fc.yhat[i] - (-t + 0.5) * fb.meta_f64[i, 0])) <= 1e-12 * fb.meta_f64[i, 0]
    y, yi = fc.yhat, fc.yhat_int
    near = lambda row, v: np.argmin(np.abs(y[row] - v))      # noqa: E731
    assert yi[0, near(0, -0.7)] == 0 and yi[2, near(2, -0.7)] == 0 and yi[2, near(2, -3.2)] == -3
    assert yi[1, near(1, -3.2)] == -2 and yi[3, near(3, 1.5)] == 3 and yi[3, near(3, 4.5)] == 4
    assert np.max(y[4]) > 2**31 and np.min(y[4]) < -2**31
    assert yi[4].max() == INT32_MAX and yi[4].min() == 0 and yi[5].min() == INT32_MIN
    assert np.all(np.isnan(y[6])) and np.all(yi[6] == INT32_MIN)

