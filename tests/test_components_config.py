"""The scorer's forecast.components option and the component columns' host side, and the trend draws of mc_kernel's
stream against fbprophet's process (DESIGN §12).  No GPU needed."""
import numpy as np
import pyarrow as pa
import pytest

import components_oracle as co
from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched
from time_series_spark_b200.frame import Frame
from time_series_spark_b200.jobs import prophet_scorer as ps
from time_series_spark_b200.jobs.prophet_scorer import ProphetScorer, forecast_time_series

_EMPTY = pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32()),
                   "floor": pa.array([], pa.float32()), "cap": pa.array([], pa.float32()),
                   "model": pa.array([], pa.binary())})


def _run_empty(fc):
    return forecast_time_series({"forecast": {"periods": 4, "frequency": "h", **fc}}).apply_batched(
        _EMPTY, ["series_id", "dim_id"])


@pytest.mark.parametrize("bad", ["yes", 1, 0, None, "true", [True]])
def test_components_must_be_a_bool(bad):
    with pytest.raises(ValueError, match="forecast.components"):
        _run_empty({"components": bad})


@pytest.mark.parametrize("intervals", [False, True])
@pytest.mark.parametrize("components", [False, True])
def test_empty_shard_schema_carries_the_component_columns(components, intervals):
    out = _run_empty({"components": components, "intervals": intervals})
    want = ["series_id", "dim_id", "ds", "yhat"] + (["yhat_lower", "yhat_upper"] if intervals else [])
    if components:
        want += list(ps.COMPONENT_COLUMNS) + (["trend_lower", "trend_upper"] if intervals else [])
    assert out.column_names == want and out.num_rows == 0
    for c in want[4:]:
        assert out.schema.field(c).type == pa.float64()


def _fake_result(n, h, intervals):
    rng = np.random.RandomState(0)
    comp = rng.randn(L.N_COMPONENTS, n, h)
    tlo = rng.randn(n, h) if intervals else None
    return batched.ForecastBatch(None, None, None, None, None, comp, tlo, tlo + 1.0 if intervals else None)


@pytest.mark.parametrize("intervals", [False, True])
def test_component_columns_null_where_the_mask_lacks_the_seasonality(intervals):
    n, h = 8, 3
    res = _fake_result(n, h, intervals)
    mask = np.arange(8, dtype=np.int32)
    cols = ps.component_columns(res, mask, h, intervals)
    assert list(cols) == list(ps.COMPONENT_COLUMNS) + (["trend_lower", "trend_upper"] if intervals else [])
    for name in ps.COMPONENT_COLUMNS:
        v = cols[name].to_numpy(zero_copy_only=False)
        ref = res.component(name).reshape(-1)
        bit = {"yearly": 1, "weekly": 2, "daily": 4}.get(name)
        valid = np.repeat(mask & bit != 0, h) if bit else np.ones(n * h, bool)
        assert np.array_equal(cols[name].is_valid().to_numpy(zero_copy_only=False), valid), name
        assert np.array_equal(v[valid], ref[valid]), name
    if intervals:
        assert np.array_equal(cols["trend_lower"].to_numpy(), res.trend_lower.reshape(-1))
        assert np.array_equal(cols["trend_upper"].to_numpy(), res.trend_upper.reshape(-1))


def _forecast_frame(n=5, components=True, intervals=True):
    t = {"series_id": pa.array(np.arange(n, dtype=np.int32)), "dim_id": pa.array(np.ones(n, np.int32)),
         "ds": pa.array(np.arange(n, dtype=np.int64) * 3600 * 10**9 + 10**18).cast(pa.timestamp("ns")),
         "yhat": pa.array(np.arange(n, dtype=np.int32))}
    if intervals:
        t["yhat_lower"] = pa.array(np.zeros(n))
        t["yhat_upper"] = pa.array(np.ones(n))
    if components:
        res = _fake_result(1, n, intervals)
        t.update(ps.component_columns(res, np.array([5]), n, intervals))
    return Frame(pa.table(t))


def test_convert_forecasts_passes_the_component_columns_through():
    f = _forecast_frame()
    out = ProphetScorer.convert_forecasts(f).table
    assert out.column_names == ["created_timestamp", "series_id", "dim_id", "forecast_date", "forecast_timestamp",
                                "forecast_quantity", "yhat_lower", "yhat_upper", *ps.COMPONENT_COLUMNS,
                                "trend_lower", "trend_upper"]
    for c in (*ps.COMPONENT_COLUMNS, "trend_lower", "trend_upper"):
        assert out[c].equals(f.table[c]), c
    assert out["weekly"].null_count == 5 and out["yearly"].null_count == 0


@pytest.mark.parametrize("intervals", [False, True])
def test_gpu_writer_refuses_a_frame_with_component_columns(intervals):
    conv = ProphetScorer.convert_forecasts(_forecast_frame(intervals=intervals))
    assert "standard six" in ps._gpu_writer_refusal(conv, big_only=False)


@pytest.mark.parametrize("growth", ["logistic", "linear"])
def test_trend_bounds_match_fbprophet_process(growth):
    """The restatement's trend draws and po.predict_uncertainty's trend bounds (fbprophet's process on numpy's RNG) at
    the same sample size agree within a few Monte-Carlo standard errors; where the draws are all equal (inside the
    history, and at early horizons for most draws) the bounds are the fitted trend itself."""
    n = 20_000
    rng = np.random.RandomState(3)
    ds = np.datetime64("2021-03-01", "ns").astype(np.int64) + 3600 * 10**9 * np.arange(720, dtype=np.int64)
    y = 100 + 10 * rng.rand(ds.size)
    oopts = po.ProphetOptions(growth=growth, seasonality_mode="multiplicative", uncertainty_samples=n)
    p = po.prepare(ds, y, 0.0, 130.0, oopts)
    delta = 0.5 * rng.laplace(size=p.S)
    beta = 0.05 * rng.randn(p.K)
    k, m, sigma = (0.8, -0.2, 0.02) if growth == "logistic" else (0.1, 0.7, 0.02)
    fr = po.FitResult(prep=p, k=k, m=m, delta=delta, sigma_obs=sigma, beta=beta, theta=None, neg_logp=0.0, iters=0,
                      n_evals=0, ret=0)
    rec = mcs.stack([mcs.record(p, k, m, sigma, delta, beta, 25, 14)], 25, 14)
    last = int(p.ds_sorted[-1])
    fut = np.concatenate([p.ds_sorted[[100, 500]], last + 3600 * 10**9 * np.array([1, 24, 72, 140, 216])])
    pr = co.predict(fr, fut, 0.0, 130.0, oopts)
    un = po.predict_uncertainty(fr, fut, pr, np.random.RandomState(0), oopts)
    d = co.trend_draws(rec, 0, fut, 0.0, 130.0, growth == "logistic", n, 99)
    lo, hi = mcs.bounds(d, oopts.interval_width)
    ys = p.y_scale
    # inside the history every draw is the fitted trend
    assert np.allclose(lo[:2], pr["trend"][:2], rtol=0, atol=1e-12 * ys)
    assert np.allclose(hi[:2], pr["trend"][:2], rtol=0, atol=1e-12 * ys)
    for q, mine, ref in ((0.1, lo, un["trend_lower"]), (0.9, hi, un["trend_upper"])):
        spread = (np.quantile(d, q + 0.02, axis=1) - np.quantile(d, q - 0.02, axis=1)) / 0.04
        se = np.sqrt(q * (1 - q) / n) * spread
        err = np.abs(mine - ref)
        assert np.all(err <= 5.0 * np.sqrt(2.0) * se + 1e-9 * ys), (growth, q, err, se)
    # the trend spread past the history grows with the horizon; lower <= upper
    assert (hi - lo)[-1] > (hi - lo)[3] > 0 and np.all(lo <= hi)
    # the restatement's trend is the one under its yhat draws: draws == trend (1 + s) + noise
    dy = mcs.draws(rec, 0, fut, 0.0, 130.0, growth == "logistic", True, n, 99)
    z = mcs.noise(*mcs.model_key(99, rec.params[0], rec.tchange[0], p.start_ns, p.t_scale_ns, ys, 0.0, 130.0), n,
                  fut.size)
    assert np.allclose(dy, d * (1.0 + pr["multiplicative_terms"][:, None]) + (sigma * ys) * z.T, rtol=0, atol=1e-9 * ys)


@pytest.mark.parametrize("mode", ["multiplicative", "additive"])
def test_oracle_components_sum_to_the_terms(mode):
    """The per-seasonality columns add up to po.predict's multiplicative / additive terms (fbprophet sums them the same
    way), and an absent seasonality is 0."""
    rng = np.random.RandomState(4)
    ds = np.datetime64("2021-03-01", "ns").astype(np.int64) + 3600 * 10**9 * np.arange(720, dtype=np.int64)
    oopts = po.ProphetOptions(growth="linear", seasonality_mode=mode)
    p = po.prepare(ds, 100 + rng.rand(ds.size), 0.0, 130.0, oopts)
    assert [s.name for s in p.seasonalities] == ["weekly", "daily"]
    fr = po.FitResult(prep=p, k=0.1, m=0.5, delta=np.zeros(p.S), sigma_obs=0.01, beta=0.1 * rng.randn(p.K), theta=None,
                      neg_logp=0.0, iters=0, n_evals=0, ret=0)
    pr = co.predict(fr, ds[-50:] + 86400 * 10**9, None, None, oopts)
    total = pr["yearly"] + pr["weekly"] + pr["daily"]
    key = "multiplicative_terms" if mode == "multiplicative" else "additive_terms"
    other = "additive_terms" if mode == "multiplicative" else "multiplicative_terms"
    assert np.allclose(total, pr[key], rtol=1e-13, atol=1e-13 * p.y_scale)
    assert np.all(pr["yearly"] == 0.0) and np.all(pr[other] == 0.0)
