"""GPU tests of seasonality tables through the jobs (DESIGN §18): the modeler and the scorer on a synthetic hive tree with
``model.seasonalities`` against the batched calls they stand for, the defaults-restating config, the backtest's
prophet_copy cutoff fits, and the refusals."""
import os
import sys

import numpy as np
import pyarrow as pa
import pyarrow.dataset as pads
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper module next to this file
import backtest_oracle as bo  # noqa: E402

pytestmark = pytest.mark.gpu

H = 3600 * 10**9
D = 24 * H
SEAS = [{"name": "monthly", "period": 30.5, "fourier_order": 3},
        {"name": "weekly", "period": 7, "fourier_order": 2, "prior_scale": 2.0}]


def _series():
    """config #3 (15-minute, 15 days: daily on, yearly off) and config #2 (daily, a year: daily and yearly off) series."""
    from time_series_spark_b200 import synth
    parts = []
    for b in (synth.config3(n=4), synth.config2(n=2)):
        for i in range(b.n):
            parts.append((b.ds[b.offsets[i]:b.offsets[i + 1]], b.y[b.offsets[i]:b.offsets[i + 1]].astype(np.int32)))
    return parts


def _write_tree(root, parts) -> str:
    """Header-less ``dim_id,timestamp,quantity`` CSV under ``series_id=<100 + i>/``, dim_id 3."""
    for i, (ds, y) in enumerate(parts):
        d = os.path.join(root, "input", f"series_id={100 + i}")
        os.makedirs(d, exist_ok=True)
        ts = ds.astype("datetime64[ns]").astype("datetime64[s]")
        with open(os.path.join(d, "part.csv"), "w") as f:
            f.write("\n".join(f"3,{str(t).replace('T', ' ')},{int(q)}" for t, q in zip(ts, y)) + "\n")
    return os.path.join(root, "input")


def _packed(parts):
    ds = np.concatenate([p[0] for p in parts])
    y = np.concatenate([p[1] for p in parts])
    off = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return ds, y, off


def _model(tmp_path, parts, **model):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    out = str(tmp_path / ("models_" + str(abs(hash(repr(sorted(model.items())))))))
    cfg = {"io": {"input": _write_tree(str(tmp_path), parts), "models": out},
           "model": dict({"floor": 0, "cap_multiplier": 1.1}, **model)}
    ProphetModeler.model(None, cfg)
    return pads.dataset(out, format="parquet").to_table().sort_by([("series_id", "ascending")])


def _score(models, **fc):
    from time_series_spark_b200.jobs.prophet_scorer import forecast_time_series
    cfg = {"io": {"aggregates": "unused"}, "forecast": dict({"periods": 96, "frequency": "15min", "seed": 5}, **fc)}
    op = forecast_time_series(cfg)
    out = op.apply_batched(models, ["series_id", "dim_id"])
    return out, op.aggregates


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).tobytes()


@pytest.fixture(scope="module")
def jobs_run(tmp_path_factory, gpu_ctx):
    from time_series_spark_b200 import batched
    parts = _series()
    models = _model(tmp_path_factory.mktemp("tab"), parts, seasonalities=SEAS)
    ds, y, off = _packed(parts)
    opts = batched.make_table_options(seasonalities=SEAS)
    direct = batched.fit_batch_host(gpu_ctx, opts, ds, y, off, 0.0, 1.1)
    return parts, models, opts, direct


def test_models_table_is_v2_and_the_direct_fit(jobs_run):
    from time_series_spark_b200 import batched, model_record
    parts, models, opts, direct = jobs_run
    col = models["model"].combine_chunks()
    assert {int.from_bytes(b[4:6], "little") for b in col.to_pylist()} == {2}
    fb, last, info = model_record.decode(col)
    assert info["table"]["seasonalities"] == [dict(SEAS[0], period=30.5), dict(SEAS[1], period=7.0)]
    assert batched.seasonality_table(model_record.table_options(info)) == batched.seasonality_table(opts)
    for f in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64"):
        assert getattr(fb, f).tobytes() == getattr(direct, f).tobytes(), f
    assert last.tolist() == [int(p[0][-1]) for p in parts]
    # config #3 keeps daily on, config #2 has neither daily nor yearly: table masks over monthly, weekly, yearly, daily
    assert fb.meta_i32[:, 3].tolist() == [0b1011] * 4 + [0b0011] * 2
    # the host restatement of the library's mask, from the built-in masks (weekly + daily, weekly)
    assert batched.table_mask(batched.seasonality_table(opts), np.array([6] * 4 + [2] * 2)).tolist() == \
        fb.meta_i32[:, 3].tolist()


def test_scorer_modes_equal_the_batched_calls(jobs_run, gpu_ctx):
    from time_series_spark_b200 import batched, model_record
    from time_series_spark_b200.jobs.prophet_scorer import quantile_column
    parts, models, _, _ = jobs_run
    fb, last, info = model_record.decode(models["model"])
    floor = models["floor"].to_numpy().astype(np.float64)
    cap = models["cap"].to_numpy().astype(np.float64)
    fut = batched.make_future(last, 96, 15 * 60 * 10**9)
    mc = model_record.table_options(info, uncertainty_samples=300, interval_width=0.8)
    det = model_record.table_options(info, uncertainty_samples=0)
    n = fb.n
    # plain
    out, _ = _score(models)
    ref = batched.predict_batch_host(gpu_ctx, det, fb, fut, floor, cap, seed=5, intervals=False)
    assert out["yhat"].to_numpy().tolist() == ref.yhat_int.reshape(-1).tolist()
    # intervals + components, with the custom column after additive_terms
    out, _ = _score(models, intervals=True, uncertainty_samples=300, components=True)
    ref = batched.predict_batch_host(gpu_ctx, mc, fb, fut, floor, cap, seed=5, intervals=True, components=True)
    assert out.column_names == ["series_id", "dim_id", "ds", "yhat", "yhat_lower", "yhat_upper", "trend", "yearly",
                                "weekly", "daily", "multiplicative_terms", "additive_terms", "monthly", "trend_lower",
                                "trend_upper"]
    assert _bits(out["yhat_lower"]) == _bits(ref.yhat_lower.reshape(-1))
    assert _bits(out["yhat_upper"]) == _bits(ref.yhat_upper.reshape(-1))
    for name in ("trend", "weekly", "multiplicative_terms", "additive_terms", "monthly"):
        assert out[name].null_count == 0
        assert _bits(out[name]) == _bits(ref.component(name).reshape(-1)), name
    assert out["yearly"].null_count == n * 96                    # yearly inactive everywhere
    daily = out["daily"].combine_chunks()
    assert daily.null_count == 2 * 96 and _bits(daily.to_numpy(zero_copy_only=False)[:4 * 96]) == \
        _bits(ref.component("daily")[:4].reshape(-1))
    # window totals and calendar-month totals
    _, agg = _score(models, intervals=True, uncertainty_samples=300, aggregate="6h")
    _, sums = batched.predict_sums_host(gpu_ctx, mc, fb, fut, floor, cap, 6 * H, 0, seed=5, intervals=True)
    keep = np.arange(sums.start.shape[1])[None, :] < sums.n_windows[:, None]
    for c, v in (("yhat", sums.yhat_sum), ("yhat_lower", sums.lower), ("yhat_upper", sums.upper)):
        assert _bits(agg[c]) == _bits(v[keep]), c
    futm = batched.make_future(last, 60, D)
    _, agg = _score(models, intervals=True, uncertainty_samples=300, aggregate_period="M", periods=60, frequency="D")
    _, sums = batched.predict_period_sums_host(gpu_ctx, mc, fb, futm, floor, cap, 1, 0, seed=5, intervals=True)
    keep = np.arange(sums.start.shape[1])[None, :] < sums.n_windows[:, None]
    for c, v in (("yhat", sums.yhat_sum), ("yhat_lower", sums.lower), ("yhat_upper", sums.upper)):
        assert _bits(agg[c]) == _bits(v[keep]), c
    # quantiles
    levels = [0.1, 0.5, 0.9]
    out, _ = _score(models, quantiles=levels, uncertainty_samples=300)
    ref = batched.predict_quantiles_host(gpu_ctx, mc, fb, fut, floor, cap, levels, seed=5, intervals=False)
    for q, lv in enumerate(levels):
        assert _bits(out[quantile_column(lv)]) == _bits(ref.quantiles[q].reshape(-1))


def test_written_forecasts_keep_the_custom_column(jobs_run, tmp_path):
    from time_series_spark_b200.jobs.prophet_scorer import ProphetScorer
    _, models, _, _ = jobs_run
    mdir = tmp_path / "models"
    os.makedirs(mdir)
    import pyarrow.parquet as pq
    pq.write_table(models, str(mdir / "part-00000.parquet"))
    cfg = {"io": {"models": str(mdir), "forecasts": str(tmp_path / "fc")},
           "forecast": {"periods": 4, "frequency": "15min", "components": True}}
    ProphetScorer.score(None, cfg)
    t = pads.dataset(str(tmp_path / "fc"), format="csv").to_table()
    assert t.column_names[-7:] == ["trend", "yearly", "weekly", "daily", "multiplicative_terms", "additive_terms",
                                   "monthly"]
    assert t.num_rows == models.num_rows * 4


def test_restating_config_writes_the_default_bytes(tmp_path):
    parts = _series()[:3]
    a = _model(tmp_path / "a", parts, yearly_seasonality=10)
    b = _model(tmp_path / "b", parts, yearly_seasonality=True)
    c = _model(tmp_path / "c", parts, seasonalities=[])
    d = _model(tmp_path / "d", parts)
    assert a["model"].to_pylist() == b["model"].to_pylist()
    assert c["model"].to_pylist() == d["model"].to_pylist()
    assert {int.from_bytes(x[4:6], "little") for x in a["model"].to_pylist() + c["model"].to_pylist()} == {1}


def test_insample_serves_a_table(tmp_path):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    parts = _series()[:2]
    cfg = {"io": {"input": _write_tree(str(tmp_path), parts), "models": str(tmp_path / "m"),
                  "fitted": str(tmp_path / "f")},
           "model": {"floor": 0, "cap_multiplier": 1.1, "seasonalities": SEAS},
           "insample": {"interval_width": 0.9, "uncertainty_samples": 100, "refit": True}}
    ProphetModeler.model(None, cfg)
    f = pads.dataset(str(tmp_path / "f"), format="parquet").to_table()
    assert f.num_rows == sum(p[0].size for p in parts)
    m = pads.dataset(str(tmp_path / "m"), format="parquet").to_table()
    assert {int.from_bytes(x[4:6], "little") for x in m["model"].to_pylist()} == {2}


def test_backtest_cutoff_fits_are_prophet_copy_fits(gpu_ctx):
    import torch
    from time_series_spark_b200 import batched
    parts = _series()
    ds, y, off = _packed(parts)
    opts = batched.make_table_options(seasonalities=SEAS, uncertainty_samples=0)
    dds, dy = torch.from_numpy(ds).cuda(), torch.from_numpy(y).cuda()
    caps = np.array([float(p[1].max()) * 1.1 for p in parts])
    hz, per, ini = D, D // 2, 3 * D
    res = batched.cross_validation_device(gpu_ctx, opts, dds, dy, off, 0.0, torch.from_numpy(caps).cuda(), hz, per, ini,
                                          rolling_window=0.1, keep_fits=True)
    assert (res.pair_status >= 0).all()
    assert sorted(set(res.pair_mask.tolist())) == [2, 6]            # yearly off everywhere, daily on config #3 only
    table = batched.seasonality_table(opts)
    he = np.concatenate([np.searchsorted(ds[off[i]:off[i + 1]], bo.generate_cutoffs(ds[off[i]:off[i + 1]], hz, per, ini),
                                         side="right") for i in range(off.size - 1)])
    f = res.fitted
    for mask in (2, 6):
        # fbprophet's prophet_copy, built independently: the custom entries, built-ins off unless the full fit had them
        oc = batched.make_table_options(seasonalities=SEAS, yearly_seasonality=bool(mask & 1),
                                        daily_seasonality=bool(mask & 4), uncertainty_samples=0)
        sel = np.flatnonzero(res.pair_mask == mask)
        hist = [(ds[off[res.pair_series[p]]:off[res.pair_series[p]] + he[p]],
                 y[off[res.pair_series[p]]:off[res.pair_series[p]] + he[p]]) for p in sel]
        hds, hy, hoff = _packed(hist)
        d = batched.fit_batch_device(gpu_ctx, oc, torch.from_numpy(hds).cuda(), torch.from_numpy(hy).cuda(), hoff, 0.0,
                                     1.0, cap=torch.from_numpy(caps[res.pair_series[sel]]).cuda()).to_host()
        w = d.params.shape[1]
        assert f.params[sel, :w].tobytes() == d.params.tobytes()
        assert not f.params[sel, w:].any()
        for name in ("tchange", "meta_i64", "meta_f64"):
            assert getattr(f, name)[sel].tobytes() == getattr(d, name).tobytes(), name
        assert np.delete(f.meta_i32[sel], 3, axis=1).tobytes() == np.delete(d.meta_i32, 3, axis=1).tobytes()
        assert (f.meta_i32[sel, 3] == int(batched.table_mask(table, mask))).all()
        # the held-out predictions of those fits, predicted with the cutoff options
        fut = np.zeros((sel.size, 96), np.int64)
        for j, p in enumerate(sel):
            s = int(res.pair_series[p])
            rows = np.flatnonzero((res.row_series == s) & (res.cutoff == res.pair_cutoff[p]))
            fut[j, :rows.size] = res.ds[rows]
            fut[j, rows.size:] = res.ds[rows][-1]
        fl = torch.zeros(sel.size, dtype=torch.float64).cuda()
        pr = batched.predict_batch_device(gpu_ctx, oc, batched.FittedBatch(
            *(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (d.params, d.tchange, d.meta_i32, d.meta_i64,
                                                                          d.meta_f64)), d.smax, d.kmax),
            torch.from_numpy(fut).cuda(), fl, torch.from_numpy(caps[res.pair_series[sel]]).cuda(), intervals=False)
        yh = pr.yhat.cpu().numpy()
        for j, p in enumerate(sel):
            s = int(res.pair_series[p])
            rows = np.flatnonzero((res.row_series == s) & (res.cutoff == res.pair_cutoff[p]))
            assert res.yhat[rows].tobytes() == yh[j, :rows.size].tobytes()
    m = res.metrics
    for s in range(off.size - 1):
        r = res.row_series == s
        want = bo.performance_metrics(res.ds[r] - res.cutoff[r], res.y[r], res.yhat[r], None, None, 0.1)
        g = m["series"] == s
        assert m["horizon"][g].tolist() == want["horizon"].tolist()
        for k in ("mse", "rmse", "mae", "mape"):
            np.testing.assert_allclose(m[k][g], want[k], rtol=1e-12, atol=0, equal_nan=True)


def test_backtest_job_takes_a_table_with_every_option(tmp_path):
    from time_series_spark_b200.jobs.prophet_backtest import ProphetBacktester
    parts = _series()[:3]
    inp = _write_tree(str(tmp_path), parts)
    base = {"model": {"floor": 0, "cap_multiplier": 1.1, "seasonalities": SEAS}}
    for k, bt in enumerate(({"intervals": True, "uncertainty_samples": 100},
                            {"intervals": True, "uncertainty_samples": 100, "aggregate": "6h"},
                            {"quantiles": [0.1, 0.9], "uncertainty_samples": 100})):
        io = {"input": inp, "metrics": str(tmp_path / f"m{k}"), "cv_rows": str(tmp_path / f"r{k}"),
              "window_metrics": str(tmp_path / f"w{k}"), "quantile_metrics": str(tmp_path / f"q{k}")}
        cfg = dict(base, io=io, backtest=dict({"horizon": "1 days"}, **bt))
        metrics, rows = ProphetBacktester.run(None, cfg)
        assert metrics.num_rows > 0 and rows.num_rows > 0
        assert np.isfinite(rows["yhat"].to_numpy()).all()


def test_refusals_end_to_end(tmp_path):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    from time_series_spark_b200.jobs.prophet_tuner import ProphetTuner
    parts = _series()[:2]
    inp = _write_tree(str(tmp_path), parts)
    models = _model(tmp_path / "prev", parts, seasonalities=SEAS)
    import pyarrow.parquet as pq
    os.makedirs(tmp_path / "prev_models")
    pq.write_table(models, str(tmp_path / "prev_models" / "part-00000.parquet"))
    cfg = {"io": {"input": inp, "models": str(tmp_path / "m"), "warm_start": str(tmp_path / "prev_models")},
           "model": {"floor": 0, "cap_multiplier": 1.1, "seasonalities": SEAS}}
    with pytest.raises(ValueError, match=r"io\.warm_start"):
        ProphetModeler.model(None, cfg)
    cfg["insample"] = {"interval_width": 0.8, "refit": True}
    with pytest.raises(ValueError, match=r"io\.warm_start.*insample\.refit"):
        ProphetModeler.model(None, cfg)
    tcfg = {"io": {"input": inp, "models": str(tmp_path / "t"), "tuning": str(tmp_path / "tt")},
            "model": {"floor": 0, "cap_multiplier": 1.1, "yearly_seasonality": 4}, "backtest": {"horizon": "1 days"}}
    with pytest.raises(ValueError, match=r"model\.yearly_seasonality: the tuner"):
        ProphetTuner.run(None, tcfg)
