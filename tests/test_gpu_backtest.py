"""GPU tests of the backtest (cv_kernel.cuh, batched.cross_validation_device, jobs/prophet_backtest.py) against the
oracle's restatement of fbprophet.diagnostics (DESIGN §9)."""
import os
import sys

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper module next to this file
import backtest_oracle as bo  # noqa: E402
from oracle import mc_stream
from oracle import prophet_oracle as po

pytestmark = pytest.mark.gpu

H = 3600 * 10**9
D = 24 * H
HORIZON, PERIOD, INITIAL = D, D // 2, 3 * D
FLOOR, CAPM = 0.0, 1.1


def _mixed_batch():
    """config #3 (15-min, 15 days: the truncated histories' auto mask lacks weekly, the full one has it) and config #2
    (daily: one-row windows) slices, plus irregular hourly series with gaps (closest-date branch, padded windows)."""
    from time_series_spark_b200 import synth
    parts = []
    b3 = synth.config3(n=5)
    b2 = synth.config2(n=3)
    for b in (b3, b2):
        for i in range(b.n):
            parts.append((b.ds[b.offsets[i]:b.offsets[i + 1]], b.y[b.offsets[i]:b.offsets[i + 1]].astype(np.int32)))
    rng = np.random.RandomState(7)
    t0 = int(b3.ds[0])
    for k in range(4):
        steps = rng.randint(1, 4, 400).astype(np.int64) * H
        steps[150 + 20 * k] += (2 + k) * D + 5 * H                 # a gap longer than the horizon
        ds = t0 + np.cumsum(steps)
        parts.append((ds, rng.randint(0, 40, ds.size).astype(np.int32)))
    offsets = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), offsets


@pytest.fixture(scope="module")
def batch():
    return _mixed_batch()


def _run(ctx, ds, y, offsets, intervals=False, keep_fits=False, budget=None, seed=3):
    import torch
    from time_series_spark_b200 import batched
    opts = batched.make_options(uncertainty_samples=200 if intervals else 0)
    dds, dy = torch.from_numpy(ds).cuda(), torch.from_numpy(y).cuda()
    cap = torch.tensor([float(y[a:b].max()) * CAPM for a, b in zip(offsets[:-1], offsets[1:])], dtype=torch.float64).cuda()
    res = batched.cross_validation_device(ctx, opts, dds, dy, offsets, FLOOR, cap, HORIZON, PERIOD, INITIAL,
                                          intervals=intervals, seed=seed, rolling_window=0.1, keep_fits=keep_fits,
                                          _row_budget=budget)
    return opts, res


@pytest.fixture(scope="module")
def run(gpu_ctx, batch):
    return _run(gpu_ctx, *batch, intervals=True, keep_fits=True)


def test_plan_matches_oracle(gpu_ctx, batch):
    import torch
    from time_series_spark_b200 import batched
    ds, y, off = batch
    plan = batched.cv_plan_device(gpu_ctx, batched.make_options(), torch.from_numpy(ds).cuda(), off, HORIZON, PERIOD, INITIAL)
    assert not plan.err.any()
    he, we, cut = plan.hist_end.cpu().numpy(), plan.win_end.cpu().numpy(), plan.cutoff.cpu().numpy()
    for i in range(off.size - 1):
        s = ds[off[i]:off[i + 1]]
        c = bo.generate_cutoffs(s, HORIZON, PERIOD, INITIAL)
        p0, p1 = plan.pair_off[i], plan.pair_off[i + 1]
        assert cut[p0:p1].tolist() == c.tolist()
        assert (he[p0:p1] - off[i]).tolist() == np.searchsorted(s, c, side="right").tolist()
        assert (we[p0:p1] - off[i]).tolist() == np.searchsorted(s, c + HORIZON, side="right").tolist()
        assert plan.mask[i] == bo.seasonality_mask(s)
    assert (plan.mask[:5] == 6).all()                      # config #3: weekly + daily from the full 15 days
    assert (np.diff(off) < 0).sum() == 0 and int((we - he).min()) >= 1


def test_plan_error_flags(gpu_ctx):
    import torch
    from time_series_spark_b200 import batched, _lib as L
    t = 10**18
    series = [np.arange(10, dtype=np.int64) * H + t,                                  # shorter than the horizon
              np.arange(30, dtype=np.int64) * H + t,                                  # no cutoff after initial
              np.concatenate(([t], t + 20 * D + np.arange(0, 5 * 24) * H)),           # one row before a cutoff
              np.arange(200, dtype=np.int64) * H + t]                                 # fine
    ds = np.concatenate(series)
    off = np.concatenate(([0], np.cumsum([s.size for s in series]))).astype(np.int64)
    plan = batched.cv_plan_device(gpu_ctx, batched.make_options(), torch.from_numpy(ds).cuda(), off, D, D // 2, D)
    assert plan.err.tolist() == [L.CV_ERR_HORIZON, L.CV_ERR_INITIAL, L.CV_ERR_FEW, 0]
    for i, bit in ((0, "Less data than horizon."), (1, "after initial window")):
        with pytest.raises(ValueError, match=bit):
            bo.generate_cutoffs(series[i], D, D // 2, D)


def test_fits_equal_direct_fits(gpu_ctx, batch, run):
    from time_series_spark_b200 import batched
    ds, y, off = batch
    opts, res = run
    f = res.fitted
    he = np.concatenate([np.searchsorted(ds[off[i]:off[i + 1]], bo.generate_cutoffs(ds[off[i]:off[i + 1]], HORIZON, PERIOD, INITIAL), side="right")
                         for i in range(off.size - 1)])
    assert (res.pair_status >= 0).all()
    for mask in np.unique(res.pair_mask):
        sel = np.flatnonzero(res.pair_mask == mask)
        oc = batched._with_mask(opts, int(mask))
        parts = [(ds[off[res.pair_series[p]]:off[res.pair_series[p]] + he[p]], y[off[res.pair_series[p]]:off[res.pair_series[p]] + he[p]])
                 for p in sel]
        o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
        cap = np.array([float(y[off[s]:off[s + 1]].max()) * CAPM for s in res.pair_series[sel]])
        d = batched.fit_batch_host(gpu_ctx, oc, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]),
                                   o2, FLOOR, 1.0, cap=cap)
        w = d.params.shape[1]
        assert f.params[sel, :w].tobytes() == d.params.tobytes()
        assert not f.params[sel, w:].any()
        for name in ("tchange", "meta_i32", "meta_i64", "meta_f64"):
            assert getattr(f, name)[sel].tobytes() == getattr(d, name).tobytes(), name


def _oracle_fit_result(ds_hist, y_hist, cap, f, p, opts_mask):
    prep = po.prepare(ds_hist, y_hist.astype(np.float64), FLOOR, cap, opts_mask)
    S, smax = int(f.meta_i32[p, 1]), f.smax
    pr = f.params[p]
    return po.FitResult(prep=prep, k=pr[0], m=pr[1], delta=pr[3:3 + S].copy(), sigma_obs=pr[2],
                        beta=pr[3 + smax:3 + smax + prep.K].copy() if prep.seasonalities else np.zeros(1),
                        theta=None, neg_logp=0.0, iters=0, n_evals=0, ret=0)


def test_prediction_and_intervals_match_oracle(batch, run):
    ds, y, off = batch
    opts, res = run
    f = res.fitted
    rng = np.random.RandomState(0)
    pairs = rng.choice(res.pair_series.size, 12, replace=False)
    for p in pairs:
        s = int(res.pair_series[p])
        a, b = off[s], off[s + 1]
        c = res.pair_cutoff[p]
        he = a + int(np.searchsorted(ds[a:b], c, side="right"))
        m = int(res.pair_mask[p])
        oc = po.ProphetOptions(yearly_seasonality=bool(m & 1), weekly_seasonality=bool(m & 2), daily_seasonality=bool(m & 4))
        cap = float(y[a:b].max()) * CAPM
        fr = _oracle_fit_result(ds[a:he], y[a:he], cap, f, p, oc)
        rows = np.flatnonzero((res.row_series == s) & (res.cutoff == c))
        assert rows.size >= 1 and np.all(res.ds[rows] > c) and np.all(res.ds[rows] <= c + HORIZON)
        assert res.ds[rows].tolist() == ds[he:he + rows.size].tolist()           # no padded column in the output
        assert res.y[rows].tolist() == y[he:he + rows.size].astype(np.float64).tolist()
        pr = po.predict(fr, res.ds[rows], FLOOR, cap, oc)
        ys = float(f.meta_f64[p, 0])
        assert np.max(np.abs(pr["yhat"] - res.yhat[rows])) <= 1e-12 * ys
        if p in pairs[:3]:
            d = mc_stream.draws(f, int(p), res.ds[rows], FLOOR, cap, True, True, opts.uncertainty_samples, 3)
            lo, hi = mc_stream.bounds(d, opts.interval_width)
            assert np.max(np.abs(lo - res.yhat_lower[rows])) <= 1e-9 * ys
            assert np.max(np.abs(hi - res.yhat_upper[rows])) <= 1e-9 * ys


def test_metrics_match_oracle(batch, run):
    ds, y, off = batch
    _, res = run
    m = res.metrics
    for s in range(off.size - 1):
        r = res.row_series == s
        want = bo.performance_metrics(res.ds[r] - res.cutoff[r], res.y[r], res.yhat[r], res.yhat_lower[r],
                                      res.yhat_upper[r], 0.1)
        g = m["series"] == s
        assert m["horizon"][g].tolist() == want["horizon"].tolist()
        assert m["coverage"][g].tolist() == want["coverage"].tolist()
        for k in ("mse", "rmse", "mae", "mape"):
            np.testing.assert_allclose(m[k][g], want[k], rtol=1e-12, atol=0, equal_nan=True)
        if np.any(res.y[r] == 0):
            assert np.all(np.isnan(m["mape"][g]))


def _series_view(res, s):
    rs = res.row_series == s
    ms = res.metrics["series"] == s
    out = {k: getattr(res, k)[rs].tobytes() for k in ("ds", "cutoff", "y", "yhat")}
    out.update({"m_" + k: res.metrics[k][ms].tobytes() for k in ("horizon", "mse", "rmse", "mae", "mape")})
    return out


def test_independent_of_batch_and_chunks(gpu_ctx, batch):
    """Series 0-4 (config #3) and 8-11 (irregular): their mask classes stay below the fit's batch-size thresholds in
    every run here, so the fit dispatch is the same and the bits must be too.  (The daily series 5-7 are left out:
    ~720 cutoffs each, their class crosses the 8-series-per-SM threshold at which the fit changes its CTA width --
    DESIGN §9.)"""
    ds, y, off = batch
    keep = [0, 1, 2, 3, 4, 8, 9, 10, 11]
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in keep]
    off = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    ds, y = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    _, full = _run(gpu_ctx, ds, y, off)
    _, tiny = _run(gpu_ctx, ds, y, off, budget=1)
    pick = [7, 2, 8, 5, 0]
    parts = [(ds[off[i]:off[i + 1]], y[off[i]:off[i + 1]]) for i in pick]
    o2 = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    _, sub = _run(gpu_ctx, np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), o2)
    for s in range(off.size - 1):
        a, b = _series_view(full, s), _series_view(tiny, s)
        assert [k for k in a if a[k] != b[k]] == [], f"series {s}, chunked"
    for j, s in enumerate(pick):
        a, b = _series_view(full, s), _series_view(sub, j)
        assert [k for k in a if a[k] != b[k]] == [], f"series {s}, sub-batch position {j}"


def _config(tmp_path, inp, rows=True, **bt):
    cfg = {"io": {"input": inp, "metrics": str(tmp_path / "metrics")}, "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": {"horizon": "30 days", "period": "15 days", "initial": "180 days", **bt}}
    if rows:
        cfg["io"]["cv_rows"] = str(tmp_path / "rows")
    return cfg


def test_job_on_golden_fixture(tmp_path, model_input_dir, golden_input):
    from time_series_spark_b200.jobs.prophet_backtest import ProphetBacktester
    metrics, rows = ProphetBacktester.run(None, _config(tmp_path, model_input_dir, intervals=True, uncertainty_samples=100))
    m = pq.read_table(str(tmp_path / "metrics"))
    r = pq.read_table(str(tmp_path / "rows"))
    assert m.schema.names == ["series_id", "dim_id", "horizon", "mse", "rmse", "mae", "mape", "coverage"]
    assert m.schema.field("horizon").type == pa.duration("ns")
    assert r.schema.names == ["series_id", "dim_id", "ds", "cutoff", "y", "yhat", "yhat_lower", "yhat_upper"]
    assert m.num_rows > 0 and r.num_rows > 0 and set(m["series_id"].to_pylist()) == {751}
    # y is the input value of that (dim_id, ds)
    gi = golden_input
    src = {}
    for d, t, q in zip(gi["dim_id"], gi["ds_ns"], gi["y"]):
        src.setdefault((int(d), int(t)), []).append(int(q))       # (the fixture repeats some timestamps)
    dims, tss, ys = r["dim_id"].to_numpy(), r["ds"].cast(pa.int64()).to_numpy(), r["y"].to_numpy()
    assert r["y"].type == pa.int32()
    assert all(int(q) in src[(int(d), int(t))] for d, t, q in zip(dims, tss, ys))
    c = m["coverage"].to_numpy()
    assert np.all((c >= 0) & (c <= 1))
    m2, r2 = ProphetBacktester.run(None, _config(tmp_path, model_input_dir, rows=False))
    assert r2 is None and m2.schema.names == ["series_id", "dim_id", "horizon", "mse", "rmse", "mae", "mape"]


def test_job_on_synth_tree_and_failed_fit_rule(tmp_path, capsys):
    import copy
    from time_series_spark_b200 import synth
    from time_series_spark_b200.jobs import prophet_backtest as pb
    b = synth.config3(n=6)
    tbl = pa.table({"series_id": pa.array(np.repeat(np.arange(b.n) + 100, np.diff(b.offsets)), pa.int32()),
                    "dim_id": pa.array(np.full(int(b.offsets[-1]), 3), pa.int32()),
                    "ds": pa.array(b.ds, pa.timestamp("ns")), "y": pa.array(b.y.astype(np.int32), pa.int32())})
    cfg = {"io": {"metrics": str(tmp_path / "m"), "cv_rows": str(tmp_path / "r")}, "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": {"horizon": "1 days"}}
    job = pb.ProphetBacktester(cfg)
    metrics, rows = job.backtest(tbl)
    assert sorted(set(metrics["series_id"].to_pylist())) == list(range(100, 106))
    assert rows["y"].type == pa.int32()
    # 15 days of 15-minute rows, horizon 1 day, period 12 h, initial 3 days: 22 cutoffs of 96 held-out rows each
    assert rows.num_rows == b.n * 22 * 96
    # the assembly rule: a series with one failed cutoff fit loses all its rows, with a printed line
    import torch
    from time_series_spark_b200 import batched
    from time_series_spark_b200.jobs.prophet_modeler import get_context
    ctx = get_context()
    opts = batched.make_options()
    cap = torch.tensor([float(b.y[a:e].max()) * 1.1 for a, e in zip(b.offsets[:-1], b.offsets[1:])], dtype=torch.float64).cuda()
    res = batched.cross_validation_device(ctx, opts, torch.from_numpy(b.ds).cuda(), torch.from_numpy(b.y.astype(np.int32)).cuda(),
                                          b.offsets, 0.0, cap, D, D // 2, 3 * D, rolling_window=0.1)
    res2 = copy.deepcopy(res)
    bad = np.flatnonzero(res2.pair_series == 2)[5]
    res2.pair_status[bad] = -1
    sid, did = np.arange(b.n) + 100, np.full(b.n, 3)
    m_ok, r_ok = pb.assemble_outputs(sid, did, res, np.int32)
    capsys.readouterr()
    m_bad, r_bad = pb.assemble_outputs(sid, did, res2, np.int32)
    out = capsys.readouterr().out
    assert "series_id: 102" in out and "cutoff:" in out
    assert 102 not in m_bad["series_id"].to_pylist() and 102 not in r_bad["series_id"].to_pylist()
    assert m_bad.num_rows == m_ok.num_rows - m_ok["series_id"].to_pylist().count(102)
    assert r_bad.num_rows == r_ok.num_rows - r_ok["series_id"].to_pylist().count(102)


def test_job_too_few_rows_before_cutoff_names_the_group(tmp_path):
    from time_series_spark_b200.jobs import prophet_backtest as pb
    t = 1_600_000_000 * 10**9
    ds = np.concatenate([np.arange(200) * H + t, np.concatenate(([t], t + 20 * D + np.arange(0, 5 * 24) * H))])
    sid = np.concatenate([np.full(200, 1), np.full(121, 42)])
    tbl = pa.table({"series_id": pa.array(sid, pa.int32()), "dim_id": pa.array(np.full(ds.size, 9), pa.int32()),
                    "ds": pa.array(ds, pa.timestamp("ns")), "y": pa.array(np.arange(ds.size) % 7 + 1, pa.int32())})
    cfg = {"io": {"metrics": str(tmp_path / "m")}, "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": {"horizon": "1 days", "period": "12 hours", "initial": "1 days"}}
    with pytest.raises(ValueError, match=r"Less than two datapoints before cutoff.*series_id 42, dim_id 9"):
        pb.ProphetBacktester(cfg).backtest(tbl)
