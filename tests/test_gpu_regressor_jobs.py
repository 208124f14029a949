"""GPU tests of extra regressors through the jobs (DESIGN §20): the modeler on a synthetic hive tree with a promotion flag
and a price against the batched fit it stands for, the join of the future values against a pandas merge, the scorer
against the batched predict with the merged values, and the refusals of missing, NaN and repeated future values."""
import os

import numpy as np
import pyarrow as pa
import pyarrow.dataset as pads
import pyarrow.parquet as pq
import pytest

pytestmark = pytest.mark.gpu

M15 = 15 * 60 * 10**9
REGS = [{"name": "promo"}, {"name": "price", "prior_scale": 0.5}]
NAMES = ["promo", "price"]


def _promo(ds):
    return ((ds // (6 * 3600 * 10**9)) % 3 == 0).astype(np.float64)


def _price(ds, i):
    return 2.0 + 0.25 * i + np.sin(ds / (86400 * 10**9 * 2.3))


def _series(n=4):
    """config #3 (15-minute, 15 days) series with a flag and a price."""
    from time_series_spark_b200 import synth
    b = synth.config3(n=n)
    out = []
    for i in range(b.n):
        ds = b.ds[b.offsets[i]:b.offsets[i + 1]]
        y = b.y[b.offsets[i]:b.offsets[i + 1]].astype(np.int32)
        reg = np.stack([_promo(ds), _price(ds, i)])
        y = np.round(y * (1 + 0.3 * reg[0])).astype(np.int32)
        out.append((ds, y, reg))
    return out


def _fmt(v):
    return "" if v is None or (isinstance(v, float) and np.isnan(v)) else repr(float(v))


def _ts(t):
    return str(np.datetime64(int(t), "ns").astype("datetime64[s]")).replace("T", " ")


def _write_input(root, parts, null_y=()):
    """Header-less ``dim_id,timestamp,quantity,promo,price`` CSV under ``series_id=<100 + i>/``, dim_id 3; the rows
    ``null_y`` (series, row) get an empty quantity and empty regressor fields."""
    for i, (ds, y, reg) in enumerate(parts):
        d = os.path.join(root, "input", f"series_id={100 + i}")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "part.csv"), "w") as f:
            for k in range(ds.size):
                if (i, k) in null_y:
                    f.write(f"3,{_ts(ds[k])},,,\n")
                else:
                    f.write(f"3,{_ts(ds[k])},{int(y[k])},{_fmt(reg[0, k])},{_fmt(reg[1, k])}\n")
    return os.path.join(root, "input")


def _write_future(root, rows):
    """``rows``: series_id -> list of (dim_id, ds, promo, price); written in the order given."""
    for sid, rs in rows.items():
        d = os.path.join(root, "future", f"series_id={sid}")
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "part.csv"), "w") as f:
            f.write("".join(f"{did},{_ts(t)},{_fmt(a)},{_fmt(b)}\n" for did, t, a, b in rs))
    return os.path.join(root, "future")


def _model(root, parts, null_y=(), **io):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    out = os.path.join(root, "models")
    cfg = {"io": dict({"input": _write_input(root, parts, null_y), "models": out}, **io),
           "model": {"floor": 0, "cap_multiplier": 1.1, "regressors": REGS}}
    ProphetModeler.model(None, cfg)
    return pads.dataset(out, format="parquet").to_table().sort_by([("series_id", "ascending")])


@pytest.fixture(scope="module")
def modeled(tmp_path_factory):
    parts = _series()
    root = str(tmp_path_factory.mktemp("reg"))
    models = _model(root, parts, null_y={(1, 5)})
    return parts, models


def test_models_are_the_batched_fit(modeled, gpu_ctx):
    import torch
    from time_series_spark_b200 import batched, model_record
    from time_series_spark_b200.jobs import prophet_modeler as pm
    parts, models = modeled
    col = models["model"].combine_chunks()
    assert {int.from_bytes(b[4:6], "little") for b in col.to_pylist()} == {4}
    fb, last, info = model_record.decode(col)
    assert info["regressors"] == [{"name": "promo", "standardize": "auto"},
                                  {"name": "price", "prior_scale": 0.5, "standardize": "auto"}]
    # the same history, packed here from the arrays written (series 1 without its null-y row)
    keep = [np.ones(p[0].size, bool) for p in parts]
    keep[1][5] = False
    ds = np.concatenate([p[0][k] for p, k in zip(parts, keep)])
    y = np.concatenate([p[1][k] for p, k in zip(parts, keep)])
    reg = np.concatenate([p[2][:, k] for p, k in zip(parts, keep)], axis=1)
    off = np.concatenate(([0], np.cumsum([k.sum() for k in keep]))).astype(np.int64)
    opts = pm.options_from_config({"model": {"regressors": REGS}})
    d = batched.fit_batch_device(gpu_ctx, opts, torch.from_numpy(ds).cuda(), torch.from_numpy(y).cuda(), off, 0.0, 1.1,
                                 regressors=torch.from_numpy(np.ascontiguousarray(reg)).cuda()).to_host()
    for f in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64", "reg_scale"):
        assert getattr(fb, f).tobytes() == getattr(d, f).tobytes(), f
    assert (fb.meta_i32[:, 4] >= 0).all()
    assert last.tolist() == [int(p[0][-1]) for p in parts]
    # the flag is used as it is, the price standardised; the rule is batched.regressor_scales'
    want = batched.regressor_scales(reg, off, ["auto", "auto"])
    assert (fb.reg_scale[:, 0] == [0.0, 1.0]).all()
    np.testing.assert_allclose(fb.reg_scale, want, rtol=1e-12, atol=1e-12)


def test_nan_on_a_kept_row_fails_the_job(tmp_path):
    parts = _series(n=3)
    parts[2][2][1, 7] = np.nan
    with pytest.raises(ValueError, match=r"Found NaN in column price \(first offender: series_id 102, dim_id 3; 1 group"):
        _model(str(tmp_path), parts)


def _pandas_join(tab, sid, did, future):
    """The reference join: one left merge of the grid on (series_id, dim_id, ds)."""
    import pandas as pd
    n, h = future.shape
    grid = pd.DataFrame({"series_id": np.repeat(sid, h), "dim_id": np.repeat(did, h), "ds": future.reshape(-1)})
    t = tab.to_pandas()
    t["ds"] = t["ds"].astype("datetime64[ns]").astype(np.int64)
    m = grid.merge(t, on=["series_id", "dim_id", "ds"], how="left")
    return np.stack([m[c].to_numpy(np.float64) for c in NAMES]).reshape(len(NAMES), n, h)


@pytest.mark.parametrize("frequency, periods", [("15min", 96), ("MS", 4)])
def test_join_is_a_pandas_merge(gpu_ctx, frequency, periods):
    import torch
    from time_series_spark_b200 import batched
    from time_series_spark_b200.jobs.prophet_scorer import frequency_to_future
    from time_series_spark_b200.pack import pack_groups_cuda
    rng = np.random.RandomState(3)
    sid = np.array([5, 5, 6, 9, 7], np.int32)
    did = np.array([0, 1, 0, 0, 2], np.int32)
    last = np.array([0, 3, 7, 1, 2], np.int64) * M15 + np.datetime64("2021-01-31T12:00", "ns").astype(np.int64)
    future = frequency_to_future(last, periods, frequency)
    rows = []
    for i in range(sid.size):
        if sid[i] == 9:
            continue                                                  # an absent group
        pts = future[i][rng.rand(periods) < 0.8]                      # some points missing
        off = pts[:3] + 7 * 10**9                                     # off-grid rows
        early = last[i] - np.arange(1, 4) * M15                       # rows before the grid
        for t in np.concatenate((pts, off, early)):
            v = rng.rand(2)
            rows.append((sid[i], did[i], t, float(v[0] < 0.5), np.nan if rng.rand() < 0.05 else v[1] * 10))
    rows = [rows[k] for k in rng.permutation(len(rows))]              # unsorted
    tab = pa.table({"series_id": pa.array([r[0] for r in rows], pa.int32()),
                    "dim_id": pa.array([r[1] for r in rows], pa.int32()),
                    "ds": pa.array([r[2] for r in rows], pa.int64()).cast(pa.timestamp("ns")),
                    "promo": pa.array([r[3] for r in rows], pa.float64()),
                    "price": pa.array([r[4] for r in rows], pa.float64())})
    pk = pack_groups_cuda(tab, device="cuda", y_col=None, reg_cols=NAMES)
    assert pk.y is None and pk.ds.numel() == len(rows)
    from time_series_spark_b200.jobs.prophet_modeler import _group_keys
    gk = _group_keys(pk.series_id, pk.dim_id)
    mk = _group_keys(sid, did)
    group = np.array([int(np.flatnonzero(gk == k)[0]) if (gk == k).any() else -1 for k in mk], np.int64)
    fut, missing, first = batched.join_future_regressors_device(
        gpu_ctx, pk.ds, pk.offsets, pk.regressors, torch.from_numpy(group).cuda(), torch.from_numpy(future).cuda())
    want = _pandas_join(tab, sid, did, future)
    assert fut.cpu().numpy().tobytes() == np.ascontiguousarray(want).tobytes()
    present = {(r[0], r[1], r[2]) for r in rows}
    miss = np.array([[(sid[i], did[i], t) not in present for t in future[i]] for i in range(sid.size)])
    assert missing.cpu().numpy().tolist() == miss.sum(axis=1).tolist()
    assert missing.cpu().numpy()[3] == periods
    firsts = [int(future[i][np.flatnonzero(miss[i])[0]]) if miss[i].any() else np.iinfo(np.int64).min
              for i in range(sid.size)]
    assert first.cpu().numpy().tolist() == firsts


def _grid_rows(models, periods, frequency, extra=True):
    """io.future_regressors rows for every model's grid (plus off-grid rows), in reverse order."""
    from time_series_spark_b200 import model_record
    from time_series_spark_b200.jobs.prophet_scorer import frequency_to_future
    _, last, _ = model_record.decode(models["model"])
    fut = frequency_to_future(last, periods, frequency)
    out = {}
    for i, (s, d) in enumerate(zip(models["series_id"].to_pylist(), models["dim_id"].to_pylist())):
        ts = np.concatenate((fut[i], fut[i][:5] + M15 // 3)) if extra else fut[i]
        rs = [(d, int(t), float(_promo(np.array([t]))[0]), float(_price(np.array([t]), i)[0])) for t in ts]
        out[s] = rs[::-1]
    return out, fut


def _score(models, future_dir, **fc):
    from time_series_spark_b200.jobs.prophet_scorer import forecast_time_series
    cfg = {"io": {"future_regressors": future_dir},
           "forecast": dict({"periods": 96, "frequency": "15min", "seed": 5}, **fc)}
    return forecast_time_series(cfg).apply_batched(models, ["series_id", "dim_id"])


def test_scorer_is_the_batched_predict(modeled, gpu_ctx, tmp_path):
    from time_series_spark_b200 import model_record
    from time_series_spark_b200 import batched
    parts, models = modeled
    rows, fut = _grid_rows(models, 96, "15min")
    fdir = _write_future(str(tmp_path), rows)
    fb, _, info = model_record.decode(models["model"])
    floor = models["floor"].to_numpy().astype(np.float64)
    cap = models["cap"].to_numpy().astype(np.float64)
    n = fb.n
    freg = np.stack([np.stack([[r[2 + k] for r in rows[s][::-1][:96]] for s in models["series_id"].to_pylist()])
                     for k in range(2)])
    assert freg.shape == (2, n, 96)
    out = _score(models, fdir)
    det = model_record.regressor_options(info, uncertainty_samples=0)
    ref = batched.predict_batch_host(gpu_ctx, det, fb, fut, floor, cap, seed=5, intervals=False, regressors=freg)
    assert out.column_names == ["series_id", "dim_id", "ds", "yhat"]
    assert out["yhat"].to_numpy().tolist() == ref.yhat_int.reshape(-1).tolist()
    assert out["ds"].cast(pa.int64()).to_numpy().tolist() == fut.reshape(-1).tolist()
    out = _score(models, fdir, intervals=True, uncertainty_samples=300)
    mc = model_record.regressor_options(info, uncertainty_samples=300, interval_width=0.8)
    ref = batched.predict_batch_host(gpu_ctx, mc, fb, fut, floor, cap, seed=5, intervals=True, regressors=freg)
    assert out["yhat"].to_numpy().tolist() == ref.yhat_int.reshape(-1).tolist()
    for c, v in (("yhat_lower", ref.yhat_lower), ("yhat_upper", ref.yhat_upper)):
        assert out[c].to_numpy().tobytes() == np.ascontiguousarray(v).reshape(-1).tobytes(), c
    # the regressors move the forecast: a zero flag everywhere gives other values
    zero = freg.copy()
    zero[0] = 0.0
    other = batched.predict_batch_host(gpu_ctx, det, fb, fut, floor, cap, seed=5, intervals=False, regressors=zero)
    assert not np.array_equal(other.yhat, ref.yhat)
    # two ranks give the rows of one
    import time_series_spark_b200.dist as pdist
    orig = pdist.world
    got = []
    try:
        for rank in (0, 1):
            pdist.world = lambda: (rank, 2, rank)
            got.append(_score(models, fdir, intervals=True, uncertainty_samples=300))
    finally:
        pdist.world = orig
    both = pa.concat_tables(got)
    assert both.num_rows == out.num_rows
    for c in out.column_names:
        assert both[c].to_pylist() == out[c].to_pylist(), c


def test_scorer_refuses_missing_nan_and_repeated_values(modeled, tmp_path):
    _, models = modeled
    rows, fut = _grid_rows(models, 96, "15min", extra=False)
    sids = models["series_id"].to_pylist()
    # a missing grid point of the second model, and the whole third model
    r1 = {s: list(v) for s, v in rows.items()}
    r1[sids[1]] = r1[sids[1]][:-1]          # reversed: its first grid point
    r1.pop(sids[2])
    with pytest.raises(ValueError, match=rf"Found NaN in column promo: io\.future_regressors has no row for 97 forecast "
                                         rf"point\(s\) of 2 model\(s\) \(first: series_id {sids[1]}, dim_id 3, ds "):
        _score(models, _write_future(str(tmp_path / "a"), r1))
    # a NaN price
    r2 = {s: list(v) for s, v in rows.items()}
    d, t, a, _ = r2[sids[3]][10]
    r2[sids[3]][10] = (d, t, a, None)
    with pytest.raises(ValueError, match=rf"Found NaN in column price: .*1 forecast point\(s\) \(first: series_id "
                                         rf"{sids[3]}, dim_id 3"):
        _score(models, _write_future(str(tmp_path / "b"), r2))
    # a repeated row
    r3 = {s: list(v) for s, v in rows.items()}
    r3[sids[0]].append(r3[sids[0]][4])
    with pytest.raises(ValueError, match=rf"more than one row for series_id {sids[0]}, dim_id 3"):
        _score(models, _write_future(str(tmp_path / "c"), r3))


def test_written_models_and_forecasts(modeled, tmp_path):
    from time_series_spark_b200.jobs.prophet_scorer import ProphetScorer
    _, models = modeled
    mdir = tmp_path / "models"
    os.makedirs(mdir)
    pq.write_table(models, str(mdir / "part-00000.parquet"))
    rows, _ = _grid_rows(models, 8, "h")
    cfg = {"io": {"models": str(mdir), "forecasts": str(tmp_path / "fc"),
                  "future_regressors": _write_future(str(tmp_path), rows)},
           "forecast": {"periods": 8, "frequency": "h", "intervals": True}}
    ProphetScorer.score(None, cfg)
    t = pads.dataset(str(tmp_path / "fc"), format="csv").to_table()
    assert t.num_rows == models.num_rows * 8
    assert t.column_names[-2:] == ["yhat_lower", "yhat_upper"]


D = 24 * 3600 * 10**9
REGS3 = REGS + [{"name": "step"}]


def _step(ds):
    """A price that is constant for the first ten days and varies after: constant before the early cutoffs."""
    return np.where(ds - ds[0] < 10 * D, 1.5, 1.5 + np.cos(ds / (3600 * 10**9 * 7.0)))


def _cv_batch():
    parts = _series()
    ds = np.concatenate([p[0] for p in parts])
    y = np.concatenate([p[1] for p in parts])
    reg = np.concatenate([np.vstack([p[2], _step(p[0])[None]]) for p in parts], axis=1)
    off = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    caps = np.array([float(p[1].max()) * 1.1 for p in parts])
    return ds, y, np.ascontiguousarray(reg), off, caps


def _dev(fb):
    import torch
    from time_series_spark_b200 import batched
    return batched.FittedBatch(
        *(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64,
                                                                     fb.meta_f64)), fb.smax, fb.kmax,
        reg_scale=torch.from_numpy(np.ascontiguousarray(fb.reg_scale)).cuda())


def test_backtest_cutoff_fits_are_prophet_copy_fits(gpu_ctx):
    import sys
    import torch
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import backtest_oracle as bo
    from time_series_spark_b200 import batched
    ds, y, reg, off, caps = _cv_batch()
    std = ["auto"] * 3
    opts = batched.make_regressor_options(REGS3, uncertainty_samples=0)
    dds, dy, dreg = torch.from_numpy(ds).cuda(), torch.from_numpy(y).cuda(), torch.from_numpy(reg).cuda()
    hz, per, ini = D, D // 2, 3 * D
    # the full histories' scales: the library's kernel against the host rule
    fs, bad = batched.regressor_scales_device(gpu_ctx, opts, dreg, off)
    fs = fs.cpu().numpy()
    assert not bad.cpu().numpy().any()
    np.testing.assert_allclose(fs, batched.regressor_scales(reg, off, std), rtol=1e-12, atol=1e-12)
    res = batched.cross_validation_device(gpu_ctx, opts, dds, dy, off, 0.0, torch.from_numpy(caps).cuda(), hz, per, ini,
                                          rolling_window=0.1, keep_fits=True, regressors=dreg)
    assert (res.pair_status >= 0).all()
    he = np.concatenate([np.searchsorted(ds[off[i]:off[i + 1]], bo.generate_cutoffs(ds[off[i]:off[i + 1]], hz, per, ini),
                                         side="right") for i in range(off.size - 1)])
    f = res.fitted
    assert f.reg_scale.shape == (res.pair_series.size, 3, 2)
    seen_const = 0
    for mask in sorted(set(res.pair_mask.tolist())):
        # fbprophet's prophet_copy, built independently: the built-ins of the full fit, z of the prefix from the full
        # scales, the full scales as the copy
        oc = batched.make_regressor_options(REGS3, yearly_seasonality=bool(mask & 1), weekly_seasonality=bool(mask & 2),
                                            daily_seasonality=bool(mask & 4), uncertainty_samples=0)
        sel = np.flatnonzero(res.pair_mask == mask)
        ser = res.pair_series[sel]
        rows = [np.arange(off[s], off[s] + he[p]) for s, p in zip(ser, sel)]
        hoff = np.concatenate(([0], np.cumsum([r.size for r in rows]))).astype(np.int64)
        hi = np.concatenate(rows)
        si = np.repeat(ser, [r.size for r in rows])
        z = np.ascontiguousarray((reg[:, hi] - fs[si, :, 0].T) / fs[si, :, 1].T)
        d = batched.fit_batch_device(gpu_ctx, oc, torch.from_numpy(ds[hi]).cuda(), torch.from_numpy(y[hi]).cuda(), hoff,
                                     0.0, 1.0, cap=torch.from_numpy(caps[ser]).cuda(), regressors=torch.from_numpy(z).cuda(),
                                     reg_scale_copy=torch.from_numpy(np.ascontiguousarray(fs[ser])).cuda()).to_host()
        w = d.params.shape[1]
        assert f.params[sel, :w].tobytes() == d.params.tobytes()
        for name in ("tchange", "meta_i64", "meta_f64", "reg_scale"):
            assert getattr(f, name)[sel].tobytes() == getattr(d, name).tobytes(), name
        assert np.delete(f.meta_i32[sel], 3, axis=1).tobytes() == np.delete(d.meta_i32, 3, axis=1).tobytes()
        # the per-cutoff (mu, std) against the host rule: the decision exact, the values to rounding
        want = batched.regressor_scales(z, hoff, std, copy=fs[ser])
        copied = np.all(want == fs[ser], axis=2)
        assert np.array_equal(copied, np.all(d.reg_scale == fs[ser], axis=2))
        np.testing.assert_allclose(d.reg_scale, want, rtol=1e-12, atol=1e-12)
        assert copied[:, 0].all()                              # the flag: (0, 1) at every cutoff
        n10 = np.array([np.searchsorted(ds[off[s]:off[s + 1]], ds[off[s]] + 10 * D) for s in ser])
        const = he[sel] <= n10
        seen_const += int(const.sum())
        assert copied[const, 2].all()                          # the step's constant prefix keeps the full scale
        # the held-out predictions, with the cutoff fits' own scales on z of the held-out rows
        hmax = int(max(((res.row_series == s) & (res.cutoff == res.pair_cutoff[p])).sum() for s, p in zip(ser, sel)))
        fut = np.zeros((sel.size, hmax), np.int64)
        zf = np.zeros((3, sel.size, hmax))
        for j, p in enumerate(sel):
            s = int(res.pair_series[p])
            r = np.flatnonzero((res.row_series == s) & (res.cutoff == res.pair_cutoff[p]))
            src = off[s] + he[p] + np.arange(r.size)
            assert (ds[src] == res.ds[r]).all()
            fut[j, :r.size], fut[j, r.size:] = res.ds[r], res.ds[r][-1]
            zf[:, j, :r.size] = (reg[:, src] - fs[s, :, :1]) / fs[s, :, 1:]
        pr = batched.predict_batch_device(gpu_ctx, oc, _dev(d), torch.from_numpy(fut).cuda(),
                                          torch.zeros(sel.size, dtype=torch.float64).cuda(),
                                          torch.from_numpy(caps[ser]).cuda(), intervals=False,
                                          regressors=torch.from_numpy(zf).cuda())
        yh = pr.yhat.cpu().numpy()
        for j, p in enumerate(sel):
            r = np.flatnonzero((res.row_series == res.pair_series[p]) & (res.cutoff == res.pair_cutoff[p]))
            assert res.yhat[r].tobytes() == yh[j, :r.size].tobytes()
    assert seen_const > 0
    m = res.metrics
    for s in range(off.size - 1):
        r = res.row_series == s
        want = bo.performance_metrics(res.ds[r] - res.cutoff[r], res.y[r], res.yhat[r], None, None, 0.1)
        g = m["series"] == s
        assert m["horizon"][g].tolist() == want["horizon"].tolist()
        for k in ("mse", "rmse", "mae", "mape"):
            np.testing.assert_allclose(m[k][g], want[k], rtol=1e-12, atol=0, equal_nan=True)


def test_backtest_of_a_flag_is_the_plain_fit(gpu_ctx):
    import torch
    from time_series_spark_b200 import batched
    ds, y, reg, off, caps = _cv_batch()
    opts = batched.make_regressor_options(REGS[:1], uncertainty_samples=0)
    flag = np.ascontiguousarray(reg[:1])
    res = batched.cross_validation_device(gpu_ctx, opts, torch.from_numpy(ds).cuda(), torch.from_numpy(y).cuda(), off,
                                          0.0, torch.from_numpy(caps).cuda(), D, D // 2, 3 * D, keep_fits=True,
                                          regressors=torch.from_numpy(flag).cuda())
    for mask in sorted(set(res.pair_mask.tolist())):
        sel = np.flatnonzero(res.pair_mask == mask)
        ser = res.pair_series[sel]
        cut = res.pair_cutoff[sel]
        rows = [np.arange(off[s], off[s] + np.searchsorted(ds[off[s]:off[s + 1]], c, side="right")) for s, c in zip(ser, cut)]
        hoff = np.concatenate(([0], np.cumsum([r.size for r in rows]))).astype(np.int64)
        hi = np.concatenate(rows)
        oc = batched.make_regressor_options(REGS[:1], yearly_seasonality=bool(mask & 1), weekly_seasonality=bool(mask & 2),
                                            daily_seasonality=bool(mask & 4), uncertainty_samples=0)
        d = batched.fit_batch_device(gpu_ctx, oc, torch.from_numpy(ds[hi]).cuda(), torch.from_numpy(y[hi]).cuda(), hoff,
                                     0.0, 1.0, cap=torch.from_numpy(caps[ser]).cuda(),
                                     regressors=torch.from_numpy(np.ascontiguousarray(flag[:, hi])).cuda()).to_host()
        w = d.params.shape[1]
        assert res.fitted.params[sel, :w].tobytes() == d.params.tobytes()
        assert res.fitted.reg_scale[sel].tobytes() == d.reg_scale.tobytes()
        assert res.fitted.meta_f64[sel].tobytes() == d.meta_f64.tobytes()


def test_backtest_job_with_regressors(tmp_path):
    from time_series_spark_b200.jobs.prophet_backtest import ProphetBacktester
    parts = _series(n=3)
    root = str(tmp_path)
    inp = _write_input(root, parts, null_y={(0, 3)})
    cfg = {"io": {"input": inp, "metrics": os.path.join(root, "m"), "cv_rows": os.path.join(root, "r")},
           "model": {"floor": 0, "cap_multiplier": 1.1, "regressors": REGS},
           "backtest": {"horizon": "1 days", "intervals": True, "uncertainty_samples": 100}}
    metrics, rows = ProphetBacktester.run(None, cfg)
    assert metrics.num_rows > 0 and rows.num_rows > 0
    assert np.isfinite(rows["yhat"].to_numpy()).all() and np.isfinite(rows["yhat_lower"].to_numpy()).all()
    bad = _series(n=3)
    bad[1][2][1, 40] = np.nan
    cfg["io"]["input"] = _write_input(os.path.join(root, "bad"), bad)
    with pytest.raises(ValueError, match=r"Found NaN in column price \(first offender: series_id 101, dim_id 3"):
        ProphetBacktester.run(None, cfg)
