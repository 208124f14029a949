"""Forecast components through the batched predict (DESIGN §12), run with -m gpu on an H100.

* The components call leaves yhat, yhat_int, yhat_lower and yhat_upper byte for byte what pb200_predict gives.
* Its planes keep fbprophet's identities: yhat == trend (1 + multiplicative_terms) exactly, multiplicative_terms is the
  sum of the seasonalities in seasonal_term's order exactly, yhat == trend + additive_terms up to the rounding of
  additive_terms; an absent seasonality is exactly 0, a failed model NaN everywhere.
* trend / additive columns within 1e-12 y_scale and multiplicative ones within 1e-12 of fbprophet's predict (the rule
  test_gpu_scorer.py holds yhat to), the trend bounds within 1e-9 y_scale of the restated trend draws.
* The scorer job's component columns.
"""
import ctypes
import functools

import numpy as np
import pyarrow as pa
import pyarrow.dataset as pads
import pytest

import components_oracle as co
from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, model_record, synth
from time_series_spark_b200.jobs import prophet_scorer as ps
from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler

pytestmark = pytest.mark.gpu

H_NS = 3600 * 10**9
DAY = 24 * H_NS
MIN15 = 15 * 60 * 10**9
MC_TOL = 1e-9
PRED_TOL = 1e-12
SEAS = {"yearly": 1, "weekly": 2, "daily": 4}
GROWTH_MODES = [("logistic", "multiplicative"), ("logistic", "additive"), ("linear", "multiplicative"),
                ("linear", "additive")]
_MASK_HIST = {7: (12 * H_NS, 1600, "auto"), 6: (H_NS, 720, "auto"), 5: (12 * H_NS, 1600, False),
              4: (H_NS, 240, "auto"), 3: (DAY, 801, "auto"), 2: (DAY, 60, "auto"), 1: (7 * DAY, 115, "auto"),
              0: (MIN15, 96, "auto")}
_measured = {"trend": 0.0, "add": 0.0, "mult": 0.0, "bounds": 0.0, "add_exact": [0, 0], "tie_rows": 0, "sort_rows": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    m = _measured
    print(f"\n[components] max deviation from the oracle: trend / additive {m['trend']:.3e} / {m['add']:.3e} (x y_scale), "
          f"multiplicative {m['mult']:.3e}; trend bounds {m['bounds']:.3e} x y_scale; yhat == trend + additive_terms "
          f"exactly at {m['add_exact'][0]} of {m['add_exact'][1]} additive points; trend rows by the tie shortcut "
          f"{m['tie_rows']}, by the bitonic sort {m['sort_rows']}")


@functools.lru_cache(maxsize=None)
def _prep(mask, growth, mode, ncp=25, cpr=0.8):
    step, T, weekly = _MASK_HIST[mask]
    ds = np.datetime64("2021-03-01", "ns").astype(np.int64) + step * np.arange(T, dtype=np.int64)
    y = 100.0 + 20.0 * np.sin(np.arange(T) / 7.0) + np.arange(T) % 5
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, n_changepoints=ncp, changepoint_range=cpr,
                              weekly_seasonality=weekly)
    p = po.prepare(ds, y, 0.0, 1.1 * y.max(), oopts)
    assert sum(mcs._MASK_BIT[s.name] for s in p.seasonalities) == mask
    return p, oopts


def _model(p, rng, sigma=0.03, delta_scale=0.3):
    delta = delta_scale * rng.laplace(size=p.S) if p.n_changepoints_real else np.zeros(p.S)
    beta = 0.05 * rng.randn(p.K) if p.seasonalities else np.zeros(p.K)
    k, m = (rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)) if p.logistic else (rng.uniform(-0.5, 0.5), rng.uniform(0.3, 0.7))
    return po.FitResult(prep=p, k=k, m=m, delta=delta, sigma_obs=sigma, beta=beta, theta=None, neg_logp=0.0, iters=0,
                        n_evals=0, ret=0)


def _batch(frs, opts, status=None):
    lay = L.get_layout(opts)
    ns = mcs.stack([mcs.record(fr.prep, fr.k, fr.m, fr.sigma_obs, fr.delta, fr.beta, lay.smax, lay.kmax) for fr in frs],
                   lay.smax, lay.kmax)
    if status is not None:
        ns.meta_i32[:, 4] = status
    return batched.FittedBatch(ns.params, ns.tchange, ns.meta_i32, ns.meta_i64, ns.meta_f64, lay.smax, lay.kmax)


def _take(fb, idx):
    return batched.FittedBatch(*(np.ascontiguousarray(a[idx]) for a in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64,
                                                                         fb.meta_f64)), fb.smax, fb.kmax)


def _future(p, H, in_history=False):
    step = int(p.ds_sorted[1] - p.ds_sorted[0])
    if in_history:
        return np.ascontiguousarray(p.ds_sorted[-H:])
    return int(p.ds_sorted[-1]) + step * np.arange(1, H + 1, dtype=np.int64)


def _kinds(d, width):
    """Per point of [H, n] draws: 'tie' if some target-rank histogram bin holds more than 64 draws and every such bin
    holds one value only (the kernel's tie shortcut), 'sort' if one such bin holds different values (its bitonic sort),
    else None."""
    H, n = d.shape
    ranks = mcs.target_ranks(n, width)
    out = []
    for p in range(H):
        row = d[p]
        mn, mx = row.min(), row.max()
        kind = None
        if mx > mn:
            b = np.minimum(255, ((row - mn) * (256.0 / (mx - mn))).astype(np.int64))
            sb = np.sort(b)
            for r in ranks:
                vals = row[b == sb[r]]
                if vals.size > 64:
                    if vals.min() != vals.max():
                        kind = "sort"
                        break
                    kind = "tie"
        out.append(kind)
    return out


def _run(gpu_ctx, fb, fut, floor, cap, growth, mode, ncp=25, n=1000, width=0.8, seed=7, intervals=True):
    """The components call and the plain call on the same inputs; checks that the plain outputs are byte-identical."""
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp, interval_width=width,
                                uncertainty_samples=n)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, floor, cap, seed=seed, intervals=intervals, components=True)
    ref = batched.predict_batch_host(gpu_ctx, opts, fb, fut, floor, cap, seed=seed, intervals=intervals)
    for a in ("yhat", "yhat_int", "yhat_lower", "yhat_upper"):
        x, y = getattr(fc, a), getattr(ref, a)
        assert (x is None) == (y is None), a
        if x is not None:
            assert x.tobytes() == y.tobytes(), a
    assert fc.components.shape == (L.N_COMPONENTS,) + fc.yhat.shape
    assert (fc.trend_lower is not None) == (intervals and n > 0)
    return fc


def _check_identities(fc, fb, mode):
    ok = fb.meta_i32[:, 4] >= 0
    comp = fc.components
    assert np.all(np.isnan(comp[:, ~ok])) and np.all(np.isnan(fc.yhat[~ok]))
    if fc.trend_lower is not None:
        assert np.all(np.isnan(fc.trend_lower[~ok])) and np.all(np.isnan(fc.trend_upper[~ok]))
        assert np.all(fc.trend_lower[ok] <= fc.trend_upper[ok])
    tr, mt, at = (fc.component(c)[ok] for c in ("trend", "multiplicative_terms", "additive_terms"))
    seas = {c: fc.component(c)[ok] for c in SEAS}
    mask = fb.meta_i32[ok, 3]
    for c, bit in SEAS.items():
        assert np.all(seas[c][(mask & bit) == 0] == 0.0), c
    yh = fc.yhat[ok]
    if mode == "multiplicative":
        assert np.all(at == 0.0)
        assert np.array_equal(mt, ((0.0 + seas["yearly"]) + seas["weekly"]) + seas["daily"])
        assert np.array_equal(yh, tr * (1.0 + mt))
    else:
        assert np.all(mt == 0.0)
        # yhat = fma(s, y_scale, trend); additive_terms = s * y_scale rounded: apart by that rounding and the sum's
        assert np.all(np.abs(yh - (tr + at)) <= np.abs(np.spacing(at)) + 2.0 * np.abs(np.spacing(yh)))
        _measured["add_exact"][0] += int(np.sum(yh == tr + at))
        _measured["add_exact"][1] += int(yh.size)
        ys = fb.meta_f64[ok, 0][:, None]
        tot = (seas["yearly"] + seas["weekly"]) + seas["daily"]
        assert np.all(np.abs(tot - at) <= 1e-13 * ys * np.maximum(1.0, np.abs(at) / ys))


def _check_oracle(fc, frs, fut, floor, cap, oopts):
    for i, fr in enumerate(frs):
        pr = co.predict(fr, fut[i], floor[i], cap[i], oopts)
        ys = fr.prep.y_scale
        for c in ("trend", "additive_terms", "multiplicative_terms", "yearly", "weekly", "daily"):
            mult = c == "multiplicative_terms" or (c in SEAS and oopts.seasonality_mode == "multiplicative")
            scale = 1.0 if mult else ys
            ref = pr[c]
            err = np.max(np.abs(fc.component(c)[i] - ref)) / (scale * max(1.0, np.max(np.abs(ref)) / scale))
            assert err <= PRED_TOL, (i, c, err)
            key = "mult" if mult else ("trend" if c == "trend" else "add")
            _measured[key] = max(_measured[key], err)


def _check_bounds(fc, fb, fut, floor, cap, growth, n, width, seed):
    kinds = []
    for i in range(fb.n):
        if fb.meta_i32[i, 4] < 0:
            continue
        d = co.trend_draws(fb, i, fut[i], floor[i], cap[i], growth == "logistic", n, seed)
        lo, hi = mcs.bounds(d, width)
        ys = fb.meta_f64[i, 0]
        err = max(np.max(np.abs(fc.trend_lower[i] - lo)), np.max(np.abs(fc.trend_upper[i] - hi))) / ys
        assert err <= MC_TOL, (i, n, width, err)
        _measured["bounds"] = max(_measured["bounds"], err)
        kinds += _kinds(d, width)
    _measured["tie_rows"] += kinds.count("tie")
    _measured["sort_rows"] += kinds.count("sort")
    return kinds


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncp", [0, 1, 25, 30])
@pytest.mark.parametrize("growth,mode", GROWTH_MODES)
def test_components_every_mask_and_changepoint_count(gpu_ctx, growth, mode, ncp):
    """All eight masks twice in one batch (the second forecast inside its history), failed rows interleaved, 17 points
    (one 16-point and two 8-point MC tiles and a tail of one)."""
    rng = np.random.RandomState(ncp + 10)
    frs, fut = [], []
    for i in range(16):
        p, oopts = _prep(i % 8, growth, mode, ncp=ncp)
        frs.append(_model(p, rng))
        fut.append(_future(p, 17, in_history=i >= 8))
    status = np.where(np.arange(16) % 7 == 5, L.ST_TOO_FEW, 0)
    opts = batched.make_options(growth=growth, seasonality_mode=mode, n_changepoints=ncp)
    fb = _batch(frs, opts, status)
    fut = np.stack(fut)
    floor = np.zeros(16) if growth == "linear" else rng.uniform(-5, 5, 16)
    cap = np.array([fr.prep.cap_value for fr in frs]) + floor
    for intervals in (False, True):
        fc = _run(gpu_ctx, fb, fut, floor, cap, growth, mode, ncp=ncp, intervals=intervals)
        _check_identities(fc, fb, mode)
    ok = status >= 0
    _check_oracle(_take_fc(fc, ok), [f for f, k in zip(frs, ok) if k], fut[ok], floor[ok], cap[ok], oopts)
    _check_bounds(fc, fb, fut, floor, cap, growth, 1000, 0.8, 7)


def _take_fc(fc, sel):
    return batched.ForecastBatch(None, fc.yhat[sel], None, None, None, fc.components[:, sel])


@pytest.mark.parametrize("H", [1, 7, 8, 9, 15, 16, 17, 672, 1025])
def test_components_horizons(gpu_ctx, H):
    """Horizons around both MC tiles (8 with trend bounds, 16 without) and predict's 1024-point tile."""
    rng = np.random.RandomState(H)
    frs, fut = [], []
    for mask, inside in ((6, False), (2, False), (7, True), (0, False)):
        p, oopts = _prep(mask, "linear", "additive")
        frs.append(_model(p, rng))
        fut.append(_future(p, H, in_history=inside))
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    fut = np.stack(fut)
    fc = _run(gpu_ctx, fb, fut, np.zeros(4), np.ones(4), "linear", "additive", seed=11)
    _check_identities(fc, fb, "additive")
    _check_oracle(fc, frs, fut, np.zeros(4), np.ones(4), oopts)
    _check_bounds(fc, fb, fut, np.zeros(4), np.ones(4), "linear", 1000, 0.8, 11)


def test_trend_bounds_sample_counts_and_widths(gpu_ctx):
    """2 ... 1024 draws x widths 0 ... 1, logistic, one model forecast inside its history (every draw equal)."""
    rng = np.random.RandomState(2)
    frs, fut = [], []
    for mask, inside in ((6, False), (2, True), (0, False)):
        p, _ = _prep(mask, "logistic", "multiplicative", ncp=0 if mask == 0 else 25)
        frs.append(_model(p, rng))
        fut.append(_future(p, 16, in_history=inside))
    # one layout for the batch: n_changepoints = 25 (the mask-0 model's dummy changepoint fits in it)
    fb = _batch(frs, batched.make_options())
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    for n in (2, 33, 512, 513, 1000, 1024):
        for w in (0.0, 0.5, 0.8, 0.95, 1.0):
            fc = _run(gpu_ctx, fb, fut, np.zeros(3), cap, "logistic", "multiplicative", n=n, width=w, seed=3)
            _check_bounds(fc, fb, fut, np.zeros(3), cap, "logistic", n, w, 3)
    assert np.array_equal(fc.trend_lower[1], fc.trend_upper[1])


def test_trend_rows_by_tie_shortcut_and_bitonic_sort(gpu_ctx):
    """Points just past a one-day history with 25 changepoints: most draws have met no simulated changepoint and their
    trends are exactly equal.  Where the crowded histogram bin holds that value only, the tie shortcut answers; where it
    also holds the trends of draws whose changepoint came just before the point, the bitonic sort does.  sigma_obs = 0
    gives the yhat rows the same ties.  Both selection paths must give the restatement's percentiles, and the yhat bounds
    stay the plain call's."""
    p, _ = _prep(0, "linear", "additive")
    rng = np.random.RandomState(4)
    frs = [_model(p, rng, sigma=s, delta_scale=1.0) for s in (0.0, 0.03, 0.0)]
    fb = _batch(frs, batched.make_options(growth="linear", seasonality_mode="additive"))
    last = int(p.ds_sorted[-1])
    fut = np.stack([last + 20 * 10**9 * np.arange(1, 33, dtype=np.int64), _future(p, 32),
                    last + 60 * 10**9 * np.arange(1, 33, dtype=np.int64)])
    kinds = []
    for w in (0.8, 0.95):
        fc = _run(gpu_ctx, fb, fut, np.zeros(3), np.ones(3), "linear", "additive", width=w, seed=5)
        kinds += _check_bounds(fc, fb, fut, np.zeros(3), np.ones(3), "linear", 1000, w, 5)
    assert kinds.count("tie") >= 2 and kinds.count("sort") >= 8, kinds      # the premise: both paths run


def test_trend_bounds_do_not_depend_on_batch_position(gpu_ctx):
    rng = np.random.RandomState(8)
    frs, fut = [], []
    for i in range(150):
        p, _ = _prep([6, 2, 0][i % 3], "logistic", "multiplicative")
        frs.append(_model(p, rng))
        fut.append(_future(p, 24))
    fb = _batch(frs, batched.make_options())
    fut = np.stack(fut)
    cap = np.array([fr.prep.cap_value for fr in frs])
    full = _run(gpu_ctx, fb, fut, np.zeros(150), cap, "logistic", "multiplicative", seed=21)
    idx = np.concatenate([np.arange(120, 140), np.arange(37, 102)[::-1]])
    sub = _run(gpu_ctx, _take(fb, idx), fut[idx], np.zeros(idx.size), cap[idx], "logistic", "multiplicative", seed=21)
    assert np.array_equal(sub.trend_lower, full.trend_lower[idx]) and np.array_equal(sub.trend_upper, full.trend_upper[idx])
    assert np.array_equal(sub.components, full.components[:, idx])


def test_device_entry_point_matches_host(gpu_ctx):
    import torch
    rng = np.random.RandomState(9)
    frs, fut = [], []
    for mask in (7, 4, 0):
        p, _ = _prep(mask, "linear", "multiplicative")
        frs.append(_model(p, rng))
        fut.append(_future(p, 40))
    fb = _batch(frs, batched.make_options(growth="linear"))
    fut = np.stack(fut)
    opts = batched.make_options(growth="linear")
    host = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(3), np.ones(3), seed=4, components=True)
    dev = torch.device("cuda", gpu_ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    dfb = batched.FittedBatch(t(fb.params), t(fb.tchange), t(fb.meta_i32), t(fb.meta_i64), t(fb.meta_f64), fb.smax, fb.kmax)
    got = batched.predict_batch_device(gpu_ctx, opts, dfb, t(fut), t(np.zeros(3)), t(np.ones(3)), seed=4, components=True)
    for a in ("yhat", "yhat_lower", "yhat_upper", "components", "trend_lower", "trend_upper"):
        assert np.array_equal(getattr(got, a).cpu().numpy(), getattr(host, a)), a
    # trend bounds without intervals are refused
    with pytest.raises(L.Pb200Error, match="trend bounds"):
        L.check(L.load().pb200_predict_components_host(
            gpu_ctx.handle, ctypes.byref(opts), fb.params.ctypes.data, fb.tchange.ctypes.data,
            fb.meta_i32.ctypes.data, fb.meta_i64.ctypes.data, fb.meta_f64.ctypes.data, 3, fut.ctypes.data, 40,
            np.zeros(3).ctypes.data, np.ones(3).ctypes.data, 0, host.yhat.ctypes.data, None, None,
            host.yhat_int.ctypes.data, host.components.ctypes.data, host.trend_lower.ctypes.data,
            host.trend_upper.ctypes.data), "pb200_predict_components_host")


# ---------------------------------------------------------------------------------------------------------------
# the scorer job
# ---------------------------------------------------------------------------------------------------------------
def _check_job_frame(out, table, periods, intervals):
    fitted, last_ds, info = model_record.decode(table["model"])
    mask = np.repeat(fitted.meta_i32[:, 3], periods)
    ok = np.repeat(fitted.meta_i32[:, 4] >= 0, periods)
    mask = mask[ok]
    for c, bit in SEAS.items():
        assert np.array_equal(out[c].is_valid().to_numpy(zero_copy_only=False), (mask & bit) != 0), c
    tr = out["trend"].to_numpy()
    mt = out["multiplicative_terms"].to_numpy()
    at = out["additive_terms"].to_numpy()
    assert np.all(np.isfinite(tr)) and (np.all(at == 0.0) if info["multiplicative"] else np.all(mt == 0.0))
    if intervals:
        assert np.all(out["trend_lower"].to_numpy() <= out["trend_upper"].to_numpy())


def test_scorer_job_components_on_the_golden_fixture(tmp_path, model_input_dir):
    models = str(tmp_path / "models")
    ProphetModeler.model(None, {"io": {"input": model_input_dir, "models": models},
                                "model": {"floor": 0, "cap_multiplier": 1.1}})
    sc = {"io": {"models": models, "forecasts": str(tmp_path / "fc")},
          "forecast": {"periods": 40, "frequency": "15min", "components": True, "intervals": True, "seed": 3}}
    scorer = ps.ProphetScorer(sc)
    mdf = scorer.read_model_dataframe(None)
    out = mdf.groupby("series_id", "dim_id").apply(ps.forecast_time_series(sc)).table
    assert out.column_names == ["series_id", "dim_id", "ds", "yhat", "yhat_lower", "yhat_upper",
                                *ps.COMPONENT_COLUMNS, "trend_lower", "trend_upper"]
    assert out.num_rows == 80
    _check_job_frame(out, mdf.table, 40, True)
    # the plain columns are those of a run without components
    plain = dict(sc, forecast={k: v for k, v in sc["forecast"].items() if k != "components"})
    ref = mdf.groupby("series_id", "dim_id").apply(ps.forecast_time_series(plain)).table
    assert out.select(ref.column_names).equals(ref)
    ps.ProphetScorer.score(None, sc)
    csv = pads.dataset(sc["io"]["forecasts"], format="csv").to_table()
    assert csv.column_names == ["created_timestamp", "series_id", "dim_id", "forecast_date", "forecast_timestamp",
                                "forecast_quantity", "yhat_lower", "yhat_upper", *ps.COMPONENT_COLUMNS,
                                "trend_lower", "trend_upper"]
    assert csv.num_rows == 80
    assert np.allclose(np.sort(csv["trend"].to_numpy()), np.sort(out["trend"].to_numpy()), rtol=1e-12)


def test_scorer_job_components_on_a_synth_tree(tmp_path):
    b = synth.config3(n=4)
    root = tmp_path / "in"
    for i in range(b.n):
        d = root / f"series_id={200 + i}"
        d.mkdir(parents=True)
        a, e = b.offsets[i], b.offsets[i + 1]
        ts = b.ds[a:e].astype("datetime64[ns]").astype("datetime64[s]")
        (d / "part.csv").write_text("".join(f"2,{str(x).replace('T', ' ')},{int(q)}\n" for x, q in zip(ts, b.y[a:e])))
    models = str(tmp_path / "models")
    ProphetModeler.model(None, {"io": {"input": str(root), "models": models}, "model": {"floor": 0, "cap_multiplier": 1.1}})
    sc = {"io": {"models": models, "forecasts": str(tmp_path / "fc")},
          "forecast": {"periods": 96, "frequency": "15min", "components": True}}
    mdf = ps.ProphetScorer(sc).read_model_dataframe(None)
    out = mdf.groupby("series_id", "dim_id").apply(ps.forecast_time_series(sc)).table
    assert out.column_names == ["series_id", "dim_id", "ds", "yhat", *ps.COMPONENT_COLUMNS]
    assert out.num_rows == 4 * 96
    _check_job_frame(out, mdf.table, 96, False)
    ps.ProphetScorer.score(None, sc)
    csv = pads.dataset(sc["io"]["forecasts"], format="csv").to_table()
    assert csv.column_names[-6:] == list(ps.COMPONENT_COLUMNS) and csv.num_rows == 4 * 96


def test_scorer_components_rank_rows_match_single_rank_run(gpu_ctx, monkeypatch):
    rng = np.random.RandomState(9)
    frs, fut = [], []
    for i in range(40):
        p, _ = _prep([6, 2, 0][i % 3], "logistic", "multiplicative")
        frs.append(_model(p, rng))
    opts = batched.make_options()
    fb = _batch(frs, opts)
    n = fb.n
    last = np.array([int(fr.prep.ds_sorted[-1]) for fr in frs], np.int64)
    tbl = pa.table({"series_id": pa.array(np.arange(n, dtype=np.int32)), "dim_id": pa.array(np.ones(n, np.int32)),
                    "floor": pa.array(np.zeros(n, np.float32)),
                    "cap": pa.array(np.array([fr.prep.cap_value for fr in frs], np.float32)),
                    "model": model_record.encode(fb, last, opts)})
    op = ps.forecast_time_series({"forecast": {"periods": 9, "frequency": "h", "intervals": True, "components": True,
                                               "seed": 5}})
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    full = op.apply_batched(tbl, ["series_id", "dim_id"]).to_pandas()
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "1")
    part = op.apply_batched(tbl, ["series_id", "dim_id"]).to_pandas()
    assert 0 < len(part) < len(full) and part["series_id"].min() > 0
    ref = full[full["series_id"].isin(part["series_id"].unique())].reset_index(drop=True)
    assert ref.equals(part.reset_index(drop=True))
    assert part["yearly"].isna().all() and part["daily"].notna().any() and part["trend_lower"].notna().all()
