"""The in-sample predict, its outlier flags and the refit without them (DESIGN §16) on the GPU (run with -m gpu on an
H100).

* pb200_predict_history_*: yhat and the bounds of every row bit-identical to pb200_predict_device on the model's history
  padded to the batch's longest by its last timestamp (both growths x both modes, masks 0-7, regular and irregular grids
  with a duplicate timestamp, lengths 2 ... 8000 mixed, sample counts, widths and seeds, a failed model);
* against the oracle: bounds within 1e-9 y_scale of mc_stream, yhat within 1e-12 y_scale of prophet_oracle;
* a model's rows do not depend on the batch; refusals launch nothing;
* the flags, kept counts and compacted batch equal numpy's for int32, float32 and float64 y;
* the modeler job with io.fitted and with insample.refit, against plain modeler runs.
"""
import ctypes as C
import os
import sys

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import insample_oracle as io_  # noqa: E402
from oracle import mc_stream as mcs  # noqa: E402
from oracle import prophet_oracle as po  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched  # noqa: E402

pytestmark = pytest.mark.gpu

H_NS = 3600 * 10**9
DAY = 24 * H_NS
MIN15 = 15 * 60 * 10**9
MC_TOL = 1e-9
PRED_TOL = 1e-12
E_ARG, E_UNSUPPORTED = -1, -4
LENGTHS = (2, 3, 15, 16, 17, 1023, 1024, 1025, 8000)
# (step, points, weekly switch) whose auto seasonalities give each mask
MASK_HIST = {7: (12 * H_NS, 1600, "auto"), 6: (H_NS, 720, "auto"), 5: (12 * H_NS, 1600, False), 4: (H_NS, 240, "auto"),
             3: (DAY, 801, "auto"), 2: (DAY, 60, "auto"), 1: (7 * DAY, 115, "auto"), 0: (MIN15, 96, "auto")}
_measured = {"mc": 0.0, "yhat": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print(f"\n[insample] max |bounds - mc_stream| / y_scale = {_measured['mc']:.3e}; "
          f"max |yhat - oracle| / y_scale = {_measured['yhat']:.3e}")


def _history(T, step, rng, irregular=False, dup=False, start="2021-03-01"):
    ds = np.datetime64(start, "ns").astype(np.int64) + step * np.arange(T, dtype=np.int64)
    if irregular and T > 2:
        ds[1:-1] += rng.randint(0, step // 2, T - 2)
    if dup and T > 3:
        ds[2] = ds[1]
    y = 100.0 + 20.0 * np.sin(np.arange(T) / 7.0) + np.arange(T) % 5
    return ds, y


def _fit_like(ds, y, growth, mode, rng, weekly="auto", sigma=0.03):
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, weekly_seasonality=weekly)
    p = po.prepare(ds, y, 0.0, 1.1 * y.max(), oopts)
    delta = 0.3 * rng.laplace(size=p.S) if p.n_changepoints_real else np.zeros(p.S)
    beta = 0.05 * rng.randn(p.K) if p.seasonalities else np.zeros(p.K)
    k, m = (rng.uniform(0.5, 2.0), rng.uniform(-0.3, 0.3)) if p.logistic else (rng.uniform(-0.5, 0.5), rng.uniform(0.3, 0.7))
    fr = po.FitResult(prep=p, k=k, m=m, delta=delta, sigma_obs=sigma, beta=beta, theta=None, neg_logp=0.0, iters=0,
                      n_evals=0, ret=0)
    return fr, oopts


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


def _mixed(growth, mode, seed=0, masks=True, lengths=True, failed=()):
    """Models on their own histories: one per seasonality mask, then one per length of LENGTHS on a 15-min grid,
    alternately regular and irregular, some with a duplicate timestamp."""
    rng = np.random.RandomState(seed)
    frs, hists, oo = [], [], []
    if masks:
        for mask, (step, T, weekly) in MASK_HIST.items():
            ds, y = _history(T, step, rng, irregular=mask in (5, 6))   # sub-daily steps: the jitter keeps the mask
            fr, oopts = _fit_like(ds, y, growth, mode, rng, weekly)
            assert sum(mcs._MASK_BIT[s.name] for s in fr.prep.seasonalities) == mask
            frs.append(fr); hists.append(ds); oo.append(oopts)
    if lengths:
        for j, T in enumerate(LENGTHS):
            ds, y = _history(T, MIN15, rng, irregular=j % 2 == 1, dup=j % 3 == 2)
            fr, oopts = _fit_like(ds, y, growth, mode, rng)
            frs.append(fr); hists.append(ds); oo.append(oopts)
    opts = batched.make_options(growth=growth, seasonality_mode=mode)
    status = np.zeros(len(frs), np.int32)
    status[list(failed)] = -1
    fb = _batch(frs, opts, status)
    offsets = np.concatenate(([0], np.cumsum([h.size for h in hists]))).astype(np.int64)
    floor = np.zeros(len(frs)) if growth == "linear" else rng.uniform(-5, 5, len(frs))
    cap = np.array([fr.prep.cap_value for fr in frs]) + floor
    return frs, oo, fb, hists, offsets, floor, cap


def _padded(hists):
    H = max(h.size for h in hists)
    return np.stack([np.concatenate((h, np.full(H - h.size, h[-1], np.int64))) for h in hists])


def _opts(growth, mode, n=1000, w=0.8):
    return batched.make_options(growth=growth, seasonality_mode=mode, uncertainty_samples=n, interval_width=w)


def _same_as_padded(ctx, opts, fb, hists, offsets, floor, cap, seed):
    hf = batched.predict_history_host(ctx, opts, fb, np.concatenate(hists), offsets, floor, cap, seed=seed)
    fc = batched.predict_batch_host(ctx, opts, fb, _padded(hists), floor, cap, seed=seed, intervals=True)
    for i, h in enumerate(hists):
        a, b = offsets[i], offsets[i + 1]
        assert hf.yhat[a:b].tobytes() == fc.yhat[i, :h.size].tobytes(), i
        assert hf.yhat_lower[a:b].tobytes() == fc.yhat_lower[i, :h.size].tobytes(), i
        assert hf.yhat_upper[a:b].tobytes() == fc.yhat_upper[i, :h.size].tobytes(), i
    return hf


# ---------------------------------------------------------------------------------------------------------------------
# 1. the ragged instances against pb200_predict_device on padded frames, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("logistic", "additive"),
                                         ("linear", "multiplicative"), ("linear", "additive")])
def test_ragged_is_the_padded_predict_bit_for_bit(gpu_ctx, growth, mode):
    frs, _, fb, hists, offsets, floor, cap = _mixed(growth, mode, seed=1, failed=(3, 12))
    hf = _same_as_padded(gpu_ctx, _opts(growth, mode), fb, hists, offsets, floor, cap, seed=5)
    for i in (3, 12):                                     # failed models: NaN rows
        a, b = offsets[i], offsets[i + 1]
        assert np.all(np.isnan(hf.yhat[a:b])) and np.all(np.isnan(hf.yhat_lower[a:b])) and np.all(np.isnan(hf.yhat_upper[a:b]))
    ok = np.ones(fb.n, bool)
    ok[[3, 12]] = False
    assert np.all(np.isfinite(hf.yhat[np.repeat(ok, np.diff(offsets))]))


@pytest.mark.parametrize("n,w", [(2, 0.8), (1000, 0.0), (1000, 0.5), (1000, 0.99), (1000, 1.0), (1024, 0.8)])
@pytest.mark.parametrize("seed", [0, 2**63 + 11])
def test_ragged_is_the_padded_predict_sample_counts_widths_seeds(gpu_ctx, n, w, seed):
    _, _, fb, hists, offsets, floor, cap = _mixed("logistic", "multiplicative", seed=2, masks=False)
    _same_as_padded(gpu_ctx, _opts("logistic", "multiplicative", n, w), fb, hists, offsets, floor, cap, seed)


def test_without_bounds_yhat_is_the_same(gpu_ctx):
    _, _, fb, hists, offsets, floor, cap = _mixed("linear", "additive", seed=3)
    ds = np.concatenate(hists)
    with_b = batched.predict_history_host(gpu_ctx, _opts("linear", "additive"), fb, ds, offsets, floor, cap, seed=1)
    no_b = batched.predict_history_host(gpu_ctx, _opts("linear", "additive"), fb, ds, offsets, floor, cap, seed=1,
                                        intervals=False)
    zero = batched.predict_history_host(gpu_ctx, _opts("linear", "additive", n=0), fb, ds, offsets, floor, cap)
    assert no_b.yhat_lower is None and zero.yhat_lower is None
    assert no_b.yhat.tobytes() == with_b.yhat.tobytes() == zero.yhat.tobytes()


def test_device_form_is_the_host_form(gpu_ctx):
    import torch
    _, _, fb, hists, offsets, floor, cap = _mixed("logistic", "additive", seed=4)
    ds = np.concatenate(hists)
    opts = _opts("logistic", "additive")
    ref = batched.predict_history_host(gpu_ctx, opts, fb, ds, offsets, floor, cap, seed=9)
    dfb = batched.FittedBatch(*(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in
                                (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64, fb.meta_f64)), fb.smax, fb.kmax)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    got = batched.predict_history_device(gpu_ctx, opts, dfb, cu(ds), offsets, cu(floor), cu(cap), seed=9)
    for x, y in ((got.yhat, ref.yhat), (got.yhat_lower, ref.yhat_lower), (got.yhat_upper, ref.yhat_upper)):
        assert x.cpu().numpy().tobytes() == y.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# 2. against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("linear", "additive")])
def test_against_the_oracle(gpu_ctx, growth, mode):
    frs, oo, fb, hists, offsets, floor, cap = _mixed(growth, mode, seed=5)
    opts = _opts(growth, mode, 1000, 0.9)
    hf = batched.predict_history_host(gpu_ctx, opts, fb, np.concatenate(hists), offsets, floor, cap, seed=17)
    for i, fr in enumerate(frs):
        a, b = offsets[i], offsets[i + 1]
        ys = fr.prep.y_scale
        yh = io_.yhat(fr, hists[i], floor[i], cap[i], oo[i])
        err = np.max(np.abs(hf.yhat[a:b] - yh) / (ys * np.maximum(1.0, np.abs(yh) / ys)))
        assert err <= PRED_TOL, (i, err)
        _measured["yhat"] = max(_measured["yhat"], err)
        lo, hi = io_.bounds(fb, i, hists[i], floor[i], cap[i], growth == "logistic", mode == "multiplicative", 1000, 0.9, 17)
        err = max(np.max(np.abs(hf.yhat_lower[a:b] - lo)), np.max(np.abs(hf.yhat_upper[a:b] - hi))) / ys
        assert err <= MC_TOL, (i, err)
        _measured["mc"] = max(_measured["mc"], err)


# ---------------------------------------------------------------------------------------------------------------------
# 3. batch independence, refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_rows_do_not_depend_on_the_batch(gpu_ctx):
    _, _, fb, hists, offsets, floor, cap = _mixed("logistic", "multiplicative", seed=6)
    opts = _opts("logistic", "multiplicative")
    full = batched.predict_history_host(gpu_ctx, opts, fb, np.concatenate(hists), offsets, floor, cap, seed=21)
    rng = np.random.RandomState(0)
    idx = rng.permutation(fb.n)
    sh = [hists[i] for i in idx]
    soff = np.concatenate(([0], np.cumsum([h.size for h in sh]))).astype(np.int64)
    sub = batched.predict_history_host(gpu_ctx, opts, _take(fb, idx), np.concatenate(sh), soff, floor[idx], cap[idx],
                                       seed=21)
    for j, i in enumerate(idx):
        for f in ("yhat", "yhat_lower", "yhat_upper"):
            assert getattr(sub, f)[soff[j]:soff[j + 1]].tobytes() == getattr(full, f)[offsets[i]:offsets[i + 1]].tobytes()
    for i in (0, 11, fb.n - 1):                           # alone: one model, one CTA
        one = batched.predict_history_host(gpu_ctx, opts, _take(fb, [i]), hists[i], [0, hists[i].size], floor[[i]],
                                           cap[[i]], seed=21)
        assert one.yhat_upper.tobytes() == full.yhat_upper[offsets[i]:offsets[i + 1]].tobytes()
        assert one.yhat.tobytes() == full.yhat[offsets[i]:offsets[i + 1]].tobytes()


def test_refusals_launch_nothing(gpu_ctx):
    _, _, fb, hists, offsets, floor, cap = _mixed("linear", "additive", seed=7, masks=False)
    ds = np.concatenate(hists)
    before = gpu_ctx.launch_count
    for opts in (_opts("linear", "additive", n=1), _opts("linear", "additive", n=1025)):
        with pytest.raises(L.Pb200Error, match=f"\\({E_UNSUPPORTED}\\)"):
            batched.predict_history_host(gpu_ctx, opts, fb, ds, offsets, floor, cap)
    for w in (-0.1, 1.5, float("nan")):
        with pytest.raises(L.Pb200Error, match=f"\\({E_ARG}\\)"):
            batched.predict_history_host(gpu_ctx, _opts("linear", "additive", w=w), fb, ds, offsets, floor, cap)
    bad = offsets.copy()
    bad[3] = bad[4] + 1
    with pytest.raises(L.Pb200Error, match="monotone"):
        batched.predict_history_host(gpu_ctx, _opts("linear", "additive"), fb, ds, bad, floor, cap)
    assert gpu_ctx.launch_count == before
    empty = batched.predict_history_host(gpu_ctx, _opts("linear", "additive"), _take(fb, []), ds[:0], [0], floor[:0],
                                         cap[:0])
    assert empty.yhat.size == 0


# ---------------------------------------------------------------------------------------------------------------------
# 4. flags and compaction
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ydt", ["int32", "float32", "float64"])
def test_flags_and_compaction_are_numpys(gpu_ctx, ydt):
    import torch
    rng = np.random.RandomState({"int32": 1, "float32": 2, "float64": 3}[ydt])
    # more series than the grid's warps (grid-stride loop), lengths across the 32-row steps, empty series
    T = rng.choice([0, 1, 2, 31, 32, 33, 64, 95, 200], size=20000)
    T[:9] = [0, 1, 2, 31, 32, 33, 64, 1000, 3000]
    off = np.concatenate(([0], np.cumsum(T))).astype(np.int64)
    R = int(off[-1])
    ds = np.sort(rng.randint(0, 10**15, R)).astype(np.int64)
    y = (rng.randn(R) * 10).astype(ydt) if ydt != "int32" else rng.randint(-50, 50, R).astype(np.int32)
    lo = rng.randn(R) * 8 - 3
    hi = lo + rng.uniform(0, 16, R)
    lo[rng.rand(R) < 0.05] = np.nan
    hi[rng.rand(R) < 0.05] = np.nan
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    got = batched.outliers_device(gpu_ctx, cu(ds), cu(y), off, cu(lo), cu(hi))
    flag = io_.flags(y, lo, hi)
    kept, noff, ds_k, y_k = io_.kept_batch(ds, y, off, flag)
    assert np.array_equal(got.flag.cpu().numpy(), flag.astype(np.uint8))
    assert np.array_equal(got.kept, kept) and np.array_equal(got.offsets, noff)
    assert got.ds.cpu().numpy().tobytes() == ds_k.tobytes()
    assert got.y.dtype == cu(y).dtype and got.y.cpu().numpy().tobytes() == y_k.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# 5 / 6. the modeler job
# ---------------------------------------------------------------------------------------------------------------------
def _write_tree(root, dim, ds, y):
    d = os.path.join(root, "series_id=751")
    os.makedirs(d, exist_ok=True)
    ts = np.asarray(ds, np.int64).astype("datetime64[ns]").astype("datetime64[s]")
    lines = [f"{int(a)},{str(t).replace('T', ' ')},{int(q)}" for a, t, q in zip(dim, ts, y)]
    with open(os.path.join(d, "part.csv"), "w") as f:
        f.write("\n".join(lines) + "\n")
    return root


def _spiky_input(seed=0, n_groups=6):
    """Daily demand over 120 days per group, with a spike of 20x the level at known rows."""
    rng = np.random.RandomState(seed)
    dims, dss, ys, spikes = [], [], [], []
    t0 = np.datetime64("2022-01-01", "ns").astype(np.int64)
    for g in range(n_groups):
        T = 120 + 7 * g
        ds = t0 + DAY * np.arange(T, dtype=np.int64)
        y = np.maximum(1, 50 + 10 * np.sin(2 * np.pi * np.arange(T) / 7) + rng.randn(T) * 2).astype(np.int64)
        for r in rng.choice(np.arange(10, T - 10), 3, replace=False):
            y[r] = 1000
            spikes.append((g, int(ds[r])))
        dims.append(np.full(T, g)); dss.append(ds); ys.append(y)
    return np.concatenate(dims), np.concatenate(dss), np.concatenate(ys), spikes


def _model(cfg):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    ProphetModeler.model(None, cfg)
    return pq.read_table(cfg["io"]["models"]).sort_by([("series_id", "ascending"), ("dim_id", "ascending")])


def _check_fitted(fr, dim, ds, y):
    assert fr.schema.names == ["series_id", "dim_id", "ds", "y", "yhat", "yhat_lower", "yhat_upper", "outlier"]
    assert [str(t) for t in fr.schema.types] == ["int32", "int32", "timestamp[ns]", "int32", "double", "double",
                                                 "double", "bool"]
    assert fr.num_rows == dim.size
    order = np.lexsort((ds, dim))
    assert np.array_equal(fr["dim_id"].to_numpy(), dim[order])
    assert np.array_equal(fr["ds"].to_numpy().astype(np.int64), ds[order])
    assert np.array_equal(fr["y"].to_numpy(), y[order].astype(np.int32))
    lo, hi, yh = (fr[c].to_numpy() for c in ("yhat_lower", "yhat_upper", "yhat"))
    assert np.all(np.isfinite(yh)) and np.all(lo <= hi)
    assert np.array_equal(fr["outlier"].to_numpy(), (y[order] < lo) | (y[order] > hi))


def test_job_fitted_frame_on_the_golden_fixture(tmp_path, golden_input, capsys):
    gi = golden_input
    inp = _write_tree(str(tmp_path / "in"), gi["dim_id"], gi["ds_ns"], gi["y"])
    model = {"floor": 0, "cap_multiplier": 1.1}
    plain = _model({"io": {"input": inp, "models": str(tmp_path / "plain")}, "model": model})
    cfg = {"io": {"input": inp, "models": str(tmp_path / "m"), "fitted": str(tmp_path / "fitted")}, "model": model,
           "insample": {"interval_width": 0.99}}
    got = _model(cfg)
    assert got.equals(plain)                              # the models table is the same bytes
    fr = pq.read_table(cfg["io"]["fitted"])
    _check_fitted(fr, gi["dim_id"], gi["ds_ns"], gi["y"])
    out = capsys.readouterr().out
    assert f"In-sample: {gi['y'].size} rows predicted, {int(fr['outlier'].to_numpy().sum())} flagged" in out


def test_job_flags_every_injected_spike(tmp_path, capsys):
    dim, ds, y, spikes = _spiky_input()
    inp = _write_tree(str(tmp_path / "in"), dim, ds, y)
    model = {"floor": 0, "cap_multiplier": 1.1}
    plain = _model({"io": {"input": inp, "models": str(tmp_path / "plain")}, "model": model})
    cfg = {"io": {"input": inp, "models": str(tmp_path / "m"), "fitted": str(tmp_path / "fitted")}, "model": model,
           "insample": {"interval_width": 0.99, "seed": 3}}
    assert _model(cfg).equals(plain)
    fr = pq.read_table(cfg["io"]["fitted"])
    _check_fitted(fr, dim, ds, y)
    key = {(int(d), int(t)): bool(o) for d, t, o in zip(fr["dim_id"].to_numpy(), fr["ds"].to_numpy().astype(np.int64),
                                                          fr["outlier"].to_numpy())}
    assert all(key[s] for s in spikes), [s for s in spikes if not key[s]]
    other = sum(o for k, o in key.items() if k not in set(spikes))
    with capsys.disabled():
        print(f"\n[insample] spikes flagged {len(spikes)}/{len(spikes)}; other rows flagged {other}/{len(key) - len(spikes)}")


@pytest.mark.parametrize("warm", [False, True])
def test_refit_is_a_plain_run_without_the_flagged_rows(tmp_path, warm):
    dim, ds, y, _ = _spiky_input(seed=1)
    inp = _write_tree(str(tmp_path / "in"), dim, ds, y)
    model = {"floor": 0, "cap_multiplier": 1.1}
    io = {}
    if warm:                                              # a previous table fitted on the first 100 days
        short = ds < ds.min() + 100 * DAY
        old = str(tmp_path / "old")
        _model({"io": {"input": _write_tree(str(tmp_path / "short"), dim[short], ds[short], y[short]), "models": old},
                "model": model})
        io["warm_start"] = old
    cfg = {"io": {"input": inp, "models": str(tmp_path / "m"), "fitted": str(tmp_path / "fitted"), **io},
           "model": model, "insample": {"interval_width": 0.95, "refit": True}}
    got = _model(cfg)
    fr = pq.read_table(cfg["io"]["fitted"])
    flagged = fr["outlier"].to_numpy()
    assert flagged.sum() >= 18                            # the premise: every spike and then some
    keep = {(int(d), int(t)) for d, t, o in zip(fr["dim_id"].to_numpy(), fr["ds"].to_numpy().astype(np.int64), flagged)
            if not o}
    sel = np.array([(int(d), int(t)) in keep for d, t in zip(dim, ds)])
    ref_in = _write_tree(str(tmp_path / "in_filtered"), dim[sel], ds[sel], y[sel])
    ref = _model({"io": {"input": ref_in, "models": str(tmp_path / "ref"), **io}, "model": model})
    assert got.equals(ref)
    # io.fitted describes the first fit: refit: false gives the same frame
    cfg2 = {"io": {"input": inp, "models": str(tmp_path / "m2"), "fitted": str(tmp_path / "fitted2"), **io},
            "model": model, "insample": {"interval_width": 0.95}}
    _model(cfg2)
    assert pq.read_table(cfg2["io"]["fitted"]).equals(fr)


def test_refit_of_a_group_left_with_one_row_raises(tmp_path):
    from time_series_spark_b200.jobs.prophet_modeler import ProphetModeler
    dim, ds, y, _ = _spiky_input(seed=2, n_groups=2)
    inp = _write_tree(str(tmp_path / "in"), dim, ds, y)
    # width 0: the interval is one point, so (nearly) every row of every group is flagged
    cfg = {"io": {"input": inp, "models": str(tmp_path / "m")}, "model": {"floor": 0, "cap_multiplier": 1.1},
           "insample": {"interval_width": 0.0, "uncertainty_samples": 2, "refit": True}}
    with pytest.raises(ValueError, match=r"Dataframe has less than 2 non-NaN rows\. \(first offender: series_id 751"):
        ProphetModeler.model(None, cfg)
