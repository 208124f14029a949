"""GPU tests of per-series prior scales (pb200_fit_prior_device) and the tuning job built on them (batched.tune_device,
jobs/prophet_tuner.py; DESIGN §10).  Contexts are pinned to the kernel families of test_gpu_scheduling.py, so that a
batch and its sub-batches run the same kernel and must give the same bits."""
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.dataset as pads
import pyarrow.parquet as pq
import pytest

from oracle import c_oracle
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 86400 * 10**9
HORIZON, PERIOD, INITIAL = D, D // 2, 3 * D
CAPM = 1.1
FIELDS = ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")

FAMILIES = {
    "g8": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 8, "PB200_PLAIN_GROUP": 1},
    "g16": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 16, "PB200_PLAIN_GROUP": 1},
    "tab32": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 0},
    "rot32": {"PB200_LC0_MAX": 1 << 30, "PB200_NO_TAB": 1},
    "default": {},
}

# four interleaved pairs; the first is the options' own
PAIRS = [(0.05, 10.0), (0.001, 0.01), (0.5, 10.0), (0.1, 1.0)]


def _ctx_with_env(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return L.Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def ctx_for():
    cache = {}

    def get(family):
        if family not in cache:
            cache[family] = _ctx_with_env(**FAMILIES[family])
        return cache[family]

    yield get
    for c in cache.values():
        c.close()


def _join(parts):
    offs = np.concatenate(([0], np.cumsum([p.offsets[-1] for p in parts]))).astype(np.int64)
    o = np.concatenate([p.offsets[:-1] + s for p, s in zip(parts, offs[:-1])] + [offs[-1:]]).astype(np.int64)
    n = o.size - 1
    return synth.RaggedBatch(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), o,
                             np.concatenate([p.ds for p in parts]), np.concatenate([p.y for p in parts]))


def _lsfail_batch():
    return _join([synth.config4(n=500_000, lo=i, hi=i + 1) for i in synth.CONFIG4_LSFAIL_IDS] + [synth.config4(n=23)])


def _tight_opts():
    o = batched.make_options(algorithm="LBFGS", max_iter=20000)
    o.tol_rel_grad = o.tol_rel_obj = o.tol_grad = o.tol_param = 0.0
    o.tol_obj = 1e-13
    o.algorithm = L.ALG_LBFGS_NEWTON
    return o


# name -> (family, batch, options)
CASES = {
    "g8": ("g8", lambda: synth.config3(n=24), batched.make_options),
    "g16": ("g16", lambda: synth.config3(n=24), batched.make_options),
    "tab32": ("tab32", lambda: synth.config3(n=12), batched.make_options),
    "rot32": ("rot32", lambda: synth.config3(n=12), batched.make_options),
    "default_4_warps": ("default", lambda: synth.config3(n=12), batched.make_options),
    "plain_g8": ("g8", lambda: synth.config4(n=32), batched.make_options),
    "newton": ("default", lambda: synth.config4(n=12), lambda: batched.make_options(algorithm="Newton")),
    "lbfgs_newton_retry": ("default", _lsfail_batch, _tight_opts),
}


def _fit(ctx, opts, b, prior=None):
    import torch
    ds, y = torch.from_numpy(b.ds).cuda(), torch.from_numpy(b.y).cuda()
    pr = torch.from_numpy(np.ascontiguousarray(prior, dtype=np.float64)).cuda() if prior is not None else None
    return batched.fit_batch_device(ctx, opts, ds, y, b.offsets, 0.0, CAPM, prior=pr).to_host()


def _with_prior(opts, pair):
    o = L.Options.from_buffer_copy(opts)
    o.changepoint_prior_scale, o.seasonality_prior_scale = pair
    return o


def _rows_equal(fa, ia, fb, ib):
    return all(getattr(fa, k)[ia].tobytes() == getattr(fb, k)[ib].tobytes() for k in FIELDS)


@pytest.mark.parametrize("case", list(CASES))
def test_per_series_priors_equal_uniform_fits(ctx_for, case):
    family, mk, mko = CASES[case]
    ctx, b, opts = ctx_for(family), mk(), mko()
    which = np.arange(b.n) % len(PAIRS)
    prior = np.array([PAIRS[j] for j in which])
    mixed = _fit(ctx, opts, b, prior)
    st = mixed.meta_i32[:, 4]
    assert np.all(st >= 0), (case, st)
    if case == "newton":
        assert np.all(st == L.ST_NEWTON)
    if case == "lbfgs_newton_retry":
        assert st[0] == L.ST_NEWTON                       # the retry series (options' pair) still takes the Newton path
    for j, pair in enumerate(PAIRS):
        sel = np.flatnonzero(which == j)
        sub = _join([b.take(int(i), int(i) + 1) for i in sel])
        uni = _fit(ctx, _with_prior(opts, pair), sub)
        for k, i in enumerate(sel):
            assert _rows_equal(mixed, i, uni, k), (case, pair, int(i))
    same = _fit(ctx, opts, b, np.tile(PAIRS[0], (b.n, 1)))
    none = _fit(ctx, opts, b)
    for k in FIELDS:
        assert getattr(same, k).tobytes() == getattr(none, k).tobytes(), (case, k)


def test_bad_priors_fail_only_their_series(ctx_for):
    ctx = ctx_for("g8")
    b = synth.config3(n=12)
    opts = batched.make_options()
    prior = np.tile(PAIRS[0], (b.n, 1))
    bad = {1: (0.0, 10.0), 4: (0.05, -1.0), 7: (np.nan, 10.0), 10: (0.05, np.inf)}
    for i, p in bad.items():
        prior[i] = p
    got = _fit(ctx, opts, b, prior)
    ref = _fit(ctx, opts, b)
    for i in range(b.n):
        if i in bad:
            assert got.meta_i32[i, 4] == L.ST_BAD_PRIOR, (i, got.meta_i32[i])
        else:
            assert _rows_equal(got, i, ref, i), i


@pytest.mark.parametrize("cp", [0.001, 0.5])
@pytest.mark.parametrize("sp", [0.01, 10.0])
def test_prior_scales_against_the_oracles(ctx_for, cp, sp):
    ctx = ctx_for("g8")
    b = synth.config3(n=4)
    opts = batched.make_options(changepoint_prior_scale=cp, seasonality_prior_scale=sp)
    oopts = po.ProphetOptions(changepoint_prior_scale=cp, seasonality_prior_scale=sp)
    copts = c_oracle.options()
    copts.tau, copts.seas_prior = cp, sp
    lay = L.get_layout(opts)
    rng = np.random.RandomState(5)
    rows, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * CAPM, oopts)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        rows.append(row)
        preps.append((p, th))
    f, g, mi = batched.objective_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, CAPM, np.array(rows))
    assert ctx.last_fit_variant_counts()[3, 6] == b.n
    for i, (p, th) in enumerate(preps):
        a, e = b.offsets[i], b.offsets[i + 1]
        err, fo, go = po.neg_logp_grad(th, p)
        cerr, fc, gc = c_oracle.objective(b.ds[a:e], b.y[a:e], 0.0, float(b.y[a:e].max()) * CAPM, th, copts)
        assert err == 0 and cerr == 0 and mi[i, 4] == 0
        for fr, gr in ((fo, go), (fc, gc)):
            assert abs(f[i] - fr) <= 1e-10 * max(1.0, abs(fr)), (cp, sp, i, f[i], fr)
            assert np.max(np.abs(g[i, :th.size] - gr)) <= 1e-8 * max(1.0, np.max(np.abs(gr))), (cp, sp, i)
    # the first accepted iterations against the oracle (DESIGN §1's trajectory tolerances)
    fb, tr = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, CAPM, trace_cap=8)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        trace = []
        po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=po.ProphetOptions(changepoint_prior_scale=cp,
               seasonality_prior_scale=sp, max_iter=6), algorithm="LBFGS", trace=trace)
        o = np.array(trace).reshape(-1, 4)
        head = min(int(fb.meta_i32[i, 5]), len(o), 6)
        assert head >= 1
        gt = tr[i, :head]
        assert np.array_equal(gt[:, 0], np.arange(1, head + 1)) and np.array_equal(gt[:, 3], o[:head, 3]), (cp, sp, i)
        assert np.all(np.abs(gt[:, 1] - o[:head, 1]) <= 1e-11 * np.maximum(1.0, np.abs(o[:head, 1]))), (cp, sp, i)
        assert np.all(np.abs(gt[:, 2] - o[:head, 2]) <= 1e-7 * np.abs(o[:head, 2])), (cp, sp, i)


# ---------------------------------------------------------------------------------------------------------------------
# the grid backtest and the selection
# ---------------------------------------------------------------------------------------------------------------------
GRID = [(0.001, 0.01), (0.001, 10.0), (0.5, 0.01), (0.5, 10.0)]


def _device(b):
    import torch
    return torch.from_numpy(b.ds).cuda(), torch.from_numpy(b.y.astype(np.int32)).cuda()


def _cap(b):
    import torch
    return torch.tensor([float(b.y[a:e].max()) * CAPM for a, e in zip(b.offsets[:-1], b.offsets[1:])], dtype=torch.float64).cuda()


def _cv(ctx, opts, b, **kw):
    ds, y = _device(b)
    return batched.cross_validation_device(ctx, opts, ds, y, b.offsets, 0.0, _cap(b), HORIZON, PERIOD, INITIAL,
                                           rolling_window=1.0, **kw)


def _tune(ctx, b, grid=GRID, metric="rmse", budget=None):
    ds, y = _device(b)
    return batched.tune_device(ctx, batched.make_options(), ds, y, b.offsets, 0.0, CAPM, HORIZON, PERIOD, INITIAL, grid,
                               metric=metric, _row_budget=budget)


def test_grid_scores_equal_uniform_backtests(ctx_for):
    ctx = ctx_for("g8")
    b = synth.config3(n=5)
    opts = batched.make_options()
    g = len(GRID)
    grid_cv = _cv(ctx, opts, b, grid=GRID, keep_fits=True)
    tuned = _tune(ctx, b)
    assert grid_cv.metrics["series"].tolist() == list(range(b.n * g))          # one score per (series, grid point)
    for j, pair in enumerate(GRID):
        uni = _cv(ctx, _with_prior(opts, pair), b, keep_fits=True)
        for s in range(b.n):
            v = s * g + j
            pv, pu = np.flatnonzero(grid_cv.pair_series == v), np.flatnonzero(uni.pair_series == s)
            assert pv.size == pu.size > 0
            assert grid_cv.pair_cutoff[pv].tobytes() == uni.pair_cutoff[pu].tobytes()
            assert grid_cv.pair_status[pv].tobytes() == uni.pair_status[pu].tobytes()
            for k in FIELDS:
                assert getattr(grid_cv.fitted, k)[pv].tobytes() == getattr(uni.fitted, k)[pu].tobytes(), (pair, s, k)
            rv, ru = grid_cv.row_series == v, uni.row_series == s
            for k in ("ds", "cutoff", "y", "yhat"):
                assert getattr(grid_cv, k)[rv].tobytes() == getattr(uni, k)[ru].tobytes(), (pair, s, k)
            mv, mu = grid_cv.metrics["series"] == v, uni.metrics["series"] == s
            for k in ("horizon", "mse", "rmse", "mae", "mape"):
                assert grid_cv.metrics[k][mv].tobytes() == uni.metrics[k][mu].tobytes(), (pair, s, k)
            assert tuned.scores[s, j].tobytes() == uni.metrics["rmse"][mu].tobytes()


def test_selection_tie_rule_and_fallback(ctx_for):
    ctx = ctx_for("g8")
    b = synth.config3(n=4)
    y = b.y.copy()
    y[b.offsets[2] + 600] = 0                                  # a zero in series 2's held-out rows: its mape is not finite
    b = synth.RaggedBatch(b.series_id, b.dim_id, b.offsets, b.ds, y)
    grid = [(0.5, 10.0), (0.001, 0.01), (0.5, 10.0), (0.01, 1.0)]   # point 2 duplicates point 0
    t = _tune(ctx, b, grid=grid)
    assert t.scores[:, 0].tobytes() == t.scores[:, 2].tobytes()
    assert t.eligible.all()
    want = np.array([min(range(len(grid)), key=lambda j: (t.scores[s, j], j)) for s in range(b.n)])
    assert t.chosen.tolist() == want.tolist() and not np.any(t.chosen == 2)
    assert np.array_equal(t.prior, np.array(grid)[t.chosen])
    m = _tune(ctx, b, grid=grid, metric="mape")
    assert not m.eligible[2].any() and m.chosen[2] == -1
    assert m.eligible[[0, 1, 3]].all() and np.all(m.chosen[[0, 1, 3]] >= 0)
    opts = batched.make_options()
    assert tuple(m.prior[2]) == (opts.changepoint_prior_scale, opts.seasonality_prior_scale)
    f = m.fitted.to_host()
    ref = _fit(ctx, opts, _join([b.take(2, 3)]))
    assert _rows_equal(f, 2, ref, 0)


def _view(t, s):
    f = t.fitted.to_host()
    return (t.scores[s].tobytes(), t.eligible[s].tobytes(), int(t.chosen[s]), t.prior[s].tobytes(),
            tuple(getattr(f, k)[s].tobytes() for k in FIELDS))


def test_tuning_independent_of_batch_and_chunks(ctx_for):
    ctx = ctx_for("g8")
    b = synth.config3(n=6)
    full = _tune(ctx, b)
    tiny = _tune(ctx, b, budget=1)
    pick = [4, 1, 5, 0]
    sub = _tune(ctx, _join([b.take(i, i + 1) for i in pick]))
    for s in range(b.n):
        assert _view(full, s) == _view(tiny, s), s
    for j, s in enumerate(pick):
        assert _view(full, s) == _view(sub, j), (s, j)


# ---------------------------------------------------------------------------------------------------------------------
# the job
# ---------------------------------------------------------------------------------------------------------------------
def _synth_table(b, sid0=100, dim=3):
    return pa.table({"series_id": pa.array(np.repeat(np.arange(b.n) + sid0, np.diff(b.offsets)), pa.int32()),
                     "dim_id": pa.array(np.full(int(b.offsets[-1]), dim), pa.int32()),
                     "ds": pa.array(b.ds, pa.timestamp("ns")), "y": pa.array(b.y.astype(np.int32), pa.int32())})


def _tune_cfg(tmp_path, inp=None, **backtest):
    cfg = {"io": {"models": str(tmp_path / "models"), "tuning": str(tmp_path / "tuning")},
           "model": {"floor": 0, "cap_multiplier": 1.1},
           "backtest": backtest or {"horizon": "1 days", "period": "12 hours", "initial": "3 days"},
           "tune": {"changepoint_prior_scale": [0.001, 0.5], "seasonality_prior_scale": [0.01, 10.0]}}
    if inp:
        cfg["io"]["input"] = inp
    return cfg


def test_tuned_models_equal_modeler_runs(ctx_for, tmp_path, monkeypatch):
    from time_series_spark_b200.jobs import prophet_modeler as pm
    from time_series_spark_b200.jobs.prophet_tuner import ProphetTuner
    monkeypatch.setitem(pm._contexts, 0, ctx_for("g8"))          # both jobs on the pinned family
    b = synth.config3(n=6)
    cfg = _tune_cfg(tmp_path)
    models, tuning = ProphetTuner(cfg).tune(_synth_table(b))
    assert models.schema == pm.MODEL_OUTPUT_SCHEMA and models.num_rows == b.n
    assert tuning.num_rows == b.n * 4 and tuning["selected"].to_pylist().count(True) == b.n
    chosen = tuning.filter(tuning["selected"])
    for sid, cp, sp in zip(chosen["series_id"].to_pylist(), chosen["changepoint_prior_scale"].to_pylist(),
                           chosen["seasonality_prior_scale"].to_pylist()):
        i = sid - 100
        mcfg = {"model": {"floor": 0, "cap_multiplier": 1.1, "changepoint_prior_scale": cp, "seasonality_prior_scale": sp}}
        one = pm.model_time_series(mcfg).apply_batched(_synth_table(b.take(i, i + 1), sid0=sid), ["series_id", "dim_id"])
        row = models.filter(pc.equal(models["series_id"], sid))
        assert row.num_rows == 1 and one.num_rows == 1
        for col in models.schema.names:
            assert row[col].to_pylist() == one[col].to_pylist(), (sid, col)


def test_job_end_to_end_on_golden_fixture_and_synth_tree(tmp_path, model_input_dir):
    from time_series_spark_b200.jobs.prophet_tuner import ProphetTuner
    cfg = _tune_cfg(tmp_path / "golden", model_input_dir, horizon="30 days", period="15 days", initial="180 days")
    ProphetTuner.run(None, cfg)
    m = pq.read_table(cfg["io"]["models"])
    t = pq.read_table(cfg["io"]["tuning"])
    assert m.column_names == ["series_id", "dim_id", "floor", "cap", "model"] and m.num_rows == 2
    assert t.column_names == ["series_id", "dim_id", "changepoint_prior_scale", "seasonality_prior_scale", "rmse", "selected"]
    assert set(t["series_id"].to_pylist()) == {751} and t["selected"].to_pylist().count(True) == 2
    # a hive tree of synth series through the drivers: the tuner's models table straight into the scorer
    b = synth.config3(n=3)
    inp = tmp_path / "input"
    for i in range(b.n):
        d = inp / f"series_id={200 + i}"
        d.mkdir(parents=True)
        a, e = b.offsets[i], b.offsets[i + 1]
        ts = b.ds[a:e].astype("datetime64[ns]").astype("datetime64[s]")
        (d / "part.csv").write_text("".join(f"7,{str(x).replace('T', ' ')},{int(q)}\n" for x, q in zip(ts, b.y[a:e])))
    import yaml
    cfg = _tune_cfg(tmp_path / "synth", str(inp))
    cfg["io"]["forecasts"] = str(tmp_path / "synth" / "forecasts")
    cfg["forecast"] = {"periods": 12, "frequency": "15min"}
    path = tmp_path / "cfg.yaml"
    path.write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=ROOT)
    for drv in ("tuner_driver", "scorer_driver"):
        r = subprocess.run([sys.executable, "-m", f"time_series_spark_b200.{drv}", str(path)], cwd=ROOT, env=env,
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, (drv, r.stdout[-2000:], r.stderr[-2000:])
    m = pq.read_table(cfg["io"]["models"])
    assert sorted(m["series_id"].to_pylist()) == [200, 201, 202]
    out = pads.dataset(cfg["io"]["forecasts"], format="csv").to_table()
    assert out.num_rows == b.n * 12
