"""Seasonality tables on the GPU (DESIGN §18): custom seasonalities and built-in Fourier orders through the table fit
class and the predict / interval kernels, held to the numpy oracle (tests/seasonality_table.py) with DESIGN §1's
tolerances: objective 1e-10 relative, gradient 1e-8 relative to max(1, |g|), predict at given parameters 1e-12 of
y_scale, fitted objective median 5e-4 / max 5e-3 relative."""
import numpy as np
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

import seasonality_table as st

pytestmark = pytest.mark.gpu

DAY = 86400 * 10**9
MONTHLY = dict(name="monthly", period=30.5, fourier_order=5)
TABLES = {
    "yearly20": (dict(yearly_seasonality=20), []),
    "monthly": (dict(), [MONTHLY]),
    "quarterly": (dict(), [dict(name="quarterly", period=91.3125, fourier_order=2, prior_scale=0.1)]),
    "k64": (dict(yearly_seasonality=20, weekly_seasonality=6, daily_seasonality=False),
            [dict(name="monthly", period=30.5, fourier_order=6)]),
    "p96": (dict(yearly_seasonality=20, weekly_seasonality=6, daily_seasonality=False, n_changepoints=29),
            [dict(name="monthly", period=30.5, fourier_order=6)]),
}


def _batch(grid, n=6, seed=5):
    b = synth.config2(n=n, T=800, seed=seed)
    if grid == "regular":
        return b
    # irregular: drop a fifth of the rows at random and repeat one timestamp per series
    rng = np.random.RandomState(seed)
    ds, y, off = [], [], [0]
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        keep = np.sort(rng.choice(e - a, size=(4 * (e - a)) // 5, replace=False))
        d, v = b.ds[a:e][keep], b.y[a:e][keep]
        j = len(d) // 2
        d = np.insert(d, j, d[j])
        v = np.insert(v, j, v[j])
        ds.append(d)
        y.append(v)
        off.append(off[-1] + len(d))
    return synth.RaggedBatch(b.series_id, b.dim_id, np.array(off, np.int64), np.concatenate(ds),
                             np.concatenate(y).astype(b.y.dtype))


def _opts(table, growth, mode):
    kw, custom = TABLES[table]
    kw = dict(kw)
    ncp = kw.pop("n_changepoints", 25)
    opts = batched.make_table_options(seasonalities=custom, growth=growth, seasonality_mode=mode, n_changepoints=ncp,
                                      **kw)
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, n_changepoints=ncp)
    builtin = {k.replace("_seasonality", ""): v for k, v in kw.items()}
    return opts, oopts, builtin, custom


def _prep(b, i, oopts, builtin, custom):
    a, e = b.offsets[i], b.offsets[i + 1]
    y = b.y[a:e].astype(np.float64)
    return st.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts, builtin, custom)


CELLS = [(t, g, m, grid) for t in TABLES for g in ("linear", "logistic") for m in ("additive", "multiplicative")
         for grid in ("regular", "irregular")]


@pytest.mark.parametrize("cell", CELLS, ids=lambda c: "-".join(c))
def test_objective_and_gradient_match_oracle(gpu_ctx, cell):
    table, growth, mode, grid = cell
    opts, oopts, builtin, custom = _opts(table, growth, mode)
    b = _batch(grid)
    lay = L.get_layout(opts)
    rng = np.random.RandomState(3)
    rows, preps = [], []
    for i in range(b.n):
        p, seas = _prep(b, i, oopts, builtin, custom)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.zeros(lay.pstride)
        row[:th.size] = th
        rows.append(row)
        preps.append((p, th, seas))
    f, g, mi = batched.objective_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, np.array(rows))
    for i, (p, th, seas) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(th, p)
        assert err == 0 and mi[i, 4] == 0
        assert (mi[i, 0], mi[i, 1]) == (p.T, p.S)
        assert bin(int(mi[i, 3])).count("1") == len(seas)
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (cell, i, f[i], fo)
        gd = np.max(np.abs(g[i, :th.size] - go)) / max(1.0, np.max(np.abs(go)))
        assert gd <= 1e-8, (cell, i, gd)
    if table == "p96":
        assert max(p.S + p.K + 3 for p, _, _ in preps) == 96


@pytest.mark.parametrize("cell", CELLS,
                         ids=lambda c: "-".join(c))
def test_fit_trajectory_end_point_and_predict_match_oracle(gpu_ctx, cell):
    table, growth, mode, grid = cell
    opts, oopts, builtin, custom = _opts(table, growth, mode)
    b = _batch(grid, n=4)
    fb, trace = batched.fit_batch_trace_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=512)
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], 60, DAY)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, intervals=False)
    relf = []
    for i in range(b.n):
        p, seas = _prep(b, i, oopts, builtin, custom)
        tr = []
        fr = st.fit(p, oopts, trace=tr)
        assert fb.meta_i32[i, 4] >= 0 and fr.ret >= 0, (cell, i, fb.meta_i32[i, 4], fr.ret)
        S, K = p.S, p.K
        assert np.array_equal(fb.tchange[i, :S], p.t_change)
        # the first six trajectory rows, to test_gpu_optimiser.py's rules: one row per iteration, the same evaluation
        # counts, f to 1e-11 and alpha to 1e-7 relative
        g, o = trace[i], np.array(tr)
        n_gpu = int(fb.meta_i32[i, 5])
        assert n_gpu >= 1 and g[min(n_gpu, 512) - 1, 0] == min(n_gpu, 512)
        head = min(n_gpu, len(o), 6)
        assert np.array_equal(g[:head, 3], o[:head, 3]), (cell, i, g[:head, 3], o[:head, 3])
        assert np.all(np.abs(g[:head, 1] - o[:head, 1]) <= 1e-11 * np.maximum(1.0, np.abs(o[:head, 1]))), (cell, i)
        assert np.all(np.abs(g[:head, 2] - o[:head, 2]) <= 1e-7 * np.abs(o[:head, 2])), (cell, i)
        relf.append(abs(fb.meta_f64[i, 3] - fr.neg_logp) / abs(fr.neg_logp))
        # predict at the GPU's own parameters against the oracle's predict
        got = po.FitResult(prep=p, k=fb.params[i, 0], m=fb.params[i, 1], delta=fb.params[i, 3:3 + S],
                           sigma_obs=fb.params[i, 2], beta=fb.params[i, 3 + fb.smax:3 + fb.smax + K], theta=None,
                           neg_logp=0.0, iters=0, n_evals=0, ret=0)
        pr = po.predict(got, fut[i], 0.0, cap32[i], oopts)
        assert np.max(np.abs(pr["yhat"] - fc.yhat[i])) <= 1e-12 * p.y_scale, cell
    relf = np.array(relf)
    assert np.median(relf) <= 5e-4 and relf.max() <= 5e-3, relf


def test_table_count_and_mask_bits(gpu_ctx):
    opts, _, _, _ = _opts("monthly", "logistic", "multiplicative")
    b = _batch("regular", n=3)
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    n = np.zeros(1, np.int64)
    L.check(L.load().pb200_last_fit_table_count(gpu_ctx.handle, n.ctypes.data), "pb200_last_fit_table_count")
    assert n[0] == 3
    # table monthly, yearly, weekly, daily: 800 daily points (2.2 years) turn yearly and weekly on, daily off
    assert np.all(fb.meta_i32[:, 3] == 0b0111)
    counts = np.zeros(32, np.int32)
    L.check(L.load().pb200_last_fit_variant_counts(gpu_ctx.handle, counts.ctypes.data), "variant counts")
    assert counts.sum() == 0


def test_builtins_as_a_table_reach_the_default_optimum(gpu_ctx):
    """weekly2 (7, 3) and daily2 (1, 4) with the built-ins off is config #3's model through the table kernel."""
    b = synth.config3(n=8, T=1440)
    dflt = batched.make_options()
    tab = batched.make_table_options(yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False,
                                     seasonalities=[dict(name="weekly2", period=7.0, fourier_order=3),
                                                    dict(name="daily2", period=1.0, fourier_order=4)])
    f0 = batched.fit_batch_host(gpu_ctx, dflt, b.ds, b.y, b.offsets, 0.0, 1.1)
    f1 = batched.fit_batch_host(gpu_ctx, tab, b.ds, b.y, b.offsets, 0.0, 1.1)
    assert np.all(f0.meta_i32[:, 3] == 6) and np.all(f1.meta_i32[:, 3] == 3)
    rel = np.abs(f1.meta_f64[:, 3] - f0.meta_f64[:, 3]) / np.abs(f0.meta_f64[:, 3])
    assert np.median(rel) <= 5e-4 and rel.max() <= 5e-3, rel
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], 96, 15 * 60 * 10**9)
    cap32 = f0.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    p0 = batched.predict_batch_host(gpu_ctx, dflt, f0, fut, np.zeros(b.n), cap32, intervals=False)
    p1 = batched.predict_batch_host(gpu_ctx, tab, f1, fut, np.zeros(b.n), cap32, intervals=False)
    r = np.max(np.abs(p1.yhat - p0.yhat), axis=1) / f0.meta_f64[:, 0]
    assert np.median(r) <= 2e-3 and r.max() <= 3e-2, r


def test_series_alone_and_in_a_batch_give_the_same_bits(gpu_ctx):
    opts, _, _, _ = _opts("quarterly", "linear", "additive")
    b = _batch("irregular", n=5)
    fa = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    for i in (0, 3):
        a, e = b.offsets[i], b.offsets[i + 1]
        one = batched.fit_batch_host(gpu_ctx, opts, b.ds[a:e], b.y[a:e], np.array([0, e - a]), 0.0, 1.1)
        assert np.array_equal(one.params[0], fa.params[i]) and np.array_equal(one.meta_f64[0], fa.meta_f64[i])


@pytest.mark.parametrize("table, growth, mode", [("monthly", "logistic", "multiplicative"), ("k64", "linear", "additive"),
                                                 ("quarterly", "logistic", "additive")])
def test_bounds_and_window_sums_match_mc_stream(gpu_ctx, monkeypatch, table, growth, mode):
    """The MC kernels read the table betas at their packed columns: bounds within 1e-9 y_scale of oracle/mc_stream.py's
    draws (its seasonal term evaluated on the table), daily... weekly window totals and their bounds likewise."""
    from oracle import mc_stream
    opts, _, _, _ = _opts(table, growth, mode)
    b = _batch("regular", n=3)
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], 28, DAY)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fl = np.zeros(b.n)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, fl, cap32, seed=7, intervals=True)
    fs, ws = batched.predict_sums_host(gpu_ctx, opts, fb, fut, fl, cap32, 7 * DAY, seed=7, intervals=True)
    assert np.array_equal(fs.yhat, fc.yhat)
    monkeypatch.setattr(mc_stream, "_seasonal", st.table_seasonal(opts, "numpy"))
    for i in range(b.n):
        ys = fb.meta_f64[i, 0]
        d = mc_stream.draws(fb, i, fut[i], 0.0, cap32[i], growth == "logistic", mode == "multiplicative",
                            opts.uncertainty_samples, 7)
        lo, hi = mc_stream.bounds(d, opts.interval_width)
        assert np.max(np.abs(lo - fc.yhat_lower[i])) <= 1e-9 * ys, (table, i)
        assert np.max(np.abs(hi - fc.yhat_upper[i])) <= 1e-9 * ys, (table, i)
        w = (fut[i] // (7 * DAY))
        nw = int(ws.n_windows[i])
        assert nw == len(np.unique(w))
        for j, wv in enumerate(np.unique(w)):
            rows = np.flatnonzero(w == wv)
            s_ = 0.0
            for r in rows:
                s_ = s_ + fc.yhat[i, r]
            assert ws.yhat_sum[i, j] == s_
            slo, shi = mc_stream.bounds(d[rows].sum(axis=0)[None, :], opts.interval_width)
            assert abs(slo[0] - ws.lower[i, j]) <= 1e-9 * ys * rows.size, (table, i, j)
            assert abs(shi[0] - ws.upper[i, j]) <= 1e-9 * ys * rows.size, (table, i, j)


@pytest.mark.parametrize("mode", ["additive", "multiplicative"])
def test_component_planes(gpu_ctx, mode):
    """One plane per custom entry after the six, in table order; a custom 'weekly' fills the weekly plane; the entry
    planes add up, in table order, to the seasonal term exactly; each is the oracle's X_c beta_c."""
    custom = [MONTHLY, dict(name="weekly", period=7.0, fourier_order=5),
              dict(name="quarterly", period=91.3125, fourier_order=2, prior_scale=0.1)]
    opts = batched.make_table_options(seasonalities=custom, seasonality_mode=mode, daily_seasonality=False)
    assert batched.component_names(opts) == L.COMPONENTS + ("monthly", "quarterly")
    oopts = po.ProphetOptions(seasonality_mode=mode)
    b = _batch("irregular", n=3)
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], 40, DAY)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fl = np.zeros(b.n)
    plain = batched.predict_batch_host(gpu_ctx, opts, fb, fut, fl, cap32, intervals=False)
    fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, fl, cap32, intervals=False, components=True)
    assert np.array_equal(fc.yhat, plain.yhat)
    assert np.all(fc.component("daily") == 0.0)
    # table order: monthly, weekly (custom), quarterly, yearly (800 daily points: yearly on)
    order = ["monthly", "weekly", "quarterly", "yearly"]
    mult = mode == "multiplicative"
    total = fc.component("multiplicative_terms" if mult else "additive_terms")
    for i in range(b.n):
        assert fb.meta_i32[i, 3] == 0b1111
        ys = fb.meta_f64[i, 0]
        acc = np.zeros(fut.shape[1])
        for name in order:
            acc = acc + (fc.component(name)[i] if mult else fc.component(name)[i] / ys)
        ref = total[i] if mult else total[i] / ys
        assert np.max(np.abs(acc - ref)) <= (0.0 if mult else 1e-13 * max(1.0, np.max(np.abs(ref)))), (mode, i)
        p, seas = _prep(b, i, oopts, {}, custom)
        assert [s_[0] for s_ in seas] == order
        X, _, _, _ = po.seasonal_features(fut[i], p.seasonalities, oopts)
        beta, col = fb.params[i, 3 + fb.smax:], 0
        for name, _, o, _ in seas:
            want = X[:, col:col + 2 * o] @ beta[col:col + 2 * o] * (1.0 if mult else ys)
            col += 2 * o
            assert np.max(np.abs(fc.component(name)[i] - want)) <= 1e-12 * (1.0 if mult else ys), (mode, name, i)


@pytest.mark.parametrize("table", ["yearly20", "p96"])
@pytest.mark.parametrize("growth", ["linear", "logistic"])
def test_newton_steps_match_oracle(gpu_ctx, table, growth):
    """PB200_ALG_NEWTON on table models after 1, 2, 3 and 5 iterations against numpy's stan_newton on the table's
    objective: status 60, the same iteration and evaluation counts (every step-halving decision), changepoints exact,
    the objective within 1e-8 of its size, and theta within 1e-6 of its size: test_newton_steps.py holds wide models to
    ten times the two CPU oracles' disagreement, ~1e-8 .. 1e-7 there, and the finite-difference Hessian of a P = 96
    table model is as ill-conditioned along the Laplace prior's kinks (measured 4.9e-7 of the size after 5 steps)."""
    for k in (1, 2, 3, 5):
        kw, custom = TABLES[table]
        kw = dict(kw)
        ncp = kw.pop("n_changepoints", 25)
        mode = "multiplicative" if growth == "logistic" else "additive"
        opts = batched.make_table_options(seasonalities=custom, growth=growth, seasonality_mode=mode,
                                          n_changepoints=ncp, max_iter=k, algorithm="Newton", **kw)
        oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, n_changepoints=ncp, max_iter=k)
        builtin = {q.replace("_seasonality", ""): v for q, v in kw.items()}
        b = synth.config2(n=2, T=150, seed=11)
        fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
        for i in range(b.n):
            p, _ = _prep(b, i, oopts, builtin, custom)
            th, f, it, ret, ne = po.stan_newton(lambda x: po.neg_logp_grad(x, p), po.initial_theta(p), oopts)
            P = p.S + p.K + 3
            if table == "p96":
                assert P == 96
            mi = fb.meta_i32[i]
            assert mi[4] == 60 == ret and (mi[5], mi[6]) == (it, ne), (table, k, i, mi, it, ne)
            assert np.array_equal(fb.tchange[i, :p.S], p.t_change)
            got = np.concatenate((fb.params[i, :2], fb.params[i, 3:3 + p.S], [np.log(fb.params[i, 2])],
                                  fb.params[i, 3 + fb.smax:3 + fb.smax + p.K]))
            ref = th.copy()
            if p.n_changepoints_real == 0:
                ref[0] += ref[2]
                ref[2] = 0.0
            assert np.max(np.abs(got - ref)) <= 1e-6 * max(1.0, np.max(np.abs(ref))), (table, k, i)
            assert abs(fb.meta_f64[i, 3] - f) <= 1e-8 * max(1.0, abs(f)), (table, k, i)


def test_refusals(gpu_ctx):
    """Per-series prior scales (the tuner) and warm starts are not built for table models: refused before any launch."""
    opts, _, _, _ = _opts("monthly", "logistic", "multiplicative")
    b = _batch("regular", n=2)
    fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    with pytest.raises(Exception, match="seasonality table"):
        batched.fit_batch_warm_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, init=fb)
    with pytest.raises(Exception, match="seasonality table"):
        batched.fit_batch_warm_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, init=None,
                                    prior=np.tile([0.05, 10.0], (b.n, 1)))
    assert L.get_layout(opts).kmax == 44
