"""The seasonality-table fit class and its predict / MC paths held to the oracle where tables go past the built-ins
(DESIGN §18): sub-daily periods and high orders, lengths around the warp, a year of 15-minute data, P = 96, a table
entry switched off in the middle of the table, K differing between the series of one call, and warps that fit series
after series in one persistent queue.

The table fit kernel builds harmonic h of every seasonality from one staged base angle by the three-term recurrence, so
its objective is fbprophet's on the "exact" columns of tests/seasonality_table.py, sin / cos(h fl(fl(2 pi) t / p)), not
on numpy's, whose arguments are rounded per harmonic (over 1e-9 off at harmonic 32 of a 6-hour period).  Per cell and
seasonality mode:

  * pb200_last_fit_table_count() puts every series in the table class;
  * T, S, the table mask and the changepoints (exactly) are the oracle's;
  * objective and gradient at random points near initial_theta within 1e-10 / 1e-8 relative of the "exact" oracle, and
    the objective no further from the "numpy" one (fbprophet's) than the exact columns are, plus 1e-10 of its size;
  * the first six L-BFGS iterations on the "exact" oracle: evaluation counts identical, alpha_k within 1e-7, f_k within
    1e-11 over the first three and 1e-9 up to the sixth, status and iteration count the oracle's.

Beside the cells: the Newton run step by step, a batch of every shape fitted on one and on three CTAs against each
series alone, predict (both sincos_reduced bands and its library fall-back) and the component planes against the
"numpy" oracle, and quantiles, calendar-month sums and in-sample intervals with outlier flags against their oracles with
the table's seasonal term.  The recipes are checked without a GPU in tests/test_seasonalities_config.py.
"""
import dataclasses
import os
import sys
from dataclasses import dataclass

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import fit_oracle as fo  # noqa: E402
import seasonality_table as st  # noqa: E402
import test_kernel_instances as ki  # noqa: E402
from oracle import prophet_oracle as po  # noqa: E402
from time_series_spark_b200 import _lib as L  # noqa: E402
from time_series_spark_b200 import batched, synth  # noqa: E402

NS_MIN, NS_DAY = ki.NS_MIN, ki.NS_DAY
MIN15 = 15 * NS_MIN
MODES = ("additive", "multiplicative")
OFF = dict(yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False)
MONTHLY = dict(name="monthly", period=30.5, fourier_order=5)

# ---------------------------------------------------------------------------------------------------------------------
# the cells: (built-in switches, custom entries), growth, and the data
# ---------------------------------------------------------------------------------------------------------------------
TABLES = {
    # yearly off: 20 daily harmonics on top of the auto yearly (10) and weekly (3) would be K = 66
    "daily20": (dict(yearly_seasonality=False, daily_seasonality=20), []),
    "h12": (OFF, [dict(name="h12", period=0.5, fourier_order=32)]),                        # K = 64
    "q6h": (OFF, [dict(name="q6h", period=0.25, fourier_order=32)]),                       # K = 64, P = 96 at 29 cps
    "hourly": (dict(), [dict(name="hourly", period=1.0 / 24.0, fourier_order=4)]),
    "gap": (dict(), [MONTHLY]),                 # monthly, yearly, weekly, daily
}


@dataclass(frozen=True)
class Cell:
    table: str
    growth: str
    ncp: int
    masks: tuple         # the table mask each series must get
    regular: tuple       # per series
    lengths: tuple       # per series
    step: int = None     # the regular series' step


def irregular15(T, span_steps, seed):
    """T timestamps on a 15-minute grid of span_steps steps from START, the first and last slot kept, about a fifth of
    the others dropped at random and one timestamp repeated (a zero gap): the smallest non-zero step stays 15 minutes."""
    rng = np.random.default_rng([29, seed])
    inner = np.sort(rng.choice(np.arange(1, span_steps), size=T - 3, replace=False))
    idx = np.concatenate(([0], inner, [span_steps]))
    j = idx.size // 2
    idx = np.insert(idx, j, idx[j])
    return ki.START + seed * 37 * NS_MIN + MIN15 * idx


def _cells():
    gap_T = ki._lengths(2, True, 32)
    return {
        "daily20": Cell("daily20", "linear", 25, (0b10,) * 5, (True,) * 5, ki.BASE_LENGTHS[32], MIN15),
        "h12": Cell("h12", "logistic", 25, (0b1,), (True,), (ki.LONG_TAB[1],), ki.LONG_TAB[0]),
        "q6h_p96": Cell("q6h", "linear", 29, (0b1,) * 3, (False,) * 3, (40, 101, 960)),
        "hourly": Cell("hourly", "logistic", 25, (0b1101,) * 2, (False,) * 2, (2304, 2100)),
        "gap": Cell("gap", "linear", 25, (0b0101,) * 7, (True,) * 5 + (False,) * 2, gap_T + (45, 60)),
        "mixed": Cell("gap", "logistic", 25, (0b0101, 0b0111) * 2, (True, True, False, False), (60, 800, 61, 801)),
    }


CELLS = _cells()


def cell_series(name):
    """[(ds, y int32)] of the cell, in its order."""
    c = CELLS[name]
    out = []
    for i, (T, reg) in enumerate(zip(c.lengths, c.regular)):
        if name == "daily20":
            s = ki._series(0, T, True, i, MIN15)
        elif name == "h12":
            ds = ki.START + MIN15 * np.arange(T, dtype=np.int64)
            s = (ds, ki._y(ds, 20))
        elif name == "q6h_p96":
            ds = irregular15(T, (5 * T) // 4, 50 + i)
            s = (ds, ki._y(ds, 50 + i))
        elif name == "hourly":
            ds = irregular15(T, 30 * 96, 60 + i)
            s = (ds, ki._y(ds, 60 + i))
        elif name == "gap":
            s = ki._series(2, T, reg, 70 + i)
        else:                                   # mixed: 60-day and 800-day daily series interleaved
            s = ki._series(2 if c.masks[i] == 0b0101 else 3, T, reg, 80 + i)
        assert s is not None, (name, i, T)
        out.append(s)
    return out


def options(table, growth, mode, ncp, **kw):
    """(library options, oracle options, built-in switches by name, custom entries) of a table."""
    bkw, custom = TABLES[table]
    opts = batched.make_table_options(seasonalities=custom, growth=growth, seasonality_mode=mode, n_changepoints=ncp,
                                      **bkw, **kw)
    oopts = po.ProphetOptions(growth=growth, seasonality_mode=mode, n_changepoints=ncp)
    return opts, oopts, {k.replace("_seasonality", ""): v for k, v in bkw.items()}, custom


def prep(ds, y, oopts, builtin, custom, columns):
    y = np.asarray(y, np.float64)
    return st.prepare(ds, y, 0.0, y.max() * 1.1, oopts, builtin, custom, columns)


def entries(table):
    bkw, custom = TABLES[table]
    return st.table_entries({k.replace("_seasonality", ""): v for k, v in bkw.items()}, custom)


def _ragged(series, ydtype=np.int32):
    b = ki._ragged(series)
    y = b.y.astype(np.float64)
    if ydtype != np.int32:
        y = y + 0.25                          # a fractional part the integer path cannot carry
    return synth.RaggedBatch(b.series_id, b.dim_id, b.offsets, b.ds, y.astype(ydtype))


def table_count(ctx):
    n = np.zeros(1, np.int64)
    L.check(L.load().pb200_last_fit_table_count(ctx.handle, n.ctypes.data), "pb200_last_fit_table_count")
    return int(n[0])


# the (cell, mode, n_changepoints, y dtype) runs of the matrix: every cell in both modes, and the options on the gap and
# daily20 (T = 101) data
OPTION_RUNS = [(ncp, dt) for ncp in (0, 1) for dt in ("int32", "float32", "float64")]
RUNS = [(name, mode, CELLS[name].ncp, "int32") for name in CELLS for mode in MODES]
RUNS += [(name, mode, ncp, dt) for name in ("gap", "daily20_101") for mode in MODES for ncp, dt in OPTION_RUNS]


def run_series(name):
    """The cell behind a run name and its series: daily20_101 is the daily20 cell's T = 101 series alone."""
    if name == "daily20_101":
        s = cell_series("daily20")
        return CELLS["daily20"], [s[ki.BASE_LENGTHS[32].index(101)]]
    return CELLS[name], cell_series(name)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
_measured = {"f": 0.0, "g": 0.0, "f_np": 0.0, "f_np_exact": 0.0, "f_k": 0.0, "f_k6": 0.0, "alpha_k": 0.0,
             "newton_f": 0.0, "newton_theta": 0.0, "pred": 0.0, "comp": 0.0, "q": 0.0, "sum": 0.0, "mc": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviations():
    yield
    m = _measured
    if any(m.values()):
        print(f"\n[table instances] max deviation: objective {m['f']:.3e} (1e-10) and gradient {m['g']:.3e} (1e-8) "
              f"relative to the exact oracle; |f - f_numpy| {m['f_np']:.3e} where |f_exact - f_numpy| is up to "
              f"{m['f_np_exact']:.3e} (relative); f_k rows 1-3 {m['f_k']:.3e} (1e-11), rows 4-6 {m['f_k6']:.3e} "
              f"(1e-9), "
              f"alpha_k {m['alpha_k']:.3e} (1e-7); Newton objective {m['newton_f']:.3e} (1e-8), theta "
              f"{m['newton_theta']:.3e} (1e-6); predict {m['pred']:.3e} and components {m['comp']:.3e} of y_scale "
              f"(1e-12); quantiles {m['q']:.3e}, month sums {m['sum']:.3e}, in-sample bounds {m['mc']:.3e} of y_scale "
              f"(1e-9)")


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode,ncp,ydt", RUNS, ids=lambda v: str(v))
def test_cell_matches_oracle(gpu_ctx, name, mode, ncp, ydt):
    cell, series = run_series(name)
    b = _ragged(series, getattr(np, ydt))
    opts, oopts, builtin, custom = options(cell.table, cell.growth, mode, ncp)
    ents = entries(cell.table)
    lay = L.get_layout(opts)
    rng = np.random.RandomState(11)
    rows, preps = [], []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        pe, seas = prep(b.ds[a:e], b.y[a:e], oopts, builtin, custom, "exact")
        pn, _ = prep(b.ds[a:e], b.y[a:e], oopts, builtin, custom, "numpy")
        th = po.initial_theta(pe) + 0.05 * rng.randn(pe.S + pe.K + 3)
        # past the series' own P the row is padding the kernel must not read: 0.5 there would enter as betas of
        # columns the series' mask does not have
        row = np.full(lay.pstride, 0.5)
        row[:th.size] = th
        rows.append(row)
        preps.append((pe, pn, th, st.table_mask(seas, ents)))
    f, g, mi = batched.objective_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, np.array(rows))
    assert table_count(gpu_ctx) == b.n
    what = (name, mode, ncp, ydt)
    for i, (pe, pn, th, mask) in enumerate(preps):
        _, fe, ge = po.neg_logp_grad(th, pe)
        _, fn, _ = po.neg_logp_grad(th, pn)
        assert mi[i, 4] == 0 and (mi[i, 0], mi[i, 1], mi[i, 3]) == (pe.T, pe.S, mask), (what, i, mi[i])
        sz = max(1.0, abs(fe))
        df = abs(f[i] - fe) / sz
        dg = np.max(np.abs(g[i, :th.size] - ge)) / max(1.0, np.max(np.abs(ge)))
        # fbprophet parity, derived from the oracle: the GPU may be no further from numpy's columns than the exact ones
        dn, dref = abs(f[i] - fn), abs(fe - fn)
        _measured["f"], _measured["g"] = max(_measured["f"], df), max(_measured["g"], dg)
        _measured["f_np"] = max(_measured["f_np"], dn / sz)
        _measured["f_np_exact"] = max(_measured["f_np_exact"], dref / sz)
        assert df <= 1e-10, (what, i, pe.T, f[i], fe)
        assert dg <= 1e-8, (what, i, pe.T, dg)
        assert dn <= dref + 1e-10 * max(1.0, abs(fn)), \
            (what, i, f"|f_gpu - f_numpy| = {dn:.3e}, |f_exact - f_numpy| = {dref:.3e}", f[i], fe, fn)
    # the first iterations of the fit, its status and iteration count
    o6, _, _, _ = options(cell.table, cell.growth, mode, ncp, max_iter=6, algorithm="LBFGS")
    o6_oracle = dataclasses.replace(oopts, max_iter=6)
    fb, tr = batched.fit_batch_trace_host(gpu_ctx, o6, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=8)
    assert table_count(gpu_ctx) == b.n
    for i, (pe, _, _, mask) in enumerate(preps):
        rr = []
        fr = st.fit(pe, o6_oracle, trace=rr)
        rr = np.array(rr).reshape(-1, 4)
        S = pe.S
        assert (fb.meta_i32[i, 0], fb.meta_i32[i, 1], fb.meta_i32[i, 3]) == (pe.T, S, mask), (what, i)
        assert np.array_equal(fb.tchange[i, :S], pe.t_change) and np.all(fb.tchange[i, S:] == 0.0), (what, i)
        n_gpu = int(fb.meta_i32[i, 5])
        fo.assert_trajectory_head(tr[i], n_gpu, rr, (what, i, pe.T), n_head=3)
        head = min(n_gpu, len(rr), 6)
        gk, ok = tr[i, :head], rr[:head]
        assert np.array_equal(gk[:, 0], ok[:, 0]) and np.array_equal(gk[:, 3], ok[:, 3]), (what, i, gk, ok)
        df = np.abs(gk[:, 1] - ok[:, 1]) / np.maximum(1.0, np.abs(ok[:, 1]))
        da = np.abs(gk[:, 2] - ok[:, 2]) / np.abs(ok[:, 2])
        _measured["f_k"] = max(_measured["f_k"], float(df[:3].max()))
        _measured["f_k6"] = max(_measured["f_k6"], float(df.max()))
        _measured["alpha_k"] = max(_measured["alpha_k"], float(da.max()))
        assert np.all(df <= 1e-9) and np.all(da <= 1e-7), (what, i, df, da)
        assert (fb.meta_i32[i, 4], n_gpu) == (fr.ret, fr.iters), (what, i, fb.meta_i32[i], fr.ret, fr.iters)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["q6h_p96", "gap"])
def test_newton_steps_match_oracle(gpu_ctx, name):
    """PB200_ALG_NEWTON after 1, 2, 3 and 5 iterations against stan_newton on the exact columns, at
    test_gpu_seasonalities.test_newton_steps_match_oracle's rules: status 60, iteration and evaluation counts equal,
    changepoints exact, the objective within 1e-8 and theta within 1e-6 of their size."""
    cell = CELLS[name]
    series = cell_series(name)[:3]
    b = _ragged(series)
    mode = "multiplicative" if cell.growth == "logistic" else "additive"
    for k in (1, 2, 3, 5):
        opts, oopts, builtin, custom = options(cell.table, cell.growth, mode, cell.ncp, max_iter=k, algorithm="Newton")
        oopts = dataclasses.replace(oopts, max_iter=k)
        fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
        for i in range(b.n):
            a, e = b.offsets[i], b.offsets[i + 1]
            p, _ = prep(b.ds[a:e], b.y[a:e], oopts, builtin, custom, "exact")
            th, f, it, ret, ne = po.stan_newton(lambda x: po.neg_logp_grad(x, p), po.initial_theta(p), oopts)
            mi = fb.meta_i32[i]
            assert mi[4] == 60 == ret and (mi[5], mi[6]) == (it, ne), (name, k, i, mi, it, ne)
            assert np.array_equal(fb.tchange[i, :p.S], p.t_change)
            got = np.concatenate((fb.params[i, :2], fb.params[i, 3:3 + p.S], [np.log(fb.params[i, 2])],
                                  fb.params[i, 3 + fb.smax:3 + fb.smax + p.K]))
            ref = th.copy()
            if p.n_changepoints_real == 0:
                ref[0] += ref[2]
                ref[2] = 0.0
            dt = np.max(np.abs(got - ref)) / max(1.0, np.max(np.abs(ref)))
            df = abs(fb.meta_f64[i, 3] - f) / max(1.0, abs(f))
            _measured["newton_theta"] = max(_measured["newton_theta"], dt)
            _measured["newton_f"] = max(_measured["newton_f"], df)
            assert dt <= 1e-6, (name, k, i, dt)
            assert df <= 1e-8, (name, k, i, df)
        if name == "q6h_p96":
            assert max(int(fb.meta_i32[i, 1]) for i in range(b.n)) + 64 + 3 == 96


def _reuse_series():
    """Series of every cell under the gap table, so that T, S, K and the mask rise and fall from one to the next."""
    d20, hr, gp, mx = cell_series("daily20"), cell_series("hourly"), cell_series("gap"), cell_series("mixed")
    return [gp[0], mx[1], d20[4], hr[0], gp[5], d20[0], mx[3], gp[2], hr[1], d20[3]]


REUSE_MASKS = (0b0101, 0b0111, 0b0001, 0b1101, 0b0101, 0b0001, 0b0111, 0b0101, 0b1101, 0b0001)


@pytest.mark.gpu
@pytest.mark.parametrize("grid_max", [1, 3])
def test_reused_slots_give_each_series_its_own_bits(grid_max):
    """One CTA (every series through one warp's queue) and three: params, changepoints, meta and the trajectory of each
    series byte-identical to the series fitted alone."""
    b = _ragged(_reuse_series())
    opts, _, _, _ = options("gap", "logistic", "multiplicative", 25)
    ctx = fo.ctx_with_env(PB200_FIT_GRID_MAX=grid_max)
    try:
        fb, tr = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=64)
        assert table_count(ctx) == b.n
        assert tuple(int(m) for m in fb.meta_i32[:, 3]) == REUSE_MASKS
        for i in range(b.n):
            a, e = b.offsets[i], b.offsets[i + 1]
            one, t1 = batched.fit_batch_trace_host(ctx, opts, b.ds[a:e], b.y[a:e], np.array([0, e - a]), 0.0, 1.1,
                                                   trace_cap=64)
            for x, y in ((one.params[0], fb.params[i]), (one.tchange[0], fb.tchange[i]),
                         (one.meta_i32[0], fb.meta_i32[i]), (one.meta_i64[0], fb.meta_i64[i]),
                         (one.meta_f64[0], fb.meta_f64[i]), (t1[0], tr[i])):
                assert x.tobytes() == y.tobytes(), (grid_max, i)
        print(f"\n[table instances] reused slots: statuses {fb.meta_i32[:, 4].tolist()}")
    finally:
        ctx.close()


PRED_CELLS = ("h12", "hourly", "q6h_p96", "gap")
PRED_STEP = {"h12": (MIN15, 192), "hourly": (MIN15, 192), "q6h_p96": (MIN15, 192), "gap": (NS_DAY, 90)}


def _fit_cell(ctx, name, mode, series=None, **kw):
    cell = CELLS[name]
    series = series if series is not None else cell_series(name)
    b = _ragged(series)
    opts, oopts, builtin, custom = options(cell.table, cell.growth, mode, cell.ncp, **kw)
    fb = batched.fit_batch_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    assert np.all(fb.meta_i32[:, 4] >= 0), fb.meta_i32[:, 4]
    return cell, b, fb, opts, oopts, builtin, custom


def _gpu_fit_result(fb, i, p):
    S, K = p.S, p.K
    return po.FitResult(prep=p, k=fb.params[i, 0], m=fb.params[i, 1], delta=fb.params[i, 3:3 + S],
                        sigma_obs=fb.params[i, 2], beta=fb.params[i, 3 + fb.smax:3 + fb.smax + K], theta=None,
                        neg_logp=0.0, iters=0, n_evals=0, ret=0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", PRED_CELLS)
@pytest.mark.parametrize("mode", MODES)
def test_predict_matches_numpy_oracle(gpu_ctx, name, mode):
    """predict_kernel<false>, <true> and the ragged in-sample predict at the GPU's parameters within 1e-12 y_scale of
    fbprophet's predict (numpy's arguments: these kernels reduce the same rounded doubles); the gap cell's component
    planes each the oracle's X_c beta_c, the planes of its switched-off entries 0."""
    cell, b, fb, opts, oopts, builtin, custom = _fit_cell(gpu_ctx, name, mode)
    step, H = PRED_STEP[name]
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], H, step)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fl = np.zeros(b.n)
    plain = batched.predict_batch_host(gpu_ctx, opts, fb, fut, fl, cap32, intervals=False)
    comp = batched.predict_batch_host(gpu_ctx, opts, fb, fut, fl, cap32, intervals=False, components=True)
    hist = batched.predict_history_host(gpu_ctx, opts, fb, b.ds, b.offsets, fb.meta_f64[:, 1], fb.meta_f64[:, 2],
                                        intervals=False)
    assert np.array_equal(plain.yhat, comp.yhat)
    ents = entries(cell.table)
    mult = mode == "multiplicative"
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        p, seas = prep(b.ds[a:e], b.y[a:e], oopts, builtin, custom, "numpy")
        ys = p.y_scale
        fr = _gpu_fit_result(fb, i, p)
        want = po.predict(fr, fut[i], 0.0, cap32[i], oopts)["yhat"]
        want_h = po.predict(fr, b.ds[a:e], fb.meta_f64[i, 1], fb.meta_f64[i, 2], oopts)["yhat"]
        for got, ref in ((plain.yhat[i], want), (comp.yhat[i], want), (hist.yhat[a:e], want_h)):
            d = np.max(np.abs(got - ref)) / ys
            _measured["pred"] = max(_measured["pred"], d)
            assert d <= 1e-12, (name, mode, i, d)
        if name != "gap":
            continue
        mask = int(fb.meta_i32[i, 3])
        assert mask == 0b0101
        beta, col = fb.params[i, 3 + fb.smax:], 0
        for j, (ename, per, o) in enumerate(ents):
            plane = comp.component(ename)[i]
            if not (mask >> j) & 1:
                assert np.all(plane == 0.0), (ename, i)
                continue
            X = st.fourier_columns(fut[i], per, o, "numpy")
            ref = X @ beta[col:col + 2 * o] * (1.0 if mult else ys)
            col += 2 * o
            d = np.max(np.abs(plane - ref)) / (1.0 if mult else ys)
            _measured["comp"] = max(_measured["comp"], d)
            assert d <= 1e-12, (mode, ename, i, d)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["gap", "mixed"])
def test_consumers_match_their_oracles(gpu_ctx, monkeypatch, name):
    """Quantiles, calendar-month sums and in-sample intervals with outlier flags on table models, against
    quantile_oracle, period_oracle and insample_oracle over oracle/mc_stream's draws with the table's seasonal term, at
    their own files' bounds (1e-9 y_scale)."""
    import torch

    import insample_oracle as io_
    import period_oracle as pdo
    import quantile_oracle as qo
    from oracle import mc_stream as mcs
    cell = CELLS[name]
    mode = "multiplicative" if cell.growth == "logistic" else "additive"
    n, width = 300, 0.8
    cell, b, fb, opts, oopts, builtin, custom = _fit_cell(gpu_ctx, name, mode, uncertainty_samples=n,
                                                          interval_width=width)
    monkeypatch.setattr(mcs, "_seasonal", st.table_seasonal(opts, "numpy"))
    logi, mult = cell.growth == "logistic", mode == "multiplicative"
    fut = batched.make_future(b.ds[b.offsets[1:] - 1], 75, NS_DAY)
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fl = np.zeros(b.n)
    levels = [0.1, 0.5, 0.9, 0.025, 0.975]
    fq = batched.predict_quantiles_host(gpu_ctx, opts, fb, fut, fl, cap32, levels, seed=5)
    _, months, shift = batched.period_rule("M")
    _, ws = batched.predict_period_sums_host(gpu_ctx, opts, fb, fut, fl, cap32, months, shift, seed=5)
    hf = batched.predict_history_host(gpu_ctx, opts, fb, b.ds, b.offsets, fb.meta_f64[:, 1], fb.meta_f64[:, 2],
                                      seed=17)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()          # noqa: E731
    out = batched.outliers_device(gpu_ctx, cu(b.ds), cu(b.y), b.offsets, cu(hf.yhat_lower), cu(hf.yhat_upper))
    flag_ref = []
    for i in range(b.n):
        ys = fb.meta_f64[i, 0]
        d = mcs.draws(fb, i, fut[i], 0.0, cap32[i], logi, mult, n, 5)
        err = np.max(np.abs(fq.quantiles[:, i] - qo.quantiles(d, 100.0 * np.asarray(levels)))) / ys
        _measured["q"] = max(_measured["q"], err)
        assert err <= 1e-9, (name, i, err)
        start, pts, lo, hi = pdo.period_sums(d, fut[i], "M", width)
        nw = start.size
        assert ws.n_windows[i] == nw and np.array_equal(ws.start[i, :nw], start), (name, i)
        assert np.array_equal(ws.points[i, :nw], pts), (name, i)
        err = max(np.max(np.abs(ws.lower[i, :nw] - lo) / pts), np.max(np.abs(ws.upper[i, :nw] - hi) / pts)) / ys
        _measured["sum"] = max(_measured["sum"], err)
        assert err <= 1e-9, (name, i, err)
        a, e = b.offsets[i], b.offsets[i + 1]
        lo, hi = io_.bounds(fb, i, b.ds[a:e], fb.meta_f64[i, 1], fb.meta_f64[i, 2], logi, mult, n, width, 17)
        err = max(np.max(np.abs(hf.yhat_lower[a:e] - lo)), np.max(np.abs(hf.yhat_upper[a:e] - hi))) / ys
        _measured["mc"] = max(_measured["mc"], err)
        assert err <= 1e-9, (name, i, err)
        flag_ref.append(io_.flags(b.y[a:e], lo, hi))
    flag_ref = np.concatenate(flag_ref)
    assert np.array_equal(out.flag.cpu().numpy(), flag_ref.astype(np.uint8)), name
    assert 0 < int(flag_ref.sum()) < flag_ref.size
