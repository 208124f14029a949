"""Extra regressors (DESIGN §19) where their columns move: held to the numpy oracle (tests/regressor_oracle.py) on
batches whose series have different table masks, at the widths §19 admits, and at the edges of the fit status, the
frame, the standardisation and the data movement.  The GPU tests run with -m gpu on an H100.

Series i's regressor r is beta[K_seas(mask_i) + r]: the table fit kernel, newton_kernel, predict_kernel and mc_kernel
each compute that offset on their own, and the table kernel stages the regressor planes after the series' own active
seasonal planes.  So:

  * mixed-mask cells: one call over series with masks 0 (K = R), 1, 2, 3, 6 and 7 (P = 67, three optimiser elements per
    lane) and lengths 31, 32, 33, on the defaults table and on [monthly] + the built-ins, R = 5 with a prior scale and a
    standardize of its own per regressor, both growths and modes;
  * width cells: K = 64 with P = 96 (p96), K = 63 with P = 96 and a half-used last plane (r15), and K = R = 16 with every
    seasonality off (off16), both growths;
  * a series fitted after a wider or narrower one in the same warp, on one CTA and on the default grid, gives its bytes
    alone; a line-search failure hands a regressor model to its Newton retry; failures and a non-finite future value
    (also past the first 1024 points, where a model spans two predict CTAs) touch only their own model;
  * reg_scale_kernel at its lane tails and decision edges, the future join and the backtest's gather at R = 16.

Without a GPU: every cell has the masks, K, S, P and R it claims, the library lays it out as claimed, and the histories
of the retry test fail their tight-stop L-BFGS runs on the numpy oracle.
"""
import dataclasses
import json
import os
import sys
from dataclasses import dataclass

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import fit_oracle as fo  # noqa: E402
import regressor_oracle as ro  # noqa: E402
import seasonality_table as st  # noqa: E402
import test_kernel_instances as ki  # noqa: E402
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

NS_MIN, NS_HOUR, NS_DAY = ki.NS_MIN, ki.NS_HOUR, ki.NS_DAY
HPS = 4.0                                   # holidays_prior_scale, away from its default of 10
STANDARDIZE = ("auto", True, False)         # regressor r takes STANDARDIZE[r % 3]
I32_MIN = np.iinfo(np.int32).min

# name -> (make_table_options' built-in switches, custom entries)
TABLES = {
    "defaults": (dict(), []),
    "monthly": (dict(), [dict(name="monthly", period=30.5, fourier_order=5, prior_scale=3.0)]),
    "wide": (dict(yearly_seasonality=20, weekly_seasonality=4, daily_seasonality=False), []),
    "off": (dict(yearly_seasonality=False, weekly_seasonality=False, daily_seasonality=False), []),
}

# the mixed-mask series (ki._series recipes: mask, T, regular grid, seed, pinned step), ordered so that a series with
# more active entries comes right before one with fewer and the reverse: 7 -> 0 -> 3 -> 2 -> 6 -> 1 -> 2
MIXED = ((7, 1601, True, 0, None),             # 12-hour steps over 800 days: P = 67 with R = 5
         (0, 31, True, 1, None),               # one day of 48-minute steps: no seasonality, K = R
         (3, 801, True, 2, None),              # daily, 800 days
         (2, 32, True, 3, None),               # weekly only, 60 days
         (6, 1400, True, 4, 15 * NS_MIN),      # weekly + daily, 15-minute data
         (1, 115, True, 5, None),              # weekly steps over 800 days: yearly only
         (2, 33, False, 6, None))              # irregular, one duplicate timestamp
WIDE = ((3, 801, True, 10, None), (3, 601, False, 11, None), (3, 33 * 24 + 1, True, 12, None))


@dataclass(frozen=True)
class Cell:
    table: str
    growth: str
    mode: str
    R: int
    series: tuple
    ncp: int = 25
    kmax: int = 0            # the layout the library gives the options
    pstride: int = 0

    @property
    def builtin(self):
        """The oracle's built-in switches (seasonality_table.seasonalities)."""
        return {k.replace("_seasonality", ""): v for k, v in TABLES[self.table][0].items()}


def _prior_scales(R):
    """R = 5: explicit and omitted (holidays_prior_scale) scales; R >= 15: distinct ones, regressor 5's omitted."""
    if R == 5:
        return (0.5, None, 2.0, None, 0.25)
    return tuple(None if r == 5 else round(0.2 + 0.15 * r, 2) for r in range(R))


def _regressors(R):
    out = []
    for r, ps in enumerate(_prior_scales(R)):
        spec = dict(name=f"x{r}", standardize=STANDARDIZE[r % 3])
        if ps is not None:
            spec["prior_scale"] = ps
        out.append(spec)
    return out


def _cells():
    cells = {}
    for table, kmax, pstride in (("defaults", 39, 67), ("monthly", 49, 77)):
        for growth in ("linear", "logistic"):
            for mode in ("additive", "multiplicative"):
                cells[f"{table}-{growth}-{mode}"] = Cell(table, growth, mode, 5, MIXED, kmax=kmax, pstride=pstride)
    for name, table, ncp, R, kmax, pstride in (("p96", "wide", 29, 16, 64, 96), ("r15", "wide", 30, 15, 63, 96),
                                               ("off16", "off", 25, 16, 16, 44)):
        for growth, mode in (("linear", "additive"), ("logistic", "multiplicative")):
            cells[f"{name}-{growth}"] = Cell(table, growth, mode, R, WIDE, ncp, kmax, pstride)
    return cells


CELLS = _cells()
WIDTH_CELLS = [k for k in CELLS if not k.startswith(("defaults", "monthly"))]


def _options(cell, **extra):
    """(library options, oracle options) of a cell; ``extra``: make_options' max_iter / algorithm."""
    kw, custom = TABLES[cell.table]
    opts = batched.make_regressor_options(_regressors(cell.R), holidays_prior_scale=HPS, seasonalities=custom,
                                          growth=cell.growth, seasonality_mode=cell.mode, n_changepoints=cell.ncp,
                                          **kw, **extra)
    oopts = po.ProphetOptions(growth=cell.growth, seasonality_mode=cell.mode, n_changepoints=cell.ncp,
                              **{k: v for k, v in extra.items() if k == "max_iter"})
    return opts, oopts


def _values(ds, R, seed):
    """[R, T] regressor values of one history (or frame): kind r % 5 is a {0, 1} flag, a price around 10, a temperature,
    a slow wave, another flag -- so that with STANDARDIZE some flags are standardised and some are not."""
    ds = np.asarray(ds, np.int64)
    rng = np.random.default_rng([71, seed])
    t = (ds - ki.START).astype(np.float64) / NS_DAY
    kinds = [lambda: (rng.random(ds.size) < 0.3).astype(np.float64), lambda: 10.0 + rng.normal(size=ds.size),
             lambda: 15.0 + 8.0 * rng.normal(size=ds.size), lambda: 1.5 + np.cos(t / 9.0 + seed),
             lambda: (rng.random(ds.size) < 0.6).astype(np.float64)]
    return np.stack([kinds[r % 5]() for r in range(R)]) if R else np.zeros((0, ds.size))


def _history(rec, R):
    """(ds, y, values) of one recipe: y carries an effect of each regressor, so that every beta is away from 0."""
    mask, T, regular, seed, step = rec
    ds, y = ki._series(mask, T, regular, seed, step)
    x = _values(ds, R, seed)
    z = (x - x.mean(axis=1, keepdims=True)) / (x.std(axis=1, keepdims=True) + 1.0)
    w = 0.08 * np.cos(np.arange(R) + seed)
    y = np.maximum(np.rint(y * (1.0 + w @ z)), 1.0).astype(np.int32)
    return ds, y, x


def _batch(series, R):
    """(RaggedBatch, values [R, rows]) of recipes, or of (ds, y, values) triples."""
    hs = [s if len(s) == 3 and isinstance(s[0], np.ndarray) else _history(s, R) for s in series]
    return ki._ragged([(ds, y) for ds, y, _ in hs]), np.ascontiguousarray(np.concatenate([x for _, _, x in hs], axis=1))


def _entries(cell):
    kw, custom = TABLES[cell.table]
    return st.table_entries(cell.builtin, custom)


def _prep(cell, oopts, b, i, reg, scale, columns="exact"):
    """ro.prepare of series i on its (mu, std) ``scale[i]``.  Returns (prepared, seasonalities, table mask)."""
    a, e = b.offsets[i], b.offsets[i + 1]
    y = b.y[a:e].astype(np.float64)
    opts, _ = _options(cell)
    p, seas = ro.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts, cell.builtin, TABLES[cell.table][1], reg[:, a:e],
                         scale[i], ro.prior_scales(opts), columns)
    return p, seas, st.table_mask(seas, _entries(cell))


# ---------------------------------------------------------------------------------------------------------------------
# the histories of the retry test: regressor models whose tight-stop L-BFGS run ends in a line-search failure
# ---------------------------------------------------------------------------------------------------------------------
LSFAIL_CELL = "defaults-logistic-multiplicative"
LSFAIL = ((7, 801, False, 42, None), (7, 801, False, 44, None), (7, 801, False, 46, None))


def _tight(opts):
    opts.tol_rel_grad = opts.tol_rel_obj = opts.tol_grad = opts.tol_param = 0.0
    opts.tol_obj = 1e-13
    return opts


def _tight_oracle(oopts):
    return dataclasses.replace(oopts, max_iter=20000, tol_rel_grad=0.0, tol_rel_obj=0.0, tol_grad=0.0, tol_param=0.0,
                               tol_obj=1e-13)


# ---------------------------------------------------------------------------------------------------------------------
# no GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CELLS))
def test_cells_have_the_layouts_they_claim(name):
    cell = CELLS[name]
    opts, oopts = _options(cell)
    lay = L.get_layout(opts)
    assert (lay.kmax, lay.pstride, batched.n_regressors(opts)) == (cell.kmax, cell.pstride, cell.R), name
    b, reg = _batch(cell.series, cell.R)
    scale = batched.regressor_scales(reg, b.offsets, [STANDARDIZE[r % 3] for r in range(cell.R)])
    shapes = []
    for i, rec in enumerate(cell.series):
        p, seas, mask = _prep(cell, oopts, b, i, reg, scale, "numpy")
        assert p.T == rec[1] and ki._is_regular(b.ds[b.offsets[i]:b.offsets[i + 1]]) == rec[2], (name, i)
        k_seas = sum(2 * o for _, _, o, _ in seas)
        assert p.K == k_seas + cell.R and p.S == min(cell.ncp, p.S) and p.S + p.K + 3 <= cell.pstride, (name, i)
        # the built-in bits are the recipe's, the custom entry always on
        builtin = sum({"yearly": 1, "weekly": 2, "daily": 4}[s[0]] for s in seas if s[0] != "monthly")
        if cell.table in ("defaults", "monthly"):
            assert builtin == rec[0], (name, i)
            assert mask == batched.table_mask(batched.seasonality_table(opts), builtin)
        shapes.append((mask, p.S, p.K, p.S + p.K + 3))
    masks = {m for m, _, _, _ in shapes}
    if cell.table == "defaults":
        assert len(masks) >= 4 and 0 in masks and max(P for *_, P in shapes) == 67, shapes
        assert [K for m, _, K, _ in shapes if m == 0] == [cell.R]               # K = R: no zero column
    elif cell.table == "monthly":
        assert len(masks) >= 4 and all(m & 1 for m in masks) and max(P for *_, P in shapes) == 77, shapes
    elif cell.table == "wide":
        assert masks == {3} and {(K, P) for _, _, K, P in shapes} == {(cell.kmax, 96)}, shapes
    else:
        assert masks == {0} and {K for _, _, K, _ in shapes} == {16}, shapes
    assert {T for _, T, *_ in MIXED} >= {31, 32, 33}


def test_one_more_column_on_p96_is_refused():
    """p96 with one more changepoint is r15 with one more regressor: P = 97."""
    kw, _ = TABLES["wide"]
    with pytest.raises((L.Pb200Error, ValueError), match=r"P = .* = 97"):
        batched.make_regressor_options(_regressors(16), n_changepoints=30, **kw)
    with pytest.raises(ValueError, match="at most 16"):
        batched.make_regressor_options(_regressors(16) + [dict(name="x16")], n_changepoints=29, **kw)


def test_line_search_failures_on_the_oracle():
    """The histories the retry test uses end their tight-stop L-BFGS runs in a line-search failure on the numpy oracle
    (with the host standardisation; the GPU's differs in the last bits)."""
    cell = CELLS[LSFAIL_CELL]
    _, oopts = _options(cell)
    b, reg = _batch(LSFAIL, cell.R)
    scale = batched.regressor_scales(reg, b.offsets, [STANDARDIZE[r % 3] for r in range(cell.R)])
    for i in range(b.n):
        p, _, mask = _prep(cell, oopts, b, i, reg, scale)
        assert mask == 7 and p.S + p.K + 3 == 67
        fr = st.fit(p, _tight_oracle(oopts))
        assert fr.ret == po.TERM_LSFAIL, (LSFAIL[i], fr.ret, fr.iters)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
# the largest error of each check over the module, relative to its bound's scale (DESIGN §19 states them); printed when
# the module's tests end (visible with -s)
MAXIMA = {}


def _note(key, value):
    MAXIMA[key] = max(MAXIMA.get(key, 0.0), float(value))


@pytest.fixture(scope="module", autouse=True)
def _report_maxima():
    yield
    if MAXIMA:
        print("\nmeasured maxima, tests/test_gpu_regressor_layouts.py: " + json.dumps(MAXIMA, sort_keys=True))


def _table_count(ctx):
    n = np.zeros(1, np.int64)
    L.check(L.load().pb200_last_fit_table_count(ctx.handle, n.ctypes.data), "pb200_last_fit_table_count")
    return int(n[0])


def _steps(b):
    """Each series' own step (its largest gap), so that a frame spans about as many t units as it has points."""
    return np.array([int(np.diff(b.ds[b.offsets[i]:b.offsets[i + 1]]).max()) if b.offsets[i + 1] - b.offsets[i] > 1
                     else NS_HOUR for i in range(b.n)], np.int64)


def _frame(b, H):
    last = b.ds[b.offsets[1:] - 1]
    return last[:, None] + _steps(b)[:, None] * np.arange(1, H + 1, dtype=np.int64)[None, :]


def _check_scales(scale, reg, offsets, standardize, what):
    """reg_scale against batched.regressor_scales: the decision exact, |dmu| <= 1e-13 max|x|, std within 1e-12."""
    ref = batched.regressor_scales(reg, offsets, standardize)
    bad = np.isnan(ref[:, :, 0])
    assert np.array_equal(bad, np.isnan(scale[:, :, 0])) and np.all(np.isnan(scale[bad])), what
    keep = lambda s: (s[:, :, 0] == 0) & (s[:, :, 1] == 1)          # noqa: E731
    assert np.array_equal(keep(ref), keep(scale)), (what, keep(ref), keep(scale))
    for i in range(offsets.size - 1):
        x = reg[:, offsets[i]:offsets[i + 1]]
        if x.shape[1] == 0:
            continue
        ok = ~bad[i]
        xmax = np.maximum(np.max(np.abs(x[ok]), axis=1), 1e-300)
        dmu = np.abs(scale[i, ok, 0] - ref[i, ok, 0]) / xmax
        dsd = np.abs(scale[i, ok, 1] - ref[i, ok, 1]) / ref[i, ok, 1]
        _note("mu_abs_over_max_abs_x", dmu.max(initial=0.0))
        _note("std_rel", dsd.max(initial=0.0))
        assert np.all(dmu <= 1e-13) and np.all(dsd <= 1e-12), (what, i, dmu, dsd)
    return ref


def _got(fb, i, p):
    """Row i of a fitted batch as an oracle FitResult on the series' prepared history."""
    S, K = p.S, p.K
    return po.FitResult(prep=p, k=fb.params[i, 0], m=fb.params[i, 1], delta=fb.params[i, 3:3 + S],
                        sigma_obs=fb.params[i, 2], beta=fb.params[i, 3 + fb.smax:3 + fb.smax + K], theta=None,
                        neg_logp=0.0, iters=0, n_evals=0, ret=0)


def _mc_bounds(monkeypatch, opts, fb, i, fut, cap, freg, mask, seed):
    """oracle/mc_stream's bounds of model i with the regressor term.  mc_stream evaluates its seasonal term only when
    its mask has a built-in bit (1 | 2 | 4), which a table mask of 0 lacks although the regressor term is there: it gets a
    copy of the fit with mask 7, and a seasonal term that ignores the mask it is given and uses the model's own."""
    from oracle import mc_stream
    f = ro.mc_seasonal(opts, freg, fb.reg_scale[i])
    monkeypatch.setattr(mc_stream, "_seasonal", lambda ds, _mask, beta: f(ds, mask, beta))
    fm = batched.FittedBatch(fb.params, fb.tchange, fb.meta_i32.copy(), fb.meta_i64, fb.meta_f64, fb.smax, fb.kmax)
    fm.meta_i32[i, 3] = 7
    d = mc_stream.draws(fm, i, fut, 0.0, cap, opts.growth == L.GROWTH_LOGISTIC, opts.multiplicative == 1,
                        opts.uncertainty_samples, seed)
    return mc_stream.bounds(d, opts.interval_width)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CELLS))
def test_cell_matches_oracle(gpu_ctx, monkeypatch, name):
    """Per series, with its own mask, K and P:
      * prep: meta_i32[:, 3] the oracle's table mask, tchange[:S] its t_change exactly, every series in the table class;
      * reg_scale against batched.regressor_scales: the decision exact, |dmu| <= 1e-13 max|x|, std within 1e-12;
      * objective and gradient at random points near initial_theta (the row past the series' own P padded with 0.5, which
        a kernel reading another series' width would take as betas) within 1e-10 / 1e-8 relative of ro.prepare's
        "exact" columns on the GPU's (mu, std);
      * the first six L-BFGS rows: evaluation counts identical, alpha_k within 1e-7, f_k within 1e-11 over rows 1-3
        and 1e-9 over rows 4-6 (§18's rules);
      * the fitted objective one-sided, cell median <= 5e-4 and every series <= 5e-2;
      * yhat within 1e-12 y_scale of ro.predict_yhat on a 60-point and an 1100-point frame (two CTAs per model), the same
        bits with intervals as without, and the 60-point bounds within 1e-9 y_scale of mc_stream's draws."""
    cell = CELLS[name]
    opts, oopts = _options(cell)
    b, reg = _batch(cell.series, cell.R)
    lay = L.get_layout(opts)
    stdz = [STANDARDIZE[r % 3] for r in range(cell.R)]
    zero = np.zeros((b.n, lay.pstride))
    _, _, _, scale = batched.objective_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, zero, regressors=reg)
    _check_scales(scale, reg, b.offsets, stdz, name)
    rng = np.random.RandomState(3)
    rows, preps = [], []
    for i in range(b.n):
        p, seas, mask = _prep(cell, oopts, b, i, reg, scale)
        th = po.initial_theta(p) + 0.05 * rng.randn(p.S + p.K + 3)
        row = np.full(lay.pstride, 0.5)
        row[:th.size] = th
        rows.append(row)
        preps.append((p, seas, mask, th))
    f, g, mi, scale2 = batched.objective_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, np.array(rows),
                                              regressors=reg)
    assert _table_count(gpu_ctx) == b.n and scale2.tobytes() == scale.tobytes()
    for i, (p, seas, mask, th) in enumerate(preps):
        err, fo_, go = po.neg_logp_grad(th, p)
        assert err == 0 and mi[i, 4] == 0 and (mi[i, 0], mi[i, 1], mi[i, 3]) == (p.T, p.S, mask), (name, i, mi[i])
        df = abs(f[i] - fo_) / max(1.0, abs(fo_))
        dg = np.max(np.abs(g[i, :th.size] - go)) / max(1.0, np.max(np.abs(go)))
        _note("objective_rel", df)
        _note("gradient_rel", dg)
        assert df <= 1e-10 and dg <= 1e-8, (name, i, p.T, mask, df, dg)
    masks = [m for _, _, m, _ in preps]
    if cell.table in ("defaults", "monthly"):
        assert len(set(masks)) >= 4 and (cell.table != "defaults" or 0 in masks), masks
    # the fit, its first six iterations and its end point
    fb, trace = batched.fit_batch_trace_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=8,
                                             regressors=reg)
    assert _table_count(gpu_ctx) == b.n
    assert fb.reg_scale.tobytes() == scale.tobytes()
    assert list(fb.meta_i32[:, 3]) == masks
    if cell.table == "wide":
        assert {int(3 + fb.meta_i32[i, 1] + 40 + 8 + cell.R) for i in range(b.n)} == {96} and fb.kmax == cell.kmax
    relf = []
    for i, (p, seas, mask, _) in enumerate(preps):
        tr = []
        fr = st.fit(p, oopts, trace=tr)
        o = np.array(tr).reshape(-1, 4)
        assert fb.meta_i32[i, 4] >= 0 and fr.ret >= 0, (name, i, fb.meta_i32[i], fr.ret)
        assert np.array_equal(fb.tchange[i, :p.S], p.t_change) and np.all(fb.tchange[i, p.S:] == 0.0), (name, i)
        # §18's rules (tests/test_gpu_table_instances.py): rows 1-3 at fo.assert_trajectory_head's tolerances, rows 4-6
        # with identical evaluation counts, alpha_k within 1e-7 and f_k within 1e-9 -- the two summation orders'
        # rounding difference grows along the identical path (to 3.3e-11 by row 6 of the 15-minute weekly + daily series)
        n_gpu = int(fb.meta_i32[i, 5])
        fo.assert_trajectory_head(trace[i], n_gpu, o, (name, i, p.T, mask), n_head=3)
        head = min(n_gpu, len(o), 6)
        gk, ok = trace[i, :head], o[:head]
        assert np.array_equal(gk[:, 0], ok[:, 0]) and np.array_equal(gk[:, 3], ok[:, 3]), (name, i, gk, ok)
        tf = np.abs(gk[:, 1] - ok[:, 1]) / np.maximum(1.0, np.abs(ok[:, 1]))
        ta = np.abs(gk[:, 2] - ok[:, 2]) / np.abs(ok[:, 2])
        _note("trajectory_f_rel_rows_1_3", tf[:3].max())
        _note("trajectory_f_rel_rows_4_6", tf.max())
        _note("trajectory_alpha_rel", ta.max())
        assert np.all(tf <= 1e-9) and np.all(ta <= 1e-7), (name, i, p.T, mask, tf, ta)
        relf.append((fb.meta_f64[i, 3] - fr.neg_logp) / abs(fr.neg_logp))
    relf = np.array(relf)
    worse = np.maximum(relf, 0.0)
    _note("fitted_objective_worse_median", np.median(worse))
    _note("fitted_objective_worse", worse.max())
    assert np.median(worse) <= 5e-4 and worse.max() <= 5e-2, (name, relf)
    # predict on two frames, with and without intervals, and the bounds against mc_stream
    cap32 = fb.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    for H, seed in ((60, 7), (1100, 9)):
        fut = _frame(b, H)
        freg = np.stack([_values(fut[i], cell.R, 100 + i) for i in range(b.n)], axis=1)
        plain = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, intervals=False,
                                           regressors=freg)
        fc = batched.predict_batch_host(gpu_ctx, opts, fb, fut, np.zeros(b.n), cap32, seed=seed, regressors=freg)
        assert fc.yhat.tobytes() == plain.yhat.tobytes(), (name, H)
        for i, (p, seas, mask, _) in enumerate(preps):
            want = ro.predict_yhat(_got(fb, i, p), seas, fut[i], 0.0, cap32[i], oopts, freg[:, i], fb.reg_scale[i])
            dp = np.max(np.abs(want - plain.yhat[i])) / p.y_scale
            _note("predict_over_y_scale", dp)
            assert dp <= 1e-12, (name, H, i, mask, dp)
            if H > 60:
                continue
            lo, hi = _mc_bounds(monkeypatch, opts, fb, i, fut[i], cap32[i], freg[:, i], mask, seed)
            db = max(np.max(np.abs(lo - fc.yhat_lower[i])), np.max(np.abs(hi - fc.yhat_upper[i]))) / fb.meta_f64[i, 0]
            _note("bounds_over_y_scale", db)
            assert db <= 1e-9, (name, i, mask, db)


NEWTON_CELLS = WIDTH_CELLS + ["defaults-logistic-multiplicative"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", NEWTON_CELLS)
def test_newton_steps_match_oracle(gpu_ctx, name):
    """PB200_ALG_NEWTON after 1, 2, 3 and 5 iterations against stan_newton on the exact columns: status 60, iteration and
    evaluation counts identical, and (fo.newton_bound) theta within 1e-6 and the objective within 1e-8 of their sizes
    plus ten times the oracle's own move when its columns change by rounding alone (stan_newton on numpy's columns).
    At P = 96 with logistic growth that move reaches 4.9e-8 of the objective and 4.3e-7 of theta after three steps: the
    finite-difference Hessian is ill-conditioned there.  96 x 96 Hessians on the width cells, every mask of a mixed
    cell, K = R on mask 0."""
    cell = CELLS[name]
    b, reg = _batch(cell.series, cell.R)
    for k in (1, 2, 3, 5):
        opts, oopts = _options(cell, max_iter=k, algorithm="Newton")
        fb = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, regressors=reg)
        for i in range(b.n):
            runs = []
            for columns in ("exact", "numpy"):
                p, _, mask = _prep(cell, oopts, b, i, reg, fb.reg_scale, columns)
                th, f, it, ret, ne = po.stan_newton(lambda x: po.neg_logp_grad(x, p), po.initial_theta(p), oopts)
                if p.n_changepoints_real == 0:
                    th[0] += th[2]
                    th[2] = 0.0
                runs.append((th, f, it, ret, ne))
            (th, f, it, ret, ne), (th_np, f_np, _, _, _) = runs
            mi = fb.meta_i32[i]
            assert mi[3] == mask and mi[4] == 60 == ret and (mi[5], mi[6]) == (it, ne), (name, k, i, mi, it, ne)
            assert np.array_equal(fb.tchange[i, :p.S], p.t_change)
            got = np.concatenate((fb.params[i, :2], fb.params[i, 3:3 + p.S], [np.log(fb.params[i, 2])],
                                  fb.params[i, 3 + fb.smax:3 + fb.smax + p.K]))
            dth, bth = fo.newton_bound(got, th, th_np, th, floor=1e-6)
            dfn, bfn = fo.newton_bound(fb.meta_f64[i, 3], f, f_np, f, floor=1e-8)
            _note("newton_theta_over_bound", dth / bth)
            _note("newton_objective_over_bound", dfn / bfn)
            assert dth <= bth and dfn <= bfn, (name, k, i, mask, dth, bth, dfn, bfn)
            if cell.table == "wide":
                assert p.S + p.K + 3 == 96


def _fit_fields(fb, i):
    return [getattr(fb, f)[i].tobytes() for f in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64", "reg_scale")]


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["defaults", "monthly"])
def test_queue_neighbours_on_one_cta(table):
    """One CTA, so one warp's queue takes the series one after another, wider before narrower and the reverse: each
    series' params, tchange, meta, reg_scale and trace rows are the bytes it gives alone."""
    cell = CELLS[f"{table}-logistic-multiplicative"]
    opts, _ = _options(cell)
    b, reg = _batch(cell.series, cell.R)
    ctx = fo.ctx_with_env(PB200_FIT_GRID_MAX=1)
    try:
        fb, tr = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=64, regressors=reg)
        assert _table_count(ctx) == b.n and len(set(fb.meta_i32[:, 3].tolist())) >= 4
        for i in range(b.n):
            a, e = b.offsets[i], b.offsets[i + 1]
            one, t1 = batched.fit_batch_trace_host(ctx, opts, b.ds[a:e], b.y[a:e], np.array([0, e - a]), 0.0, 1.1,
                                                   trace_cap=64, regressors=reg[:, a:e])
            assert _fit_fields(one, 0) == _fit_fields(fb, i), (table, i)
            assert t1[0].tobytes() == tr[i].tobytes(), (table, i)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["defaults", "monthly"])
def test_series_alone_and_in_a_mixed_batch_give_the_same_bits(gpu_ctx, table):
    cell = CELLS[f"{table}-linear-additive"]
    opts, _ = _options(cell)
    b, reg = _batch(cell.series, cell.R)
    fa = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, regressors=reg)
    fut = _frame(b, 40)
    freg = np.stack([_values(fut[i], cell.R, 200 + i) for i in range(b.n)], axis=1)
    cap32 = fa.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    pa = batched.predict_batch_host(gpu_ctx, opts, fa, fut, np.zeros(b.n), cap32, seed=3, regressors=freg)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        one = batched.fit_batch_host(gpu_ctx, opts, b.ds[a:e], b.y[a:e], np.array([0, e - a]), 0.0, 1.1,
                                     regressors=reg[:, a:e])
        assert _fit_fields(one, 0) == _fit_fields(fa, i), (table, i)
        p1 = batched.predict_batch_host(gpu_ctx, opts, one, fut[i:i + 1], np.zeros(1), cap32[i:i + 1], seed=3,
                                        regressors=np.ascontiguousarray(freg[:, i:i + 1]))
        for x, y in ((p1.yhat, pa.yhat), (p1.yhat_lower, pa.yhat_lower), (p1.yhat_upper, pa.yhat_upper),
                     (p1.yhat_int, pa.yhat_int)):
            assert x[0].tobytes() == y[i].tobytes(), (table, i)


@pytest.mark.gpu
def test_line_search_failure_gets_its_newton_retry(gpu_ctx):
    """Of the oracle's failing regressor histories (P = 67) at least one fails on the GPU too; every one that does ends
    as the Newton-only run's model, counted with both runs, no worse than where L-BFGS stopped."""
    cell = CELLS[LSFAIL_CELL]
    b, reg = _batch(LSFAIL, cell.R)
    kw = dict(max_iter=20000)
    lb = batched.fit_batch_host(gpu_ctx, _tight(_options(cell, algorithm="LBFGS", **kw)[0]), b.ds, b.y, b.offsets,
                                0.0, 1.1, regressors=reg)
    both = batched.fit_batch_host(gpu_ctx, _tight(_options(cell, algorithm="LBFGS+Newton", **kw)[0]), b.ds, b.y,
                                  b.offsets, 0.0, 1.1, regressors=reg)
    nw = batched.fit_batch_host(gpu_ctx, _options(cell, algorithm="Newton", **kw)[0], b.ds, b.y, b.offsets, 0.0, 1.1,
                                regressors=reg)
    assert np.all(nw.meta_i32[:, 4] == L.ST_NEWTON), nw.meta_i32
    failed = np.flatnonzero(lb.meta_i32[:, 4] == L.ST_LSFAIL)
    assert failed.size >= 1, lb.meta_i32
    for i in range(b.n):
        assert lb.meta_i32[i, 3] == 7 and lb.meta_i32[i, 1] + 34 + cell.R + 3 == 67
        if i not in failed:
            assert both.meta_i32[i].tobytes() == lb.meta_i32[i].tobytes()
            continue
        assert both.meta_i32[i, 4] == L.ST_NEWTON, both.meta_i32[i]
        assert both.meta_i32[i, 5] == lb.meta_i32[i, 5] + nw.meta_i32[i, 5], (both.meta_i32[i], lb.meta_i32[i])
        assert both.meta_i32[i, 6] == lb.meta_i32[i, 6] + nw.meta_i32[i, 6], (both.meta_i32[i], lb.meta_i32[i])
        assert both.params[i].tobytes() == nw.params[i].tobytes()
        assert both.reg_scale[i].tobytes() == nw.reg_scale[i].tobytes()
        fg = both.meta_f64[i, 3]
        assert fg <= lb.meta_f64[i, 3] + 1e-9 * max(1.0, abs(fg)), (i, fg, lb.meta_f64[i, 3])


@pytest.mark.gpu
def test_failures_touch_only_their_own_series(gpu_ctx):
    """In one mixed batch: a T = 1 series keeps the status it has without regressors, a NaN in a mask-0 history and an
    inf in another give PB200_ST_BAD_REGRESSOR, and every other series keeps its bits.  On an 1100-point frame a single
    NaN future value at h >= 1024 fails the whole model, h < 1024 included, and no other model's rows move."""
    cell = CELLS["defaults-logistic-multiplicative"]
    opts, _ = _options(cell)
    hs = [_history(rec, cell.R) for rec in MIXED]
    ds1 = hs[2][0][:1]
    hs.insert(3, (ds1, hs[2][1][:1], hs[2][2][:, :1]))                   # T = 1
    b, reg = _batch(hs, cell.R)
    f0 = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, regressors=reg)
    alone = batched.fit_batch_host(gpu_ctx, batched.make_table_options(), ds1, hs[3][1], np.array([0, 1]), 0.0, 1.1)
    assert f0.meta_i32[3, 4] == alone.meta_i32[0, 4] < 0, (f0.meta_i32[3], alone.meta_i32[0])
    assert f0.meta_i32[1, 3] == 0
    bad = reg.copy()
    bad[4, b.offsets[1] + 7] = np.nan                                    # the mask-0 series
    bad[2, b.offsets[5] + 100] = np.inf                                  # weekly + daily
    f1 = batched.fit_batch_host(gpu_ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, regressors=bad)
    for i in range(b.n):
        if i in (1, 5):
            assert f1.meta_i32[i, 4] == L.ST_BAD_REGRESSOR, (i, f1.meta_i32[i])
            assert np.all(np.isnan(f1.reg_scale[i, 4 if i == 1 else 2]))
        else:
            assert _fit_fields(f1, i) == _fit_fields(f0, i), i
    ok = [i for i in range(b.n) if f0.meta_i32[i, 4] >= 0]
    fut = _frame(b, 1100)
    freg = np.stack([_values(fut[i], cell.R, 300 + i) for i in range(b.n)], axis=1)
    cap32 = f0.meta_f64[:, 2].astype(np.float32).astype(np.float64)
    fbad = freg.copy()
    fbad[3, ok[0], 1050] = np.nan
    for intervals in (False, True):
        p0 = batched.predict_batch_host(gpu_ctx, opts, f0, fut, np.zeros(b.n), cap32, seed=5, intervals=intervals,
                                        regressors=freg)
        p1 = batched.predict_batch_host(gpu_ctx, opts, f0, fut, np.zeros(b.n), cap32, seed=5, intervals=intervals,
                                        regressors=fbad)
        outs = [(p0.yhat, p1.yhat), (p0.yhat_int, p1.yhat_int)]
        if intervals:
            outs += [(p0.yhat_lower, p1.yhat_lower), (p0.yhat_upper, p1.yhat_upper)]
        i = ok[0]
        assert np.all(np.isfinite(p0.yhat[i])) and np.all(np.isnan(p1.yhat[i])) and np.all(p1.yhat_int[i] == I32_MIN)
        if intervals:
            assert np.all(np.isnan(p1.yhat_lower[i])) and np.all(np.isnan(p1.yhat_upper[i]))
        for j in range(b.n):
            if j != i:
                for x, y in outs:
                    assert x[j].tobytes() == y[j].tobytes(), (intervals, j)


@pytest.mark.gpu
def test_reg_scale_kernel_edges(gpu_ctx):
    """reg_scale_kernel through pb200_regressor_scales_device and a fit's reg_scale, against batched.regressor_scales, at
    R = 16 with a standardize per index: lane tails (T = 1, 2, 31, 32, 33, 1000), {0, 1} under 'auto' and True,
    {-0.0, 1.0} under 'auto' (fbprophet's set equality), {0, 2} under 'auto', two values at T = 2, a constant column
    under True, 1e9 + N(0, 1) (std within 1e-12 needs the two-pass form), and +inf / NaN (flagged, (NaN, NaN))."""
    import torch
    std = ["auto", True, "auto", "auto", True, True, "auto", False, False, "auto", True, "auto", True, "auto", False,
           True]
    regs = [dict(name=f"x{r}", standardize=s) for r, s in enumerate(std)]
    opts = batched.make_regressor_options(regs, holidays_prior_scale=HPS)
    rng = np.random.default_rng(5)

    def column(r, T):
        kind = r % 8
        if kind == 0:
            return (np.arange(T) % 2).astype(np.float64)                   # {0, 1}
        if kind == 1:
            return np.where(np.arange(T) % 3 == 0, 1.0, 0.0)              # {0, 1} (under True at r = 1, 9)
        if kind == 2:
            return np.where(np.arange(T) % 2 == 0, -0.0, 1.0)             # {-0.0, 1.0}
        if kind == 3:
            return 2.0 * (np.arange(T) % 2)                               # {0, 2}
        if kind == 4:
            return rng.normal(size=T)
        if kind == 5:
            return np.full(T, 3.25)                                       # constant
        if kind == 6:
            return 1e9 + rng.normal(size=T)
        return 10.0 + rng.normal(size=T)

    lengths = (1, 2, 31, 32, 33, 1000, 2, 64, 64)
    cols = [np.stack([column(r, T) for r in range(16)]) for T in lengths]
    cols[6][:, 1] = cols[6][:, 0] + 0.5                                    # T = 2: two distinct values everywhere
    cols[7][4, 10] = np.inf
    cols[8][9, 63] = np.nan
    reg = np.ascontiguousarray(np.concatenate(cols, axis=1))
    off = np.concatenate(([0], np.cumsum(lengths))).astype(np.int64)
    ds = np.concatenate([ki.START + NS_DAY * np.arange(T, dtype=np.int64) for T in lengths])
    y = np.concatenate([(50 + np.arange(T) % 7).astype(np.int32) for T in lengths])
    sc, bad = batched.regressor_scales_device(gpu_ctx, opts, torch.from_numpy(reg).cuda(), off)
    sc, bad = sc.cpu().numpy(), bad.cpu().numpy()
    ref = _check_scales(sc, reg, off, std, "regressor_scales_device")
    assert bad.tolist() == [False] * 7 + [True, True]
    assert np.all(np.isnan(sc[7, 4])) and np.all(np.isnan(sc[8, 9])) and not np.isnan(sc[7, 5]).any()
    kept = (ref[:, :, 0] == 0) & (ref[:, :, 1] == 1)
    assert kept[0].all() and kept[1, 0] and not kept[1, 1]                 # T = 1; T = 2: {0, 1} under 'auto' / True
    assert not kept[5, 1] and kept[5, 0] and kept[5, 2] and not kept[5, 3] and kept[5, 5] and not kept[5, 6]
    assert not kept[6, 1] and not kept[6, 2] and kept[6, 7]
    # the fit's own standardisation (one iteration: column 14, 1e9 + N(0, 1) not standardised, makes a slow fit)
    o1 = batched.make_regressor_options(regs, holidays_prior_scale=HPS, max_iter=1)
    fb = batched.fit_batch_host(gpu_ctx, o1, ds, y, off, 0.0, 1.1, regressors=reg)
    assert fb.reg_scale.tobytes() == sc.tobytes()
    assert list(fb.meta_i32[7:, 4]) == [L.ST_BAD_REGRESSOR] * 2


def _join_reference(tab_ds, tab_off, tab_reg, group, future):
    """An exact-timestamp merge of each model's grid with its group's rows: ([R, n, H] values, NaN where no row, the
    missing counts, the first missing timestamp or INT64_MIN)."""
    R = tab_reg.shape[0]
    n, H = future.shape
    out = np.full((R, n, H), np.nan)
    missing = np.zeros(n, np.int32)
    first = np.full(n, np.iinfo(np.int64).min, np.int64)
    for i in range(n):
        g = group[i]
        a, e = (tab_off[g], tab_off[g + 1]) if g >= 0 else (0, 0)
        d = tab_ds[a:e]
        j = np.searchsorted(d, future[i])
        hit = (j < d.size) & (d[np.minimum(j, max(d.size - 1, 0))] == future[i]) if d.size else np.zeros(H, bool)
        out[:, i, hit] = tab_reg[:, a + j[hit]]
        missing[i] = int((~hit).sum())
        if (~hit).any():
            first[i] = future[i][np.flatnonzero(~hit)[0]]
    return out, missing, first


@pytest.mark.gpu
def test_join_sixteen_planes(gpu_ctx):
    """pb200_join_future_regressors_device with 16 planes and a 100-point horizon (four lane rounds), groups of one row,
    an absent group and off-grid rows: the exact-timestamp merge byte for byte, with the missing counts and the first
    missing timestamps."""
    import torch
    rng = np.random.default_rng(11)
    n, H, R = 6, 100, 16
    step = 15 * NS_MIN
    last = ki.START + step * np.array([0, 5, 9, 2, 7, 3], np.int64)
    future = last[:, None] + step * np.arange(1, H + 1, dtype=np.int64)[None, :]
    group = np.array([2, 0, -1, 3, 1, 4], np.int64)                       # model 2: no group
    rows = {0: future[1][rng.random(H) < 0.9], 1: future[4][[37]], 2: future[0],
            3: np.concatenate((future[3][:50], future[3][50:] + 7 * 10**9)), 4: future[5][[0]] - step}
    tab_ds = np.concatenate([np.sort(rows[g]) for g in range(5)])
    tab_off = np.concatenate(([0], np.cumsum([rows[g].size for g in range(5)]))).astype(np.int64)
    tab_reg = rng.normal(size=(R, tab_ds.size))
    tab_reg[3, 5] = np.nan                                                 # a NaN value is copied as it is
    dev = torch.device("cuda")
    got, missing, first = batched.join_future_regressors_device(
        gpu_ctx, torch.from_numpy(tab_ds).to(dev), tab_off, torch.from_numpy(np.ascontiguousarray(tab_reg)).to(dev),
        torch.from_numpy(group).to(dev), torch.from_numpy(future).to(dev))
    want, wmiss, wfirst = _join_reference(tab_ds, tab_off, tab_reg, group, future)
    assert got.cpu().numpy().tobytes() == want.tobytes()
    assert missing.cpu().numpy().tolist() == wmiss.tolist()
    assert first.cpu().numpy().tolist() == wfirst.tolist()
    assert wmiss[2] == H and wmiss[4] == H - 1 and wmiss[5] == H and wmiss[0] == 0 and 0 < wmiss[3] < H


@pytest.mark.gpu
def test_backtest_sixteen_regressors_over_long_windows(gpu_ctx):
    """cross_validation_device(regressors=) at R = 16 on 15-minute data with held-out windows of 288 rows
    (cv_gather_regressors_kernel's 256-thread stride loops twice): the cutoff fits bit-identical to fit_batch_device with
    the copy scales on numpy-built z, the held-out yhat byte-identical to predict_batch_device."""
    import torch
    import backtest_oracle as bo
    R = 16
    regs = _regressors(R)
    std = [STANDARDIZE[r % 3] for r in range(R)]
    step = 15 * NS_MIN
    parts = []
    for s, T in enumerate((1152, 1300, 1500)):
        ds = ki.START + s * 37 * NS_MIN + step * np.arange(T, dtype=np.int64)
        parts.append((ds, ki._y(ds, s), _values(ds, R, 40 + s)))
    ds = np.concatenate([p[0] for p in parts])
    y = np.concatenate([p[1] for p in parts])
    reg = np.ascontiguousarray(np.concatenate([p[2] for p in parts], axis=1))
    off = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    caps = np.array([float(p[1].max()) * 1.1 for p in parts])
    opts = batched.make_regressor_options(regs, holidays_prior_scale=HPS, uncertainty_samples=0)
    dev = torch.device("cuda")
    dds, dy, dreg = (torch.from_numpy(x).to(dev) for x in (ds, y, reg))
    hz, per, ini = 3 * NS_DAY, 2 * NS_DAY, 6 * NS_DAY
    fs, bad = batched.regressor_scales_device(gpu_ctx, opts, dreg, off)
    fs = fs.cpu().numpy()
    assert not bad.cpu().numpy().any()
    _check_scales(fs, reg, off, std, "full histories")
    res = batched.cross_validation_device(gpu_ctx, opts, dds, dy, off, 0.0, torch.from_numpy(caps).to(dev), hz, per,
                                          ini, keep_fits=True, regressors=dreg)
    assert (res.pair_status >= 0).all()
    he = np.concatenate([np.searchsorted(ds[off[i]:off[i + 1]], bo.generate_cutoffs(ds[off[i]:off[i + 1]], hz, per, ini),
                                         side="right") for i in range(off.size - 1)])
    f = res.fitted
    longest = 0
    for mask in sorted(set(res.pair_mask.tolist())):
        oc = batched.make_regressor_options(regs, holidays_prior_scale=HPS, yearly_seasonality=bool(mask & 1),
                                            weekly_seasonality=bool(mask & 2), daily_seasonality=bool(mask & 4),
                                            uncertainty_samples=0)
        sel = np.flatnonzero(res.pair_mask == mask)
        ser = res.pair_series[sel]
        rows = [np.arange(off[s], off[s] + he[p]) for s, p in zip(ser, sel)]
        hoff = np.concatenate(([0], np.cumsum([r.size for r in rows]))).astype(np.int64)
        hi = np.concatenate(rows)
        si = np.repeat(ser, [r.size for r in rows])
        z = np.ascontiguousarray((reg[:, hi] - fs[si, :, 0].T) / fs[si, :, 1].T)
        d = batched.fit_batch_device(gpu_ctx, oc, torch.from_numpy(ds[hi]).to(dev), torch.from_numpy(y[hi]).to(dev),
                                     hoff, 0.0, 1.0, cap=torch.from_numpy(caps[ser]).to(dev),
                                     regressors=torch.from_numpy(z).to(dev),
                                     reg_scale_copy=torch.from_numpy(np.ascontiguousarray(fs[ser])).to(dev)).to_host()
        w = d.params.shape[1]
        assert f.params[sel, :w].tobytes() == d.params.tobytes()
        for name in ("tchange", "meta_i64", "meta_f64", "reg_scale"):
            assert getattr(f, name)[sel].tobytes() == getattr(d, name).tobytes(), name
        assert np.delete(f.meta_i32[sel], 3, axis=1).tobytes() == np.delete(d.meta_i32, 3, axis=1).tobytes()
        hmax = int(max(((res.row_series == s) & (res.cutoff == res.pair_cutoff[p])).sum() for s, p in zip(ser, sel)))
        longest = max(longest, hmax)
        fut = np.zeros((sel.size, hmax), np.int64)
        zf = np.zeros((R, sel.size, hmax))
        for j, p in enumerate(sel):
            s = int(res.pair_series[p])
            r = np.flatnonzero((res.row_series == s) & (res.cutoff == res.pair_cutoff[p]))
            src = off[s] + he[p] + np.arange(r.size)
            assert (ds[src] == res.ds[r]).all()
            fut[j, :r.size], fut[j, r.size:] = res.ds[r], res.ds[r][-1]
            zf[:, j, :r.size] = (reg[:, src] - fs[s, :, :1]) / fs[s, :, 1:]
        pr = batched.predict_batch_device(gpu_ctx, oc, _dev(d), torch.from_numpy(fut).to(dev),
                                          torch.zeros(sel.size, dtype=torch.float64, device=dev),
                                          torch.from_numpy(caps[ser]).to(dev), intervals=False,
                                          regressors=torch.from_numpy(zf).to(dev))
        yh = pr.yhat.cpu().numpy()
        for j, p in enumerate(sel):
            r = np.flatnonzero((res.row_series == res.pair_series[p]) & (res.cutoff == res.pair_cutoff[p]))
            assert res.yhat[r].tobytes() == yh[j, :r.size].tobytes()
    assert longest == hz // step > 256


def _dev(fb):
    import torch
    return batched.FittedBatch(
        *(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (fb.params, fb.tchange, fb.meta_i32, fb.meta_i64,
                                                                     fb.meta_f64)), fb.smax, fb.kmax,
        reg_scale=torch.from_numpy(np.ascontiguousarray(fb.reg_scale)).cuda())
