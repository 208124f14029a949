"""Every compiled fit kernel instance held to the numpy oracle (the GPU tests run with -m gpu on an H100).

The fit path is a set of compile-time instances: fit_kernel<NT, LOGI, YO, WO, DO, REG> (csrc/fit_inst.cu, 64 of them)
and grp::fit_group_kernel<G, LOGI, MULT, SEAS> (csrc/fit_group_inst.cu, 12).  They differ in which feature planes are
stored, where the yearly / weekly / daily blocks of beta start when one is missing, how long a chunk the rotation
recurrence runs, and how many threads of a CTA hold no point -- exactly where a kernel goes wrong without the rest of
the suite noticing.  CELLS names one batch per instance: the instance it must reach, the environment switches
(read at pb200_create) that route it there, and the data recipe.  Per cell and seasonality mode:

  * last_fit_variant_counts() puts every series in the cell's (variant, seasonality class), and nowhere else;
  * T, S, the mask and the changepoints (exactly) are the oracle's prepare;
  * objective and gradient at random points near initial_theta within 1e-10 / 1e-8 relative;
  * the first six L-BFGS iterations: evaluation counts identical, alpha_k within 1e-7, f_k within 1e-11 over the first
    three and 1e-9 up to the sixth (as tests/test_gpu_fullsize.py), status and iteration count the oracle's.

Beside the cells: newton_kernel's per-mask branches against the oracle's Newton run, prep_kernel's seasonality switches
1 ns either side of each threshold, and (no GPU) a check that CELLS covers exactly the instances the dispatch rules
compile and that every recipe gives its intended mask, grid and length.
"""
import dataclasses
import os
import sys
from dataclasses import dataclass, field

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper module next to this file
import fit_oracle as fo  # noqa: E402
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

NS_MIN = 60 * 10**9
NS_HOUR = 60 * NS_MIN
NS_DAY = 24 * NS_HOUR
MODES = ("additive", "multiplicative")
_BIT = {"yearly": 1, "weekly": 2, "daily": 4}

# ---------------------------------------------------------------------------------------------------------------------
# data recipes: fbprophet's set_auto_seasonalities decides the mask from the span and the smallest non-zero step
# ---------------------------------------------------------------------------------------------------------------------
# mask -> (nominal step, nominal span, smallest step [lo, hi), span [lo, hi), Prophet options); None: unbounded
RECIPES = {
    0: (15 * NS_MIN, NS_DAY, (1, None), (1, 2 * NS_DAY), {}),                                # one day of 15-minute data
    1: (7 * NS_DAY, 800 * NS_DAY, (7 * NS_DAY, None), (730 * NS_DAY, None), {}),             # weekly cadence, 800 days
    2: (NS_DAY, 60 * NS_DAY, (NS_DAY, 7 * NS_DAY), (14 * NS_DAY, 730 * NS_DAY), {}),         # daily, 60 days
    3: (NS_DAY, 800 * NS_DAY, (NS_DAY, 7 * NS_DAY), (730 * NS_DAY, None), {}),               # daily, 800 days
    4: (NS_HOUR, 10 * NS_DAY, (1, NS_DAY), (2 * NS_DAY, 14 * NS_DAY), {}),                   # hourly, 10 days
    5: (12 * NS_HOUR, 800 * NS_DAY, (1, NS_DAY), (730 * NS_DAY, None), {"weekly_seasonality": False}),
    6: (NS_HOUR, 30 * NS_DAY, (1, NS_DAY), (14 * NS_DAY, 730 * NS_DAY), {}),                 # hourly, 30 days
    7: (12 * NS_HOUR, 800 * NS_DAY, (1, NS_DAY), (730 * NS_DAY, None), {}),                  # 12-hour step, 800 days
}
START = np.datetime64("2019-01-01T05:17", "ns").astype(np.int64)        # off midnight, off the week's start


def _in(v, bounds):
    lo, hi = bounds
    return v >= lo and (hi is None or v < hi)


def _regular_step(mask, T, step=None):
    """The step of a regular series of T points with the recipe's mask (None if none exists): the nominal span spread
    over T points, in whole minutes, clamped into the mask's range of smallest steps; ``step`` pins it (tables)."""
    st0, span, dt, sp, _ = RECIPES[mask]
    if step is None:
        step = max(span // (T - 1) // NS_MIN * NS_MIN, NS_MIN)
        lo, hi = dt
        step = max(step, lo)
        if hi is not None and step >= hi:
            step = hi - hi // 24
    return step if _in(step, RECIPES[mask][2]) and _in((T - 1) * step, sp) else None


def _irregular_gaps(mask, T, rng):
    """T - 1 jittered gaps with one duplicate timestamp (a zero gap), whose smallest non-zero one and total keep the
    recipe's mask (None if T points cannot)."""
    st0, span, dt, sp, _ = RECIPES[mask]
    n = T - 1
    if n < 3:
        return None
    m = max(min(st0, span // (2 * n) // NS_MIN * NS_MIN), dt[0])
    if dt[1] is not None and m >= dt[1]:
        return None
    span = max(span, -(-5 * n * m // 4))
    if not _in(span, sp):
        return None
    dup = n // 2
    w = rng.uniform(0.2, 1.0, n)
    w[0] = w[dup] = 0.0
    g = m + np.floor((span - (n - 1) * m) * w / w.sum()).astype(np.int64)
    g[0], g[dup] = m, 0
    g[-1 if dup != n - 1 else -2] += span - int(g.sum())
    return g


def _y(ds, seed):
    rng = np.random.default_rng([91, seed])
    d = ds / NS_DAY
    u = (ds - ds[0]) / max(int(ds[-1] - ds[0]), 1)
    level = np.exp(rng.uniform(np.log(2e2), np.log(2e4))) * (0.5 + 0.5 / (1.0 + np.exp(-rng.uniform(2, 8) * (u - 0.5))))
    seas = (1.0 + 0.2 * np.sin(2 * np.pi * d / 365.25 + rng.uniform(0, 6)) + 0.1 * np.sin(2 * np.pi * d / 7.0 + 1.0)
            + 0.15 * np.sin(2 * np.pi * d + rng.uniform(0, 6)))
    return np.maximum(np.rint(level * seas * (1.0 + rng.normal(0.0, 0.05, ds.size))), 1.0).astype(np.int32)


def _series(mask, T, regular, seed, step=None):
    """(ds, y) of one series of the recipe, or None when T points cannot have the mask on that grid."""
    if regular:
        st = _regular_step(mask, T, step)
        if st is None:
            return None
        ds = START + seed * 37 * NS_MIN + st * np.arange(T, dtype=np.int64)
    else:
        g = _irregular_gaps(mask, T, np.random.default_rng([17, seed]))
        if g is None:
            return None
        ds = START + seed * 37 * NS_MIN + np.concatenate(([0], np.cumsum(g)))
    return ds, _y(ds, seed)


def tab_chunk(T, P):
    """Host mirror of fit_kernel.cuh tab_chunk (the seasonal-table variants' chunk; -1: the series keeps rotation)."""
    c0 = (T + 31) // 32
    for c in range(c0, c0 + 13):
        if all((c * dl) % P not in (0, 1, P - 1) for dl in range(1, 32)):
            return c
    return -1


# ---------------------------------------------------------------------------------------------------------------------
# the cells: one per compiled instance
# ---------------------------------------------------------------------------------------------------------------------
ENV = {
    "nt32": {"PB200_LC0_MAX": 1 << 30, "PB200_NO_TAB": 1},   # one warp per series, no tables: REG 0 / 1 at NT 32
    "nt128": {"PB200_LC0_MAX": 0},                            # every series with T > 0 on four warps
    "tab32": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 0},   # one warp per series with the week (REG 2) / day (REG 3) table
    "g8": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 8, "PB200_PLAIN_GROUP": 1},
    "g16": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 16, "PB200_PLAIN_GROUP": 1},
}
# lengths around the thread geometry: under one warp, NT - 1 / NT / NT + 1, and one that is not a multiple of NT
BASE_LENGTHS = {32: (13, 31, 32, 33, 101), 128: (13, 33, 127, 128, 129, 301)}
# one long regular series per yearly-bearing mask on the rotation path (the recurrence's drift over a long chunk)
LONG = {1: (7 * NS_DAY, 12000), 3: (NS_DAY, 26280), 5: (NS_HOUR, 26280), 7: (NS_HOUR, 26280)}
# a year of 15-minute data on G = 8
LONG_TAB = (15 * NS_MIN, 35040)


@dataclass(frozen=True)
class Cell:
    instance: tuple          # ("fit", NT, logistic, mask, REG) or ("group", G, logistic, multiplicative, seasonal)
    env: str                 # key of ENV
    mask: int
    regular: bool
    step: int = None         # pinned regular step (the table variants)
    modes: tuple = MODES     # seasonality modes to run (one for the grouped kernel, whose mode is compiled in)
    long: tuple = ()         # (step, T) of extra long regular series, run in multiplicative mode
    lengths: tuple = field(default=(), compare=False)

    @property
    def vcell(self):
        """The (variant, seasonality class) last_fit_variant_counts reports for the cell."""
        if self.instance[0] == "group":
            return 3, self.mask
        return self.instance[4], self.mask

    @property
    def growth(self):
        return "logistic" if self.instance[2] else "linear"


def _lengths(mask, regular, geom, step=None, chunk=None):
    """BASE_LENGTHS of the geometry, each moved up by whole multiples of it until the recipe (and the table's chunk
    rule) admits it, so that T mod NT stays the edge it was chosen for."""
    out = []
    for i, T0 in enumerate(BASE_LENGTHS[geom]):
        T = T0
        while T < 40000 and (_series(mask, T, regular, i, step) is None or (chunk is not None and chunk(T) < 0)):
            T += geom
        assert T < 40000, (mask, regular, T0)
        out.append(T)
    return tuple(out)


def _build_cells():
    cells = {}

    def add(name, **kw):
        c = Cell(**kw)
        geom = c.instance[1] if c.instance[0] == "fit" else 32
        chunk = None
        if c.instance[0] == "group" and c.instance[4]:
            chunk = lambda T: fo.grp_chunk(T, 96, c.instance[1])       # noqa: E731
        elif c.instance[0] == "fit" and c.instance[4] >= 2:
            P = 168 if c.instance[4] == 2 else 96
            chunk = lambda T: tab_chunk(T, P)                          # noqa: E731
        cells[name] = Cell(**kw, lengths=_lengths(c.mask, c.regular, geom, c.step, chunk))

    for nt in (32, 128):
        for logi in (0, 1):
            g = "logistic" if logi else "linear"
            for mask in range(8):
                for reg in ((0,) if mask == 0 else (0, 1)):
                    lg = LONG.get(mask, ()) if reg == 1 and logi else ()
                    add(f"nt{nt}_{g}_m{mask}_reg{reg}", instance=("fit", nt, logi, mask, reg), env=f"nt{nt}", mask=mask,
                        regular=reg == 1 or mask == 0, modes=MODES if mask else ("multiplicative",),
                        long=(lg,) if lg else ())
            add(f"nt32_{g}_m6_reg2", instance=("fit", 32, logi, 6, 2), env="tab32", mask=6, regular=True, step=NS_HOUR)
            add(f"nt32_{g}_m6_reg3", instance=("fit", 32, logi, 6, 3), env="tab32", mask=6, regular=True,
                step=15 * NS_MIN)
    for G in (8, 16):
        for logi in (0, 1):
            g = "logistic" if logi else "linear"
            for mult in (0, 1):
                lg = (LONG_TAB,) if G == 8 and logi and mult else ()
                add(f"g{G}_{g}_{MODES[mult]}", instance=("group", G, logi, mult, True), env=f"g{G}", mask=6,
                    regular=True, step=15 * NS_MIN, modes=(MODES[mult],), long=lg)
            add(f"g{G}_{g}_plain", instance=("group", G, logi, 0, False), env=f"g{G}", mask=0, regular=True,
                modes=("multiplicative",))
    return cells


CELLS = _build_cells()


def _compiled_instances():
    """The instances the dispatch compiles, from its rules: fit_inst.cu instantiates every mask 0..7 at NT 32 / 128 x
    growth x REG 0 (stored planes) / 1 (per-thread rotation), except REG 1 for mask 0 (no Fourier features to rotate),
    plus the table variants REG 2 / 3 for mask 6 at NT 32; fit_group_inst.cu instantiates G 8 / 16 x growth x mode for
    the seasonal class and G x growth for the class without seasonality."""
    fit = {("fit", nt, logi, mask, reg) for nt in (32, 128) for logi in (0, 1) for mask in range(8) for reg in (0, 1)
           if not (mask == 0 and reg == 1)}
    fit |= {("fit", 32, logi, 6, reg) for logi in (0, 1) for reg in (2, 3)}
    grp = {("group", G, logi, mult, True) for G in (8, 16) for logi in (0, 1) for mult in (0, 1)}
    grp |= {("group", G, logi, 0, False) for G in (8, 16) for logi in (0, 1)}
    return fit, grp


def _cell_series(cell, mode):
    out = [_series(cell.mask, T, cell.regular, i, cell.step) for i, T in enumerate(cell.lengths)]
    if cell.mask == 0 and cell.instance[0] == "fit":      # mask 0 has no rotation variant: both grids share REG 0
        out += [_series(0, T, False, 10 + i) for i, T in enumerate(cell.lengths[:2])]
    if mode == "multiplicative":
        for i, (st, T) in enumerate(cell.long):
            ds = START + st * np.arange(T, dtype=np.int64)
            out.append((ds, _y(ds, 20 + i)))
    return out


def _ragged(series):
    offs = np.zeros(len(series) + 1, np.int64)
    np.cumsum([s[0].size for s in series], out=offs[1:])
    n = len(series)
    return synth.RaggedBatch(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), offs,
                             np.concatenate([s[0] for s in series]), np.concatenate([s[1] for s in series]))


def _oracle_mask(p):
    return sum(_BIT[s.name] for s in p.seasonalities)


def _options(cell, mode, **kw):
    extra = RECIPES[cell.mask][4]
    return (dict(growth=cell.growth, seasonality_mode=mode, **extra, **kw),
            po.ProphetOptions(growth=cell.growth, seasonality_mode=mode, **extra))


# ---------------------------------------------------------------------------------------------------------------------
# no GPU: the table is complete and the recipes are what they claim
# ---------------------------------------------------------------------------------------------------------------------
def test_cells_cover_every_compiled_instance():
    fit, grp = _compiled_instances()
    assert len(fit) == 64 and len(grp) == 12
    got = [c.instance for c in CELLS.values()]
    assert len(got) == len(set(got)), "two cells for one instance"
    assert set(got) == fit | grp, (sorted(fit | grp - set(got)), sorted(set(got) - fit - grp))
    for c in CELLS.values():
        assert c.env in ENV
        if c.instance[0] == "group":
            assert c.mask == (6 if c.instance[4] else 0) and c.regular and len(c.modes) == 1
            assert c.modes == (MODES[c.instance[3]],) or not c.instance[4]       # the plain class has no mode
        else:
            assert (c.instance[4] >= 1) == (c.regular and c.mask != 0)
            assert c.modes == (MODES if c.mask else ("multiplicative",))
    # every yearly-bearing mask has its long rotation case at both CTA widths, the day table its long grouped one
    assert {(c.instance[1], c.mask) for c in CELLS.values() if c.long and c.instance[0] == "fit"} == \
        {(nt, m) for nt in (32, 128) for m in (1, 3, 5, 7)}
    assert any(c.long == (LONG_TAB,) for c in CELLS.values() if c.instance[0] == "group")


def _is_regular(ds):
    d = np.diff(ds)
    return bool(np.all(d == d[0]) and d[0] > 0)


@pytest.mark.parametrize("name", list(CELLS))
def test_recipe_gives_its_mask_grid_and_length(name):
    cell = CELLS[name]
    geom = cell.instance[1] if cell.instance[0] == "fit" else 32
    Ts = [T for T in cell.lengths]
    assert [T % geom for T in Ts] == [T % geom for T in BASE_LENGTHS[geom]]
    for mode in cell.modes:
        _, oopts = _options(cell, mode)
        series = _cell_series(cell, mode)
        n_long = len(cell.long) if mode == "multiplicative" else 0
        for j, (ds, y) in enumerate(series):
            p = po.prepare(ds, y.astype(np.float64), 0.0, 1.1 * y.max(), oopts)
            assert _oracle_mask(p) == cell.mask, (name, j, ds.size)
            assert p.T == ds.size and np.all(np.diff(ds) >= 0)
            if j < len(cell.lengths):
                assert p.T == cell.lengths[j]
                assert _is_regular(ds) == cell.regular, (name, j)
            elif j >= len(series) - n_long:
                assert _is_regular(ds) and p.T == cell.long[j - (len(series) - n_long)][1]
            else:                                                   # mask 0's irregular companions
                assert cell.mask == 0 and not _is_regular(ds)
            if not _is_regular(ds):
                assert np.sum(np.diff(ds) == 0) == 1                # one duplicate timestamp
            if cell.step is not None and _is_regular(ds):
                assert ds[1] - ds[0] == cell.step
            if cell.instance[0] == "fit" and cell.instance[4] >= 2:
                assert tab_chunk(p.T, 168 if cell.instance[4] == 2 else 96) > 0
            if cell.instance[0] == "group" and cell.instance[4]:
                assert fo.grp_chunk(p.T, 96, cell.instance[1]) > 0 and p.S + 17 <= 44


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every cell against the oracle
# ---------------------------------------------------------------------------------------------------------------------
_measured = {"f": 0.0, "g": 0.0, "f_k": 0.0, "f_k6": 0.0, "alpha_k": 0.0, "newton_f": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report_measured_deviations():
    yield
    if any(_measured.values()):
        print(f"\n[kernel instances] max relative deviation from the oracle: objective {_measured['f']:.3e} (1e-10), "
              f"gradient {_measured['g']:.3e} (1e-8), f_k rows 1-3 {_measured['f_k']:.3e} (1e-11), "
              f"f_k rows 4-6 {_measured['f_k6']:.3e} (1e-9), "
              f"alpha_k {_measured['alpha_k']:.3e} (1e-7), Newton objective {_measured['newton_f']:.3e} (1e-4)")


@pytest.fixture(scope="module")
def ctx_env():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = fo.ctx_with_env(**ENV[name])
        return cache[name]

    yield get
    for c in cache.values():
        c.close()


_GPU_CASES = [(name, mode) for name, c in CELLS.items() for mode in c.modes]


@pytest.mark.gpu
@pytest.mark.parametrize("name,mode", _GPU_CASES)
def test_instance_matches_oracle(ctx_env, name, mode):
    cell = CELLS[name]
    ctx = ctx_env(cell.env)
    b = _ragged(_cell_series(cell, mode))
    kw, oopts = _options(cell, mode)
    opts = batched.make_options(**kw)
    lay = L.get_layout(opts)
    # objective and gradient at random points near the initial one
    th, preps = fo.thetas(b, oopts, lay, np.random.RandomState(11))
    f, g, mi = batched.objective_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    vc = ctx.last_fit_variant_counts()
    assert vc[cell.vcell] == b.n and vc.sum() == b.n, (name, vc)
    for i, (p, t) in enumerate(preps):
        err, fo_, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0, (name, i, mi[i])
        assert (mi[i, 0], mi[i, 1], mi[i, 3]) == (p.T, p.S, _oracle_mask(p)), (name, i, mi[i])
        df = abs(f[i] - fo_) / max(1.0, abs(fo_))
        dg = np.max(np.abs(g[i, :t.size] - go)) / max(1.0, np.max(np.abs(go)))
        _measured["f"], _measured["g"] = max(_measured["f"], df), max(_measured["g"], dg)
        assert df <= 1e-10, (name, i, p.T, f[i], fo_)
        assert dg <= 1e-8, (name, i, p.T, dg)
    # the first iterations of the fit, its status and iteration count
    o6 = batched.make_options(**kw, max_iter=6, algorithm="LBFGS")
    o6_oracle = dataclasses.replace(oopts, max_iter=6)
    fb, tr = batched.fit_batch_trace_host(ctx, o6, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=8)
    vc = ctx.last_fit_variant_counts()
    assert vc[cell.vcell] == b.n and vc.sum() == b.n, (name, vc)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr, rows = fo.oracle_rows(b.ds[a:e], b.y[a:e].astype(np.float64), o6_oracle)
        S = fr.prep.S
        assert (fb.meta_i32[i, 0], fb.meta_i32[i, 1], fb.meta_i32[i, 3]) == (fr.prep.T, S, _oracle_mask(fr.prep)), (name, i)
        assert np.array_equal(fb.tchange[i, :S], fr.prep.t_change) and np.all(fb.tchange[i, S:] == 0.0), (name, i)
        n_gpu = int(fb.meta_i32[i, 5])
        # rows 1-3 at _assert_trajectory_head's tolerances; rows 4-6 keep evaluation counts and alpha_k, and f_k within
        # 1e-9, as test_gpu_fullsize: the two summation orders' rounding difference grows along the identical path
        # (to ~1e-10 by row 6 on the 13-point yearly + daily series, whose Fourier features carry ~1e-13 of rounding)
        fo.assert_trajectory_head(tr[i], n_gpu, rows, (name, mode, i, fr.prep.T), n_head=3)
        head = min(n_gpu, len(rows), 6)
        gk, ok = tr[i, :head], rows[:head]
        assert np.array_equal(gk[:, 0], ok[:, 0]) and np.array_equal(gk[:, 3], ok[:, 3]), (name, mode, i, gk, ok)
        df = np.abs(gk[:, 1] - ok[:, 1]) / np.maximum(1.0, np.abs(ok[:, 1]))
        da = np.abs(gk[:, 2] - ok[:, 2]) / np.abs(ok[:, 2])
        _measured["f_k"] = max(_measured["f_k"], float(df[:3].max()))
        _measured["f_k6"] = max(_measured["f_k6"], float(df.max()))
        _measured["alpha_k"] = max(_measured["alpha_k"], float(da.max()))
        assert np.all(df <= 1e-9) and np.all(da <= 1e-7), (name, mode, i, df, da)
        assert (fb.meta_i32[i, 4], n_gpu) == (fr.ret, fr.iters), (name, i, fb.meta_i32[i], fr.ret, fr.iters)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: newton_kernel's run-time branch per mask bit
# ---------------------------------------------------------------------------------------------------------------------
NEWTON_MASKS = (1, 2, 3, 4, 5, 7)


@pytest.mark.gpu
@pytest.mark.parametrize("mask", NEWTON_MASKS)
def test_newton_matches_oracle_newton(ctx_env, mask):
    """The recipe's regular series and a short irregular one through fbprophet's Newton run, against the oracle's
    stan_newton at DESIGN's 1e-4 relative (see test_newton_only_matches_oracle_newton for why not tighter)."""
    step, span = RECIPES[mask][:2]
    series = [_series(mask, span // step + 1, True, 30, step), _series(mask, 45, False, 31)]
    b = _ragged(series)
    extra = RECIPES[mask][4]
    opts = batched.make_options(algorithm="Newton", **extra)
    oopts = po.ProphetOptions(**extra)
    ctx = ctx_env("nt32")
    fb = batched.fit_batch_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=oopts, algorithm="Newton")
        assert _oracle_mask(fr.prep) == mask and fb.meta_i32[i, 3] == mask
        assert fb.meta_i32[i, 4] == L.ST_NEWTON == fr.ret, (mask, i, fb.meta_i32[i])
        assert np.array_equal(fb.tchange[i, :fr.prep.S], fr.prep.t_change)
        d = abs(fb.meta_f64[i, 3] - fr.neg_logp) / max(1.0, abs(fr.neg_logp))
        _measured["newton_f"] = max(_measured["newton_f"], d)
        assert d <= 1e-4, (mask, i, fb.meta_f64[i, 3], fr.neg_logp)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: prep_kernel's seasonality switches on and 1 ns either side of each threshold
# ---------------------------------------------------------------------------------------------------------------------
def _threshold_series():
    out = []
    for span in (730 * NS_DAY, 14 * NS_DAY, 2 * NS_DAY):          # span decides (smallest step one hour)
        for d in (-1, 0, 1):
            head = NS_HOUR * np.arange(24, dtype=np.int64)
            tail = np.linspace(30 * NS_HOUR, span + d, 16).astype(np.int64)
            tail[-1] = span + d
            out.append(np.concatenate((head, tail)))
    for step, big in ((7 * NS_DAY, 9 * NS_DAY), (NS_DAY, 2 * NS_DAY)):    # smallest step decides (span above 14 days)
        for d in (-1, 0, 1):
            g = np.array([step + d] + [big + 3 * NS_HOUR * j for j in range(12)], np.int64)
            out.append(np.concatenate(([0], np.cumsum(g))))
        # a duplicate timestamp is not a step: the smallest one stays `step`
        g = np.array([step, 0] + [big + 3 * NS_HOUR * j for j in range(12)], np.int64)
        out.append(np.concatenate(([0], np.cumsum(g))))
    return [START + ds for ds in out]


def test_threshold_series_sit_on_their_thresholds():
    ds = _threshold_series()
    spans = [int(s[-1] - s[0]) for s in ds]
    steps = [int(np.diff(s)[np.diff(s) > 0].min()) for s in ds]
    for k, th in enumerate((730, 14, 2)):
        assert spans[3 * k:3 * k + 3] == [th * NS_DAY - 1, th * NS_DAY, th * NS_DAY + 1]
    for k, th in enumerate((7 * NS_DAY, NS_DAY)):
        assert steps[9 + 4 * k:12 + 4 * k] == [th - 1, th, th + 1] and steps[12 + 4 * k] == th
        assert np.sum(np.diff(ds[12 + 4 * k]) == 0) == 1
    assert min(spans[9:]) >= 14 * NS_DAY
    # each switch flips exactly at its threshold, and the duplicate leaves the smallest step where it was
    m = [_oracle_mask(po.prepare(s, np.arange(s.size, dtype=np.float64) % 7 + 1, 0.0, 9.0, po.ProphetOptions()))
         for s in ds]
    for k, bit in enumerate((1, 2, 4)):
        assert m[3 * k] & bit == 0 and m[3 * k + 1] & bit and m[3 * k + 2] & bit, m
    for k, bit in enumerate((2, 4)):
        i = 9 + 4 * k
        assert m[i] & bit and not m[i + 1] & bit and not m[i + 2] & bit and m[i + 3] == m[i + 1], m


@pytest.mark.gpu
def test_seasonality_switches_at_their_thresholds(gpu_ctx):
    ds = _threshold_series()
    ys = [(50 + 10 * np.sin(np.arange(s.size)) + np.arange(s.size) % 3).astype(np.int32) for s in ds]
    b = _ragged(list(zip(ds, ys)))
    fb = batched.fit_batch_host(gpu_ctx, batched.make_options(max_iter=1), b.ds, b.y, b.offsets, 0.0, 1.1)
    want = [_oracle_mask(po.prepare(s, y.astype(np.float64), 0.0, 1.1 * y.max(), po.ProphetOptions()))
            for s, y in zip(ds, ys)]
    assert list(fb.meta_i32[:, 3]) == want, (list(fb.meta_i32[:, 3]), want)
    assert np.all(fb.meta_i32[:, 4] >= 0)
