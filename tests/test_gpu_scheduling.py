"""GPU tests of how the fit kernels SCHEDULE series (run with -m gpu on an H100), against the oracle and against themselves.

tests/test_gpu_parity.py and tests/test_gpu_optimiser.py check every kernel on small batches of equal series, where each
workspace slot stages exactly one series.  A full-size batch does more: a slot takes series after series (its workspace,
shared state and registers still holding the last one), the groups of one grouped-kernel warp hold series of different
length and cadence and enter and leave on different rounds, slots past the L2-resident share stream evict-first, and the
options are not always the defaults.  These tests reach all of that at test size:

  * mixed warps: day-table series of 674..8000 points on 15 / 20 / 30-minute grids, off-midnight starts, in one warp of the
    grouped kernel (4 series at 8 lanes each, 2 at 16) -- objective and gradient against the oracle and bit-equal to the
    same series evaluated alone (a series' result must not depend on its warp neighbours);
  * PB200_FIT_GRID_MAX (read at pb200_create) caps the CTAs of every fit / Newton launch, so that one slot fits dozens of
    series in turn: every output must be byte-identical to the uncapped launch, for every kernel family;
  * the L2 cache-hint modes of the grouped kernel (PB200_L2_KEEP_PCT), stale workspace across calls, and the Prophet
    options the C ABI accepts (changepoints, changepoint range, history size, max_iter, seasonality prior scale).
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper module next to this file
import fit_oracle  # noqa: E402
from fit_oracle import grp_chunk  # noqa: E402
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

pytestmark = pytest.mark.gpu

NS_MIN = 60 * 10**9
NS_DAY = 86400 * 10**9

# kernel families (the environment switches are read by pb200_create)
FAMILIES = {
    "g8": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 8, "PB200_PLAIN_GROUP": 1},     # grouped, 8 lanes per series
    "g16": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 16, "PB200_PLAIN_GROUP": 1},   # grouped, 16 lanes per series
    "tab32": {"PB200_LC0_MAX": 1 << 30, "PB200_GROUP": 0},                          # one warp per series, day table
    "rot32": {"PB200_LC0_MAX": 1 << 30, "PB200_NO_TAB": 1},                         # one warp per series, rotation
    "default": {},                                                                  # small batch: 4 warps per series
}


@pytest.fixture(scope="module")
def ctx_for():
    """ctx_for(family, **more_env) -> a context of the module (one per distinct environment)."""
    cache = {}

    def get(family, **more):
        env = dict(FAMILIES[family], **more)
        key = tuple(sorted((k, str(v)) for k, v in env.items()))
        if key not in cache:
            cache[key] = fit_oracle.ctx_with_env(**env)
        return cache[key]

    yield get
    for c in cache.values():
        c.close()


# ---- host mirrors of the grouped kernel's geometry (fit_kernel.cuh grp_chunk, fit_group.cuh group_plane_doubles) ----
def last_lane_points(T, step_min, G):
    return max(0, T - (G - 1) * grp_chunk(T, NS_DAY // (step_min * NS_MIN), G))


def plane_doubles(tmax, G, U=2, slack=24, hmax=5, gppad=44):
    cmax = (tmax + G - 1) // G + slack
    d = (cmax + U - 1) // U * G * U + 8 + 2 * hmax * gppad
    return (d + 1) & ~1


# ---- series of config #3's shape on other grids, lengths and start times ----
def _series(T, step_min, start, seed):
    rng = np.random.default_rng([77, seed])
    ds = np.datetime64(start, "ns").astype(np.int64) + step_min * NS_MIN * np.arange(T, dtype=np.int64)
    days = ds / NS_DAY
    u = np.linspace(0.0, 1.0, T)
    lvl = np.exp(rng.uniform(np.log(1e3), np.log(1e5)))
    r = rng.uniform(2.0, 10.0) * rng.choice([-1.0, 1.0], p=[0.3, 0.7])
    level = lvl * (0.25 + 0.75 / (1.0 + np.exp(-r * (u - rng.uniform(0.2, 0.8)))))
    daily = 1.0 + rng.uniform(0.05, 0.4) * np.sin(2 * np.pi * days + rng.uniform(0, 2 * np.pi))
    weekly = 1.0 + rng.uniform(0.0, 0.2) * np.sin(2 * np.pi * days / 7.0 + rng.uniform(0, 2 * np.pi))
    y = level * daily * weekly * (1.0 + rng.normal(0.0, 0.05, T))
    return ds, np.maximum(np.rint(y), 1.0).astype(np.int32)


def _batch(specs):
    """specs: (T, step in minutes, start) per series."""
    parts = [_series(T, st, s0, i) for i, (T, st, s0) in enumerate(specs)]
    offs = np.zeros(len(parts) + 1, np.int64)
    np.cumsum([p[0].size for p in parts], out=offs[1:])
    n = len(parts)
    return synth.RaggedBatch(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), offs,
                             np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))


# Lengths chosen with grp_chunk: near the shortest with weekly seasonality on each grid (two weeks + 1 point), where the
# last lane has an odd number of points (G = 8: 674 @ 30 min -> 79, 1010 @ 20 min -> 121, 1346 @ 15 min -> 163), and at
# 16 lanes, where the chunk is widened, none (737 @ 30 min) or one (751 @ 30 min); beside the 8000-point series (chunk
# 1000 at G = 8), whose steps the whole warp runs
LONG = (8000, 15, "2021-03-01T00:00")             # a Monday, midnight
ODD30 = (674, 30, "2021-03-03T07:30")             # Wednesday
ODD20 = (1010, 20, "2021-03-06T13:20")            # Saturday
ODD15 = (1346, 15, "2021-03-04T05:45")            # Thursday
ZERO30 = (737, 30, "2021-03-02T22:00")
ONE30 = (751, 30, "2021-03-07T11:30")

MIXED = {
    "g8_mixed4": ("g8", [ODD30, LONG, ODD20, ODD15]),
    "g8_one": ("g8", [ODD30]),
    "g8_three": ("g8", [LONG, ODD30, ODD20]),
    "g8_five": ("g8", [ODD15, LONG, ODD30, ZERO30, ODD20]),
    "g16_odd": ("g16", [LONG, ODD30]),
    "g16_zero": ("g16", [ZERO30, LONG]),
    "g16_one": ("g16", [LONG, ONE30]),
}


def test_mixed_lengths_are_the_edges_they_claim():
    assert all(last_lane_points(T, st, 8) % 2 == 1 for T, st, _ in (ODD30, ODD20, ODD15))
    assert last_lane_points(*ZERO30[:2], 16) == 0 and last_lane_points(*ONE30[:2], 16) == 1
    for T, st, _ in (ODD30, ODD20, ODD15, ZERO30, ONE30, LONG):
        assert (T - 1) * st * NS_MIN >= 14 * NS_DAY                      # weekly seasonality on: the day-table class
        assert grp_chunk(T, NS_DAY // (st * NS_MIN), 8) > 0 and grp_chunk(T, NS_DAY // (st * NS_MIN), 16) > 0
    for T, st, _ in (ZERO30, ONE30):
        assert grp_chunk(T, NS_DAY // (st * NS_MIN), 16) > (T + 15) // 16    # widened: the last lane runs short


@pytest.mark.parametrize("point", ["near_initial", "steep"])
@pytest.mark.parametrize("which", list(MIXED))
def test_mixed_warp_objective_matches_oracle_and_series_alone(ctx_for, which, point):
    family, specs = MIXED[which]
    ctx = ctx_for(family)
    b = _batch(specs)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    lay = L.get_layout(opts)
    th, preps = fit_oracle.thetas(b, oopts, lay, np.random.RandomState(3), steep=point == "steep")
    f, g, mi = batched.objective_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    vc = ctx.last_fit_variant_counts()
    assert vc[3, 6] == b.n and vc.sum() == b.n, vc
    for i, (p, t) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(t, p)
        assert err == 0 and np.isfinite(fo) and np.all(np.isfinite(go))
        assert mi[i, 4] == 0, (which, point, i, mi[i])
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (which, point, i, f[i], fo)
        gd = np.max(np.abs(g[i, :t.size] - go)) / max(1.0, np.max(np.abs(go)))
        assert gd <= 1e-8, (which, point, i, gd)
        one = b.take(i, i + 1)
        f1, g1, m1 = batched.objective_host(ctx, opts, one.ds, one.y, one.offsets, 0.0, 1.1, th[i:i + 1])
        assert m1[0, 4] == 0
        assert f1[0].tobytes() == f[i].tobytes() and g1[0].tobytes() == g[i].tobytes(), (which, point, i)


# ---------------------------------------------------------------------------------------
# grid cap: one slot fits many series in turn; nothing may change
# ---------------------------------------------------------------------------------------
def _tight_opts():
    o = batched.make_options(algorithm="LBFGS", max_iter=20000)
    o.tol_rel_grad = o.tol_rel_obj = o.tol_grad = o.tol_param = 0.0
    o.tol_obj = 1e-13
    o.algorithm = L.ALG_LBFGS_NEWTON
    return o


def _irregular(n=6):
    rng = np.random.RandomState(42)
    step = 3 * 3600 * 10**9
    ds_l, y_l = [], []
    for i in range(n):
        idx = np.sort(rng.choice(np.arange(3000), 1500 + 100 * i, replace=False))
        ds = np.datetime64("2016-02-01T00:00", "ns").astype(np.int64) + step * idx + i * 7 * NS_MIN
        days = (ds - ds[0]) / NS_DAY
        y = 400 * (1 + 0.1 * np.sin(2 * np.pi * days / 7 + i) + 0.2 * np.sin(2 * np.pi * days)) * (1 + 0.3 * days / days.max())
        ds_l.append(ds)
        y_l.append(np.maximum(np.rint(y + rng.normal(0, 10, ds.size)), 1).astype(np.int32))
    offs = np.zeros(n + 1, np.int64)
    np.cumsum([d.size for d in ds_l], out=offs[1:])
    return synth.RaggedBatch(np.zeros(n, np.int32), np.arange(n, dtype=np.int32), offs, np.concatenate(ds_l), np.concatenate(y_l))


def _lsfail_batch():
    parts = [synth.config4(n=500_000, lo=i, hi=i + 1) for i in synth.CONFIG4_LSFAIL_IDS] + [synth.config4(n=40)]
    offs = np.concatenate(([0], np.cumsum(np.concatenate([np.diff(p.offsets) for p in parts])))).astype(np.int64)
    return synth.RaggedBatch(np.zeros(offs.size - 1, np.int32), np.zeros(offs.size - 1, np.int32), offs,
                             np.concatenate([p.ds for p in parts]), np.concatenate([p.y for p in parts]))


MIXED16 = [LONG, ODD30, ODD20, ODD15, ZERO30, ONE30, (1500, 15, "2021-03-05T01:15"), (700, 30, "2021-03-01T12:00"),
           (2016, 20, "2021-03-02T04:40"), (3000, 15, "2021-03-06T23:45"), (1100, 20, "2021-03-03T00:20"),
           (5000, 15, "2021-03-07T18:00"), (900, 30, "2021-03-04T09:30"), (1400, 15, "2021-03-01T02:30"),
           (2500, 30, "2021-03-05T16:00"), (1800, 20, "2021-03-02T19:40")]

# name -> (family, batch, options, expected (variant, seasonality mask) cell or None)
GRID_CASES = {
    "g8_config3": ("g8", lambda: synth.config3(n=48), batched.make_options, (3, 6)),
    "g8_mixed": ("g8", lambda: _batch(MIXED16), batched.make_options, (3, 6)),
    "g16_config3": ("g16", lambda: synth.config3(n=24), batched.make_options, (3, 6)),
    "g16_mixed": ("g16", lambda: _batch(MIXED16), batched.make_options, (3, 6)),
    "tab32": ("tab32", lambda: synth.config3(n=16), batched.make_options, (3, 6)),
    "rot32": ("rot32", lambda: synth.config3(n=16), batched.make_options, (1, 6)),
    "irregular_planes": ("tab32", _irregular, batched.make_options, (0, 6)),
    "default_4_warps": ("default", lambda: synth.config3(n=16), batched.make_options, (1, 6)),
    "plain_g8": ("g8", lambda: synth.config4(n=64), batched.make_options, (3, 0)),
    "plain_g16": ("g16", lambda: synth.config4(n=64), batched.make_options, (3, 0)),
    "newton_only": ("default", lambda: synth.config4(n=12), lambda: batched.make_options(algorithm="Newton"), None),
    "lbfgs_newton_retry": ("default", _lsfail_batch, _tight_opts, None),
}


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _assert_same_fit(x, y, what):
    (fa, ta), (fb, tb) = x, y
    for name in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64"):
        assert np.array_equal(_bits(getattr(fa, name)), _bits(getattr(fb, name))), (what, name)
    assert np.array_equal(_bits(ta), _bits(tb)), (what, "trace")


@pytest.mark.parametrize("case", list(GRID_CASES))
def test_grid_cap_changes_no_result(ctx_for, case):
    family, mk, mko, cell = GRID_CASES[case]
    b, opts = mk(), mko()
    runs = {}
    for cap in (0, 1, 3):
        ctx = ctx_for(family, **({"PB200_FIT_GRID_MAX": cap} if cap else {}))
        runs[cap] = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=64)
        vc = ctx.last_fit_variant_counts()
        if cap == 0:
            vc0 = vc
            if cell is not None:
                assert vc[cell] == b.n, (case, vc)
        assert np.array_equal(vc, vc0), (case, cap, vc, vc0)
    st = runs[0][0].meta_i32[:, 4]
    assert np.all(st >= 0), (case, st)
    if case == "newton_only":
        assert np.all(st == L.ST_NEWTON)
    if case == "lbfgs_newton_retry":
        assert np.any(st == L.ST_NEWTON)                  # the retry queue is not empty
    for cap in (1, 3):
        _assert_same_fit(runs[0], runs[cap], (case, cap))


def test_reused_slots_follow_the_oracle(ctx_for):
    """At one CTA a G = 8 warp fits the 16 series of the mixed batch four at a time, groups refilling on different
    rounds: every series' first iterations still match the oracle's."""
    ctx = ctx_for("g8", PB200_FIT_GRID_MAX=1)
    b = _batch(MIXED16)
    fb, tr = batched.fit_batch_trace_host(ctx, batched.make_options(), b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=8)
    assert ctx.last_fit_variant_counts()[3, 6] == b.n
    oopts = po.ProphetOptions(max_iter=6)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr, rows = fit_oracle.oracle_rows(b.ds[a:e], b.y[a:e].astype(np.float64), oopts)
        assert fb.meta_i32[i, 4] >= 0
        assert np.array_equal(fb.tchange[i, :fr.prep.S], fr.prep.t_change)
        fit_oracle.assert_trajectory_head(tr[i], int(fb.meta_i32[i, 5]), rows, i)


def test_stale_workspace_from_a_longer_batch_changes_nothing(ctx_for):
    """The workspace of a context is reused across calls: after a batch of 8000-point series has filled it, a batch of short
    series must give what a fresh context gives."""
    opts = batched.make_options()
    short = _batch([ODD30, ODD20, ODD15, ZERO30, ONE30, (1500, 15, "2021-03-05T01:15")])
    long_ = _batch([(8000, 15, f"2021-03-0{d}T0{d}:15") for d in range(1, 9)])
    used = fit_oracle.ctx_with_env(**FAMILIES["g8"])
    fresh = fit_oracle.ctx_with_env(**FAMILIES["g8"])
    try:
        batched.fit_batch_trace_host(used, opts, long_.ds, long_.y, long_.offsets, 0.0, 1.1, trace_cap=16)
        x = batched.fit_batch_trace_host(used, opts, short.ds, short.y, short.offsets, 0.0, 1.1, trace_cap=16)
        y = batched.fit_batch_trace_host(fresh, opts, short.ds, short.y, short.offsets, 0.0, 1.1, trace_cap=16)
    finally:
        used.close()
        fresh.close()
    _assert_same_fit(x, y, "stale workspace")
    assert np.all(x[0].meta_i32[:, 4] >= 0)


def test_l2_cache_hint_modes_change_no_result(ctx_for):
    """PB200_L2_KEEP_PCT: -1 no hints, 0 every slot evict-first, 1 a mix, 65 (default) every slot evict_last at this size."""
    import torch
    b = synth.config3(n=96)
    opts = batched.make_options()
    cap, G = 16, 8
    nslots = min((b.n + 32 // G - 1) // (32 // G), cap) * (32 // G)
    slot_bytes = plane_doubles(1440, G) * 8
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    keep = {pct: min(nslots, (l2 // 100) * pct // slot_bytes) for pct in (0, 1, 65)}
    assert keep[0] == 0 and 0 < keep[1] < nslots and keep[65] == nslots, (keep, nslots)
    runs = []
    for pct in (-1, 0, 1, 65):
        ctx = ctx_for("g8", PB200_FIT_GRID_MAX=cap, PB200_L2_KEEP_PCT=pct)
        runs.append(batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=16))
        assert ctx.last_fit_variant_counts()[3, 6] == b.n
    for r, pct in zip(runs[1:], (0, 1, 65)):
        _assert_same_fit(runs[0], r, ("l2 keep pct", pct))


# ---------------------------------------------------------------------------------------
# Prophet options on the grouped kernel and its neighbours
# ---------------------------------------------------------------------------------------
OPTION_CASES = {
    "n_changepoints_0": {"n_changepoints": 0},
    "n_changepoints_1": {"n_changepoints": 1},
    "n_changepoints_27": {"n_changepoints": 27},       # S + 17 = 44: the grouped kernel's longest vector
    "n_changepoints_28": {"n_changepoints": 28},       # one longer: the one-warp rotation variant takes the class
    "changepoint_range_0.5": {"changepoint_range": 0.5},
    "changepoint_range_1.0": {"changepoint_range": 1.0},
    "history_size_1": {"history_size": 1},
    "history_size_3": {"history_size": 3},
    "max_iter_1": {"max_iter": 1},
    "max_iter_7": {"max_iter": 7},
    "seasonality_prior_scale_0.1": {"seasonality_prior_scale": 0.1},
}


@pytest.mark.parametrize("case", list(OPTION_CASES))
def test_options_on_the_grouped_kernel(ctx_for, case):
    kw = dict(OPTION_CASES[case])
    hist = kw.pop("history_size", 5)
    opts = batched.make_options(**kw)
    opts.history_size = hist
    oopts = po.ProphetOptions(history_size=hist, **kw)
    ctx = ctx_for("g8")
    b = _batch([ODD30, LONG, ODD20, ODD15])
    cell = (1, 6) if kw.get("n_changepoints") == 28 else (3, 6)
    lay = L.get_layout(opts)
    # objective and gradient at random points near the initial one
    th, preps = fit_oracle.thetas(b, oopts, lay, np.random.RandomState(9))
    f, g, mi = batched.objective_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, th)
    assert ctx.last_fit_variant_counts()[cell] == b.n, (case, ctx.last_fit_variant_counts())
    for i, (p, t) in enumerate(preps):
        err, fo, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0 and (mi[i, 1], mi[i, 2]) == (p.S, len(p.t_change) if kw.get("n_changepoints") != 0 else 0)
        assert abs(f[i] - fo) <= 1e-10 * max(1.0, abs(fo)), (case, i, f[i], fo)
        assert np.max(np.abs(g[i, :t.size] - go)) <= 1e-8 * max(1.0, np.max(np.abs(go))), (case, i)
    # the fit: changepoints exactly, the first iterations, and (max_iter) the status of the whole run
    fb, tr = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=8)
    assert ctx.last_fit_variant_counts()[cell] == b.n
    short_run = "max_iter" in kw
    # changepoint_range 1.0 puts the last changepoint ON the last point, where the likelihood's derivative in its delta is
    # exactly zero in the oracle (t_last - t_change = 0) and rounding noise in the grouped kernel (t_i = i h, one rounding
    # from (ds_i - start) / span).  The Laplace prior's kink at delta = 0 turns the sign of that noise into a +-1 / tau
    # gradient from the second iteration on, so only the first is compared there (the objective and gradient above are)
    n_head = 1 if kw.get("changepoint_range") == 1.0 else 6
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        o_run = oopts if short_run else po.ProphetOptions(history_size=hist, **dict(kw, max_iter=6))
        fr, rows = fit_oracle.oracle_rows(b.ds[a:e], b.y[a:e].astype(np.float64), o_run)
        S = fr.prep.S
        assert fb.meta_i32[i, 1] == S and np.array_equal(fb.tchange[i, :S], fr.prep.t_change), (case, i)
        assert np.all(fb.tchange[i, S:] == 0.0)
        fit_oracle.assert_trajectory_head(tr[i], int(fb.meta_i32[i, 5]), rows, (case, i), n_head=n_head)
        if short_run:
            assert fb.meta_i32[i, 4] == fr.ret and fb.meta_i32[i, 5] == fr.iters, (case, i, fb.meta_i32[i], fr.ret, fr.iters)
            if kw["max_iter"] == 1:
                assert fr.ret == L.ST_MAXIT
