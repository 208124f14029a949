"""Stan's five L-BFGS convergence tests on every optimiser code path, held to the oracle through the status alone (the
tests run with -m gpu on an H100).

BFGSMinimizer::step ends a fit on ABSF (|f_{k-1} - f_k| < tol_obj, status 20), RELF (that over
eps max(|f_{k-1}|, |f_k|, 1) < tol_rel_obj, 21), ABSGRAD (||g|| < tol_grad, 30), RELGRAD (|g . p| over
eps max(|f_k|, 1) < tol_rel_grad, 31) and ABSX (||s|| < tol_param, 10), tested in that order before MAXIT (40).  The
kernels compute these inputs in their own code (post_accept in fit_kernel.cuh, with a WIDE variant for P > 64, and
g_post_accept in fit_group.cuh) and do not expose them.  Each is pinned from outside instead: the oracle's run with every
tolerance 0 gives the value v_j of a rule at iteration j; at a record low (every earlier value at least 1 % above it) a
fit with max_iter = j, every other tolerance 0 and the rule's tolerance at v_j (1 + delta) must end with that rule's
status at iteration j, and at v_j (1 - delta) with MAXIT there -- status, iterations and evaluations exactly.  The two
runs put the kernel's value within delta of the oracle's.

Per cell (one per optimiser code path, routed by test_kernel_instances.ENV and checked with last_fit_variant_counts):
  * the brackets of all five rules at iteration 1 (the reset path), 2, and the last record low past the history size
    on series fitted with history_size 5, 3 and 1 (the ring buffer has wrapped), plus a series whose f_k crosses the
    max(|f|, 1) floor or changes sign (test_stop_rules_oracle.py checks each series has the property it is chosen for);
  * the trajectory head of each series against the oracle's;
  * each pair of rules with both tolerances above their values: the earlier rule in the chain wins; a tolerance of +inf
    fires its rule at iteration 1, and 0 or NaN never fires it (as in both oracles).
Beside the cells: one G = 8 and one G = 16 batch with several series per warp under one set of tolerances that stops them
at different iterations under different rules, each series as it is alone and as the oracle has it; and refits from each
series' own optimum under the default tolerances (the modeler's warm start), held to the oracle wherever the oracle's
values are clear of the tolerances.
"""
import dataclasses
import itertools
import os
import sys
from dataclasses import dataclass

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import fit_oracle as fo  # noqa: E402
import test_kernel_instances as ki  # noqa: E402
import test_wide_params as wp  # noqa: E402
import warm_oracle as wo  # noqa: E402
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

MAX_ITER = 12
HISTORIES = (5, 3, 1)            # history_size of a cell's three recipe series
DELTAS = (1e-8, 1e-6, 1e-4)      # the reported bracket widths, tightest first


def noisy_y(ds, seed):
    """Values at 1 or 1000 at random: the scaled residuals stay large, so f_k falls from about +T/8 to a few units below
    zero slowly enough for some iterates to lie in (-1, 1)."""
    rng = np.random.default_rng([73, seed])
    return np.where(rng.random(ds.size) < 0.5, 1, 1000).astype(np.int32)


@dataclass(frozen=True)
class StopCell:
    env: str                 # key of test_kernel_instances.ENV
    vcell: tuple             # (variant, seasonality class) of last_fit_variant_counts
    base: str = None         # test_kernel_instances cell whose recipe the series follow; None: the P = 67 series
    mode: str = "multiplicative"
    floor: tuple = None      # (T, seed) of the noisy series that crosses the floor

    @property
    def growth(self):
        return "linear" if self.base and "_linear_" in self.base else "logistic"

    @property
    def kw(self):
        """make_options / ProphetOptions keywords."""
        extra = ki.RECIPES[ki.CELLS[self.base].mask][4] if self.base else {}
        ncp = {} if self.base else {"n_changepoints": 30}
        return dict(growth=self.growth, seasonality_mode=self.mode, **extra, **ncp)


CELLS = {
    "nt32_planes": StopCell("nt32", (0, 6), "nt32_logistic_m6_reg0", floor=(13, 11)),
    "nt32_rotation": StopCell("nt32", (1, 6), "nt32_logistic_m6_reg1", floor=(45, 2)),
    "nt128": StopCell("nt128", (0, 6), "nt128_logistic_m6_reg0", floor=(13, 14)),
    "tab32_week": StopCell("tab32", (2, 6), "nt32_logistic_m6_reg2", floor=(365, 43)),
    "tab32_day": StopCell("tab32", (3, 6), "nt32_logistic_m6_reg3", floor=(1375, 12)),
    "g8_seasonal": StopCell("g8", (3, 6), "g8_logistic_multiplicative", floor=(1375, 12)),
    "g8_plain": StopCell("g8", (3, 0), "g8_logistic_plain", floor=(13, 8)),
    "g16_seasonal": StopCell("g16", (3, 6), "g16_logistic_multiplicative", floor=(1375, 12)),
    "g16_plain": StopCell("g16", (3, 0), "g16_logistic_plain", floor=(13, 10)),
    "wide_nt32": StopCell("nt32", (0, 7), floor=(801, 17)),
    "wide_nt128": StopCell("nt128", (0, 7), floor=(801, 17)),
    # no floor series: on linear additive noisy histories the oracle's own path turns at a relative perturbation of 1e-14
    # of the start point (the noisy series that cross the floor end in a line-search failure then), so rounding decides it
    "nt32_linear_additive": StopCell("nt32", (0, 6), "nt32_linear_m6_reg0", mode="additive"),
}


def cell_series(name):
    """[(ds, y, history_size)]: three recipe series with histories 5, 3 and 1, then the floor series (history 5)."""
    c = CELLS[name]
    if c.base is None:
        out = [wp._wide_series(False, 10 + i) for i in range(3)]
        ds = wp._wide_series(False, c.floor[1])[0]
    else:
        base = ki.CELLS[c.base]
        out = ki._cell_series(base, c.mode)[:3]
        if c.floor is None:
            return [(d, y, h) for (d, y), h in zip(out, HISTORIES)]
        ds = ki._series(base.mask, c.floor[0], base.regular, c.floor[1], base.step)[0]
    return [(d, y, h) for (d, y), h in zip(out, HISTORIES)] + [(ds, noisy_y(ds, c.floor[1]), 5)]


def oracle_options(name):
    return po.ProphetOptions(**CELLS[name].kw)


def floor_crossings(run):
    """The record-low targets at which the oracle's max(|f|, 1) floor or the sign of f decides the scale: RELGRAD's with
    |f_j| < 1, RELF's with max(|f_{j-1}|, |f_j|) < 1 or f_{j-1} f_j < 0."""
    out = [("RELGRAD", j) for j in run.record_lows("RELGRAD") if abs(run.f(j)) < 1.0]
    out += [("RELF", j) for j in run.record_lows("RELF")
            if max(abs(run.f(j - 1)), abs(run.f(j))) < 1.0 or run.f(j - 1) * run.f(j) < 0.0]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
_tightest = {}            # (cell, rule) -> the widest bracket any of its targets needed
_nan_report = []


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _tightest:
        rows = [f"  {name:22s} " + " ".join(f"{r} {_tightest[(name, r)]:.0e}" for r in fo.RULES)
                for name in CELLS if all((name, r) in _tightest for r in fo.RULES)]
        print("\n[stop rules] widest bracket a target needed, per cell and rule (tried 1e-8, 1e-6, 1e-4 and the "
              "rule's bound):\n" + "\n".join(rows))
    if _nan_report:
        print("[stop rules] NaN tolerance: " + "; ".join(sorted(set(_nan_report))))


@pytest.fixture(scope="module")
def ctx_env():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = fo.ctx_with_env(**ki.ENV[name])
        return cache[name]

    yield get
    for c in cache.values():
        c.close()


def _one(ctx, name, ds, y, history, max_iter, tols, trace_cap=0):
    """One series fitted alone: ((status, iters, n_evals), trace rows), after checking it ran on the cell's kernel."""
    opts = batched.make_options(**CELLS[name].kw, max_iter=max_iter, algorithm="LBFGS")
    opts.history_size = history
    for k, v in tols.items():
        setattr(opts, k, v)
    offs = np.array([0, ds.size], np.int64)
    fb, tr = batched.fit_batch_trace_host(ctx, opts, ds, y, offs, 0.0, 1.1, trace_cap=max(trace_cap, 1))
    vc = ctx.last_fit_variant_counts()
    assert vc[CELLS[name].vcell] == 1 and vc.sum() == 1, (name, vc)
    mi = fb.meta_i32[0]
    return (int(mi[4]), int(mi[5]), int(mi[6])), tr[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CELLS))
def test_stop_rule_brackets(ctx_env, name):
    ctx = ctx_env(CELLS[name].env)
    oopts = oracle_options(name)
    for s, (ds, y, hist) in enumerate(cell_series(name)):
        run = fo.StopRun(ds, y, oopts, MAX_ITER, hist)
        # the run to its end with every tolerance 0, and its trajectory head
        got, tr = _one(ctx, name, ds, y, hist, MAX_ITER, fo.ZERO_TOLS, trace_cap=MAX_ITER)
        assert got == (run.fr.ret, run.fr.iters, run.fr.n_evals), (name, s, got, run.fr.ret, run.fr.iters)
        assert np.array_equal(tr[:got[1], 3], run.rows[:, 3]), (name, s)
        if s < 3:
            fo.assert_trajectory_head(tr, got[1], run.rows, (name, s), n_head=3)
        else:
            # the floor series' f_k near 0 is the difference of terms of size ~T/8 (T log sigma against the residuals),
            # each rounded relative to its own size: held at test_kernel_instances' 1e-9 of rows 4-6, not 1e-11
            g, o = tr[:got[1]], run.rows
            assert np.all(np.abs(g[:, 1] - o[:, 1]) <= 1e-9 * np.maximum(1.0, np.abs(o[:, 1]))), (name, s, g, o)
            assert np.all(np.abs(g[:, 2] - o[:, 2]) <= 1e-7 * np.abs(o[:, 2])), (name, s, g, o)
        for rule in fo.RULES:
            for j in run.targets(rule):
                need = run.delta(rule, j)
                # tightest first; the brackets nest, so one that holds implies every wider one does
                held, miss = None, None
                for d in sorted(set(DELTAS) | {need}):
                    res = []
                    for side in (+1, -1):
                        tols, want = run.bracket(rule, j, side, d)
                        res.append((want, _one(ctx, name, ds, y, hist, j, tols)[0]))
                    if all(w == g for w, g in res):
                        held = d
                        break
                    if d >= need and miss is None:
                        miss = (d, res)
                assert held is not None and held <= need, (name, s, hist, rule, j, need, miss, run.values[rule][:j])
                key = (name, rule)
                _tightest[key] = max(_tightest.get(key, 0.0), held)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CELLS))
def test_stop_rule_priority(ctx_env, name):
    ctx = ctx_env(CELLS[name].env)
    ds, y, hist = cell_series(name)[0]
    run = fo.StopRun(ds, y, oracle_options(name), MAX_ITER, hist)
    v1 = {r: float(run.values[r][0]) for r in fo.RULES}
    n1 = int(run.rows[0, 3])
    for a, b in itertools.combinations(fo.RULES, 2):          # a comes first in the chain
        tols = dict(fo.ZERO_TOLS, **{fo.RULE_TOL[a]: 2.0 * v1[a], fo.RULE_TOL[b]: 2.0 * v1[b]})
        got, _ = _one(ctx, name, ds, y, hist, MAX_ITER, tols)
        assert got == (fo.RULE_STATUS[a], 1, n1), (name, a, b, got)
    for rule in fo.RULES:
        got, _ = _one(ctx, name, ds, y, hist, MAX_ITER, dict(fo.ZERO_TOLS, **{fo.RULE_TOL[rule]: np.inf}))
        assert got == (fo.RULE_STATUS[rule], 1, n1), (name, rule, got)
        # NaN compares false: the rule never fires, as in the oracle
        got, _ = _one(ctx, name, ds, y, hist, 3, dict(fo.ZERO_TOLS, **{fo.RULE_TOL[rule]: np.nan}))
        assert got == (po.TERM_MAXIT, 3, int(run.rows[2, 3])), (name, rule, got)
        _nan_report.append("a NaN tolerance never fires its rule (the fit runs to max_iter), as in both oracles")
    got, _ = _one(ctx, name, ds, y, hist, 3, {k: np.nan for k in fo.ZERO_TOLS})
    assert got == (po.TERM_MAXIT, 3, int(run.rows[2, 3])), (name, got)


# ---------------------------------------------------------------------------------------------------------------------
# several series per warp of the grouped kernel under one set of tolerances
# ---------------------------------------------------------------------------------------------------------------------
MIXED_ITER = 40


def mixed_batch(G):
    """Eight plain-class series (four warps' worth at G = 16, two at G = 8) of the recipe's lengths and the noisy ones."""
    base = ki.CELLS[f"g{G}_logistic_plain"]
    out = [ki._series(0, T, True, 40 + i) for i, T in enumerate(base.lengths[:4])]
    for i, T in enumerate(base.lengths[:4]):
        ds = ki._series(0, T, True, 50 + i)[0]
        out.append((ds, noisy_y(ds, 50 + i)))
    return out


def mixed_tolerances(runs, margin=1e-4):
    """One set of tolerances under which the oracle stops the series at different iterations under at least three
    different rules, every value up to each stop more than ``margin`` (relative) from its tolerance; and the oracle's
    (status, iters) per series under it."""
    for q in (0.3, 0.4, 0.5, 0.2, 0.6):
        tols = {}
        for r in fo.RULES:
            v = np.concatenate([run.values[r] for run in runs])
            tols[fo.RULE_TOL[r]] = float(np.quantile(v, q) if r != "ABSF" else np.quantile(v, q / 4))
        out, clear = [], True
        for run in runs:
            stop = (po.TERM_MAXIT, MIXED_ITER)
            for j in range(1, len(run.rows) + 1):
                for r in fo.RULES:
                    t, v = tols[fo.RULE_TOL[r]], run.values[r][j - 1]
                    clear &= abs(v - t) > margin * t
                fired = [r for r in fo.RULES if run.values[r][j - 1] < tols[fo.RULE_TOL[r]]]
                if fired:
                    stop = (fo.RULE_STATUS[fired[0]], j)
                    break
            out.append(stop)
        if clear and len({s for s, _ in out}) >= 3 and len({j for _, j in out}) >= 3:
            return tols, out
    raise AssertionError("no tolerance set separates the series")


def _mixed_runs(G):
    oopts = po.ProphetOptions()
    return [fo.StopRun(ds, y, oopts, MIXED_ITER, 5) for ds, y in mixed_batch(G)]


@pytest.mark.gpu
@pytest.mark.parametrize("G", (8, 16))
def test_mixed_warp_stops_each_series_on_its_own(ctx_env, G):
    ctx = ctx_env(f"g{G}")
    series = mixed_batch(G)
    runs = _mixed_runs(G)
    tols, want = mixed_tolerances(runs)
    b = ki._ragged(series)
    opts = batched.make_options(max_iter=MIXED_ITER, algorithm="LBFGS")
    for k, v in tols.items():
        setattr(opts, k, v)
    fb, tr = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=MIXED_ITER)
    vc = ctx.last_fit_variant_counts()
    assert vc[3, 0] == b.n and vc.sum() == b.n, vc
    for i, ((ds, y), run, (st, it)) in enumerate(zip(series, runs, want)):
        nev = int(run.rows[it - 1, 3])
        got = (int(fb.meta_i32[i, 4]), int(fb.meta_i32[i, 5]), int(fb.meta_i32[i, 6]))
        assert got == (st, it, nev), (G, i, got, st, it, nev)
        o1 = batched.make_options(max_iter=MIXED_ITER, algorithm="LBFGS")
        for k, v in tols.items():
            setattr(o1, k, v)
        f1, t1 = batched.fit_batch_trace_host(ctx, o1, ds, y, np.array([0, ds.size], np.int64), 0.0, 1.1,
                                              trace_cap=MIXED_ITER)
        assert f1.meta_i32[0].tobytes() == fb.meta_i32[i].tobytes(), (G, i)
        assert t1[0].tobytes() == tr[i].tobytes(), (G, i)
        fo.assert_trajectory_head(tr[i], it, run.rows, ("mixed", G, i), n_head=3)


# ---------------------------------------------------------------------------------------------------------------------
# warm start from each series' own optimum under the default tolerances
# ---------------------------------------------------------------------------------------------------------------------
def _default_tols():
    o = po.ProphetOptions()
    return {t: getattr(o, t) for t in fo.RULE_TOL.values()}


def warm_clear(run, stop, delta=1e-6):
    """Whether every rule's value at each iteration up to ``stop`` is more than delta (the df rules: their bracket's
    delta) from its default tolerance."""
    tols = _default_tols()
    for j in range(1, stop + 1):
        for r in fo.RULES:
            t, v = tols[fo.RULE_TOL[r]], run.values[r][j - 1]
            if abs(v - t) <= max(delta, run.delta(r, j)) * t:
                return False
    return True


@pytest.mark.gpu
@pytest.mark.parametrize("env", ("nt32", "g8"))
def test_warm_start_stops_where_the_oracle_does(ctx_env, env):
    ctx = ctx_env(env)
    name = "nt32_planes" if env == "nt32" else "g8_seasonal"
    c = CELLS[name]
    series = ki._cell_series(ki.CELLS[c.base], c.mode)[:len(ki.CELLS[c.base].lengths)]     # (not the year-long one)
    b = ki._ragged(series)
    opts = batched.make_options(**c.kw, algorithm="LBFGS")
    cold = batched.fit_batch_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    warm, tr = batched.fit_batch_warm_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, cold, trace_cap=64)
    vc = ctx.last_fit_variant_counts()
    assert vc[c.vcell] == b.n, vc
    codes, x = batched.warm_start(cold, cold.meta_i32[:, 1], cold.meta_i32[:, 3], cold.meta_i32[:, 4] >= 0)
    oopts = dataclasses.replace(oracle_options(name), **_default_tols())
    held = 0
    for i in range(b.n):
        assert codes[i] == L.WARM_USED and warm.warm[i] == L.WARM_USED, (env, i)
        a, e = b.offsets[i], b.offsets[i + 1]
        P = int(cold.meta_i32[i, 1]) + int(batched._seasonal_k(cold.meta_i32[i, 3])) + 3
        y = b.y[a:e].astype(np.float64)
        fr = wo.fit(b.ds[a:e], y, opts=dataclasses.replace(oopts, max_iter=10000), algorithm="LBFGS", init=x[i, :P])
        run = fo.StopRun(b.ds[a:e], y, oopts, max(fr.iters, 1), 5, init=x[i, :P])
        got = (int(warm.meta_i32[i, 4]), int(warm.meta_i32[i, 5]), int(warm.meta_i32[i, 6]))
        assert fr.ret in fo.RULE_STATUS.values() and got[0] in fo.RULE_STATUS.values(), (env, i, got, fr.ret)
        if fr.ret >= 0 and warm_clear(run, fr.iters):
            assert got == (fr.ret, fr.iters, fr.n_evals), (env, i, got, fr.ret, fr.iters, fr.n_evals)
            held += 1
    assert held >= b.n // 2, (env, held, b.n)
