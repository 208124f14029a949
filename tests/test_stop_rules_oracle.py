"""The stop-rule brackets of tests/test_gpu_stop_rules.py checked without a GPU.

The numpy oracle's ``crit`` record gives, per accepted iteration, what Stan's five convergence tests compare with their
tolerances.  Here: the record leaves the fit's bits alone and agrees with the trace; the C oracle (which shares no code
with the numpy one and has a fixed history of 5) gives the bracketed outcome at every record low of every series the GPU
module uses; each series has the property it is chosen for; and a NaN or infinite tolerance does in both oracles what
the GPU module expects of the kernels.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import fit_oracle as fo  # noqa: E402
import test_gpu_stop_rules as sr  # noqa: E402
from oracle import c_oracle as co
from oracle import prophet_oracle as po
from time_series_spark_b200 import synth


def _c_opts(name, max_iter, tols):
    kw = sr.CELLS[name].kw
    sw = {True: 1, False: 0}
    o = co.options(growth=kw["growth"], seasonality_mode=kw["seasonality_mode"],
                   yearly=sw.get(kw.get("yearly_seasonality"), -1), weekly=sw.get(kw.get("weekly_seasonality"), -1),
                   daily=sw.get(kw.get("daily_seasonality"), -1))
    o.n_changepoints = kw.get("n_changepoints", 25)
    o.max_iter, o.algorithm = max_iter, co.ALG_LBFGS
    for k, v in tols.items():
        setattr(o, k, v)
    return o


def _c_outcome(name, ds, y, max_iter, tols):
    _, _, info = co.fit_batch(ds, np.asarray(y, np.float64), np.array([0, ds.size]), 0.0, 1.1,
                              _c_opts(name, max_iter, tols))
    return int(info[0, 0]), int(info[0, 1]), int(info[0, 2])


def test_crit_leaves_the_fit_alone_and_agrees_with_the_trace():
    b = synth.config3(n=3)
    series = [(b.ds[b.offsets[i]:b.offsets[i + 1]], b.y[b.offsets[i]:b.offsets[i + 1]]) for i in range(b.n)]
    series += [s[:2] for s in sr.cell_series("nt32_planes")]
    for ds, y in series:
        y = y.astype(np.float64)
        for opts in (po.ProphetOptions(max_iter=12, **fo.ZERO_TOLS), po.ProphetOptions()):
            t0, t1, crit = [], [], []
            a = po.fit(ds, y, opts=opts, algorithm="LBFGS", trace=t0)
            c = po.fit(ds, y, opts=opts, algorithm="LBFGS", trace=t1, crit=crit)
            assert a.theta.tobytes() == c.theta.tobytes() and t0 == t1
            assert (a.neg_logp, a.iters, a.ret, a.n_evals) == (c.neg_logp, c.iters, c.ret, c.n_evals)
            cr, rows = np.array(crit), np.array(t1)
            assert len(crit) == len(t1) == a.iters and np.array_equal(cr[:, 0], rows[:, 0])
            f = rows[:, 1]
            assert np.array_equal(cr[1:, 1], np.abs(f[:-1] - f[1:]))
            assert np.array_equal(cr[1:, 2], np.maximum(np.abs(f[:-1]), np.maximum(np.abs(f[1:]), 1.0)))
            assert np.array_equal(cr[:, 5], np.maximum(np.abs(f), 1.0))
            assert np.all(cr[:, 1:] >= 0.0) and np.all(np.isfinite(cr))
            assert np.all(f[1:] < f[:-1]) and cr[0, 1] > 0.0          # each accepted step lowers f (StopRun.f)


@pytest.mark.parametrize("name", list(sr.CELLS))
def test_c_oracle_gives_every_bracketed_outcome(name):
    """Every record low up to MAX_ITER of every rule, on each of the cell's series at history 5, both sides of its
    bracket at the delta the GPU test holds the kernels to."""
    oopts = sr.oracle_options(name)
    n = 0
    for ds, y, _ in sr.cell_series(name):
        run = fo.StopRun(ds, y, oopts, sr.MAX_ITER, 5)
        assert _c_outcome(name, ds, y, sr.MAX_ITER, fo.ZERO_TOLS) == (run.fr.ret, run.fr.iters, run.fr.n_evals)
        for rule in fo.RULES:
            for j in run.record_lows(rule):
                for side in (+1, -1):
                    tols, want = run.bracket(rule, j, side, run.delta(rule, j))
                    got = _c_outcome(name, ds, y, j, tols)
                    assert got == want, (name, rule, j, side, got, want)
                    n += 1
    assert n >= 40, n


@pytest.mark.parametrize("name", list(sr.CELLS))
def test_cell_series_have_their_properties(name):
    oopts = sr.oracle_options(name)
    series = sr.cell_series(name)
    floor = sr.CELLS[name].floor is not None
    assert [h for _, _, h in series] == [5, 3, 1] + [5] * floor
    assert floor or name == "nt32_linear_additive"
    at2 = False
    for s, (ds, y, hist) in enumerate(series):
        p = po.prepare(ds, y.astype(np.float64), 0.0, 1.1 * y.max(), oopts)
        assert p.T == ds.size
        if sr.CELLS[name].base is None:
            assert p.S + p.K + 3 == 67
        run = fo.StopRun(ds, y, oopts, sr.MAX_ITER, hist)
        assert run.fr.iters == sr.MAX_ITER and run.fr.ret == po.TERM_MAXIT, (name, s, run.fr.ret)
        targets = {r: run.targets(r) for r in fo.RULES}
        assert all(targets[r][:1] == [1] for r in fo.RULES), (name, s)         # iteration 1, the reset path
        at2 |= any(2 in t for t in targets.values())
        if s < 3:                                                               # the ring buffer has wrapped
            assert any(t[-1] > hist for t in targets.values()), (name, s, targets)
    assert at2, name
    # the floor series: some record low at which max(|f|, 1)'s floor or the sign of f decides the scale
    if floor:
        ds, y, hist = series[3]
        assert sr.floor_crossings(fo.StopRun(ds, y, oopts, sr.MAX_ITER, hist)), name


def test_nan_never_fires_and_inf_fires_at_once_in_both_oracles():
    ds, y, _ = sr.cell_series("nt32_planes")[0]
    run = fo.StopRun(ds, y, sr.oracle_options("nt32_planes"), 3, 5)
    for rule, tol in fo.RULE_TOL.items():
        for v, want in ((np.nan, (po.TERM_MAXIT, 3)), (np.inf, (fo.RULE_STATUS[rule], 1))):
            tols = dict(fo.ZERO_TOLS, **{tol: v})
            fr = po.fit(ds, y.astype(np.float64), opts=po.ProphetOptions(max_iter=3, **tols), algorithm="LBFGS")
            assert (fr.ret, fr.iters) == want, (rule, v, fr.ret, fr.iters)
            assert _c_outcome("nt32_planes", ds, y, 3, tols) == want + (int(run.rows[want[1] - 1, 3]),), (rule, v)


@pytest.mark.parametrize("G", (8, 16))
def test_mixed_tolerances_separate_the_series(G):
    runs = sr._mixed_runs(G)
    tols, want = sr.mixed_tolerances(runs)
    for (ds, y), run, (st, it) in zip(sr.mixed_batch(G), runs, want):
        fr = po.fit(ds, y.astype(np.float64), opts=po.ProphetOptions(max_iter=sr.MIXED_ITER, **tols), algorithm="LBFGS")
        assert (fr.ret, fr.iters, fr.n_evals) == (st, it, int(run.rows[it - 1, 3]))
        _, _, info = co.fit_batch(ds, y.astype(np.float64), np.array([0, ds.size]), 0.0, 1.1,
                                  _c_opts_default(sr.MIXED_ITER, tols))
        assert tuple(info[0, :3]) == (st, it, fr.n_evals)


def _c_opts_default(max_iter, tols):
    o = co.options()
    o.max_iter, o.algorithm = max_iter, co.ALG_LBFGS
    for k, v in tols.items():
        setattr(o, k, v)
    return o
