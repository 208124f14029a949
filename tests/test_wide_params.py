"""Models wider than 64 parameters through every path that can fit them (the GPU tests run with -m gpu on an H100).

P = S + K + 3 reaches 65 .. 67 with yearly + weekly + daily seasonality (K = 34) and 28 .. 30 changepoints, the most the
options admit.  A warp's vector code holds up to three elements per lane there, where everything below holds two, so
the tests fit mask-7 histories (12-hour steps over 800 days) at 27 changepoints (P = 64, the control) and 28 .. 30:

  * L-BFGS on all eight mask-7 fit_kernel instances (both CTA widths, both growths, stored planes and rotation), held
    to the oracle like tests/test_kernel_instances.py: objective and gradient, the first six iterations, changepoints,
    status and iteration count;
  * schedule independence: a P = 67 series fitted after another in the same persistent CTA gives the bytes it gives
    alone;
  * fbprophet's Newton run with 28 .. 30 changepoints on weekly + daily (P = 45 .. 47) and mask-7 series, held per
    iteration as tests/test_newton_steps.py, and as the retry of a P = 67 series whose L-BFGS run ends in a line-search
    failure.
"""
import dataclasses
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import fit_oracle as fo  # noqa: E402
import test_kernel_instances as ki  # noqa: E402
import test_newton_steps as ns  # noqa: E402
from oracle import c_oracle as co
from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched

NCPS = (27, 28, 29, 30)                # P = 64 (control), 65, 66, 67
# (context, logistic, regular grid) -> the fit_kernel instance's variant (REG 1: rotation on the regular grid)
INSTANCES = [(env, logi, reg) for env in ("nt32", "nt128") for logi in (0, 1) for reg in (False, True)]
# P = 67 histories whose L-BFGS runs end in a line-search failure under the tight stops below (numpy and C oracles)
LSFAIL = [(7, 801, False, seed) for seed in (42, 44, 46)]


def _wide_series(regular, seed):
    return ki._series(7, 1601, True, seed) if regular else ki._series(7, 801, False, seed)


def _tight(opts):
    opts.tol_rel_grad = opts.tol_rel_obj = opts.tol_grad = opts.tol_param = 0.0
    opts.tol_obj = 1e-13
    return opts


@pytest.fixture(scope="module")
def ctx_env():
    cache = {}

    def get(name, **extra):
        key = (name, tuple(sorted(extra.items())))
        if key not in cache:
            cache[key] = fo.ctx_with_env(**ki.ENV[name], **extra)
        return cache[key]

    yield get
    for c in cache.values():
        c.close()


def test_wide_series_have_the_widths_they_claim():
    for ncp in NCPS:
        for regular in (False, True):
            ds, y = _wide_series(regular, 3)
            p = po.prepare(ds, y.astype(np.float64), 0.0, 1.1 * y.max(), po.ProphetOptions(n_changepoints=ncp))
            assert ki._oracle_mask(p) == 7 and ki._is_regular(ds) == regular
            assert p.S + p.K + 3 == ncp + 37
    for rec in LSFAIL:
        ds, y = ki._series(*rec)
        p = po.prepare(ds, y.astype(np.float64), 0.0, 1.1 * y.max(), po.ProphetOptions(n_changepoints=30))
        assert p.S + p.K + 3 == 67


@pytest.mark.gpu
@pytest.mark.parametrize("ncp", NCPS)
@pytest.mark.parametrize("env,logi,regular", INSTANCES)
def test_wide_lbfgs_matches_oracle(ctx_env, env, logi, regular, ncp):
    growth = "logistic" if logi else "linear"
    ctx = ctx_env(env)
    b = ki._ragged([_wide_series(regular, 10 + s) for s in range(2)])
    kw = dict(growth=growth, n_changepoints=ncp)
    oopts = po.ProphetOptions(**kw)
    vcell = (1 if regular else 0, 7)
    th, preps = fo.thetas(b, oopts, L.get_layout(batched.make_options(**kw)), np.random.RandomState(11))
    f, g, mi = batched.objective_host(ctx, batched.make_options(**kw), b.ds, b.y, b.offsets, 0.0, 1.1, th)
    vc = ctx.last_fit_variant_counts()
    assert vc[vcell] == b.n and vc.sum() == b.n, vc
    for i, (p, t) in enumerate(preps):
        assert t.size == ncp + 37
        err, fo_, go = po.neg_logp_grad(t, p)
        assert err == 0 and mi[i, 4] == 0
        assert abs(f[i] - fo_) <= 1e-10 * max(1.0, abs(fo_)), (i, f[i], fo_)
        assert np.max(np.abs(g[i, :t.size] - go)) <= 1e-8 * max(1.0, np.max(np.abs(go))), i
    o6 = batched.make_options(**kw, max_iter=6, algorithm="LBFGS")
    fb, tr = batched.fit_batch_trace_host(ctx, o6, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=8)
    vc = ctx.last_fit_variant_counts()
    assert vc[vcell] == b.n and vc.sum() == b.n, vc
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr, rows = fo.oracle_rows(b.ds[a:e], b.y[a:e].astype(np.float64), dataclasses.replace(oopts, max_iter=6))
        S = fr.prep.S
        what = (env, growth, regular, ncp, i)
        assert np.array_equal(fb.tchange[i, :S], fr.prep.t_change) and np.all(fb.tchange[i, S:] == 0.0), what
        n_gpu = int(fb.meta_i32[i, 5])
        fo.assert_trajectory_head(tr[i], n_gpu, rows, what, n_head=3)
        head = min(n_gpu, len(rows), 6)
        gk, ok = tr[i, :head], rows[:head]
        assert np.array_equal(gk[:, 0], ok[:, 0]) and np.array_equal(gk[:, 3], ok[:, 3]), (what, gk, ok)
        assert np.all(np.abs(gk[:, 1] - ok[:, 1]) <= 1e-9 * np.maximum(1.0, np.abs(ok[:, 1]))), (what, gk, ok)
        assert np.all(np.abs(gk[:, 2] - ok[:, 2]) <= 1e-7 * np.abs(ok[:, 2])), (what, gk, ok)
        assert (fb.meta_i32[i, 4], n_gpu) == (fr.ret, fr.iters), (what, fb.meta_i32[i], fr.ret, fr.iters)


@pytest.mark.gpu
@pytest.mark.parametrize("env", ("nt32", "nt128"))
def test_wide_fit_does_not_depend_on_its_neighbour(ctx_env, env):
    """One CTA for the whole launch: B fitted after A in the same slot gives the bytes B gives alone."""
    ctx = ctx_env(env, PB200_FIT_GRID_MAX=1)
    A, B = _wide_series(False, 21), _wide_series(False, 22)
    opts = batched.make_options(n_changepoints=30)
    out = []
    for series in ([A, B], [B]):
        b = ki._ragged(series)
        fb, tr = batched.fit_batch_trace_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=64)
        assert ctx.last_fit_variant_counts()[0, 7] == b.n
        out.append((fb, tr))
    (f2, t2), (f1, t1) = out
    assert f1.meta_i32[0, 1] + fo.seasonal_k(7) + 3 == 67
    for name in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64"):
        assert getattr(f2, name)[1].tobytes() == getattr(f1, name)[0].tobytes(), name
    assert t2[1].tobytes() == t1[0].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("k", (1, 3))
@pytest.mark.parametrize("ncp", (28, 29, 30))
def test_wide_newton_steps_match_both_oracles(gpu_ctx, ncp, k):
    """Every series is fitted, whatever its own P: weekly + daily (P = ncp + 17) beside mask 7 (P = ncp + 37)."""
    series = [ki._series(6, 721, True, 50 + ncp), ki._series(6, 45, False, 51), _wide_series(False, 52),
              _wide_series(True, 53)]
    b = ki._ragged(series)
    extra = {"n_changepoints": ncp}
    fb = batched.fit_batch_host(gpu_ctx, batched.make_options(max_iter=k, algorithm="Newton", **extra), b.ds, b.y,
                                b.offsets, 0.0, 1.1)
    frs, th, f, info = ns._oracles(b, "logistic", "multiplicative", extra, k)
    assert sorted(int(m) for m in fb.meta_i32[:, 3]) == [6, 6, 7, 7]
    for i in range(b.n):
        fo.assert_newton_row(fb, i, frs[i], th[i], f[i], info[i], ns._measured, ("wide newton", ncp, k, i))
    full = batched.fit_batch_host(gpu_ctx, batched.make_options(algorithm="Newton", **extra), b.ds, b.y, b.offsets,
                                  0.0, 1.1)
    assert np.all(full.meta_i32[:, 4] == L.ST_NEWTON) and np.all(full.params[:, 2] > 0), full.meta_i32


@pytest.mark.gpu
def test_wide_line_search_failure_gets_its_newton_retry(gpu_ctx):
    """Past a few hundred iterations the GPU's L-BFGS path is its own (summation order), so of the oracles' failing
    series at least one must fail on the GPU too; every one that does ends as the Newton run, counted with both runs."""
    b = ki._ragged([ki._series(*rec) for rec in LSFAIL])
    kw = dict(n_changepoints=30, max_iter=20000)
    lb = batched.fit_batch_host(gpu_ctx, _tight(batched.make_options(algorithm="LBFGS", **kw)), b.ds, b.y, b.offsets,
                                0.0, 1.1)
    both = batched.fit_batch_host(gpu_ctx, _tight(batched.make_options(algorithm="LBFGS+Newton", **kw)), b.ds, b.y,
                                  b.offsets, 0.0, 1.1)
    nw = batched.fit_batch_host(gpu_ctx, batched.make_options(algorithm="Newton", **kw), b.ds, b.y, b.offsets, 0.0, 1.1)
    assert np.all(nw.meta_i32[:, 4] == L.ST_NEWTON), nw.meta_i32
    failed = np.flatnonzero(lb.meta_i32[:, 4] == L.ST_LSFAIL)
    assert failed.size >= 1, lb.meta_i32
    for i in range(b.n):
        assert lb.meta_i32[i, 1] + fo.seasonal_k(int(lb.meta_i32[i, 3])) + 3 == 67
        if i not in failed:
            assert both.meta_i32[i].tobytes() == lb.meta_i32[i].tobytes()
            continue
        # both runs are counted; the retry starts from stan_init again, so its model is the Newton-only run's
        assert both.meta_i32[i, 4] == L.ST_NEWTON, both.meta_i32[i]
        assert both.meta_i32[i, 5] == lb.meta_i32[i, 5] + nw.meta_i32[i, 5], (both.meta_i32[i], lb.meta_i32[i], nw.meta_i32[i])
        assert both.meta_i32[i, 6] == lb.meta_i32[i, 6] + nw.meta_i32[i, 6], (both.meta_i32[i], lb.meta_i32[i], nw.meta_i32[i])
        assert both.params[i].tobytes() == nw.params[i].tobytes()
        fg = both.meta_f64[i, 3]
        assert fg <= lb.meta_f64[i, 3] + 1e-9 * max(1.0, abs(fg)), (i, fg, lb.meta_f64[i, 3])
    i = int(failed[0])
    a, e = b.offsets[i], b.offsets[i + 1]
    fr = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=po.ProphetOptions(n_changepoints=30), algorithm="Newton")
    assert abs(both.meta_f64[i, 3] - fr.neg_logp) <= 1e-4 * max(1.0, abs(fr.neg_logp)), (both.meta_f64[i, 3], fr.neg_logp)


def test_wide_line_search_failure_on_the_oracles():
    """The series the retry test uses fail their tight-stop L-BFGS runs on both CPU oracles."""
    o = co.options()
    o.n_changepoints, o.max_iter, o.algorithm = 30, 20000, co.ALG_LBFGS
    o.tol_rel_grad = o.tol_rel_obj = o.tol_grad = o.tol_param = 0.0
    o.tol_obj = 1e-13
    for rec in LSFAIL:
        ds, y = ki._series(*rec)
        y = y.astype(np.float64)
        fr = po.fit(ds, y, opts=po.ProphetOptions(n_changepoints=30, max_iter=20000, tol_rel_grad=0.0, tol_rel_obj=0.0,
                                                  tol_grad=0.0, tol_param=0.0, tol_obj=1e-13), algorithm="LBFGS")
        _, _, info = co.fit_batch(ds, y, np.array([0, ds.size]), 0.0, 1.1, o)
        assert fr.ret == po.TERM_LSFAIL and info[0, 0] == -1, (rec, fr.ret, info[0])
