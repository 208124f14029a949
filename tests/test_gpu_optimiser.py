"""GPU tests that pin the OPTIMISER (run with -m gpu on an H100), not just the cloud of points it ends in.

tests/test_gpu_parity.py holds the fitted forecasts to distribution-level tolerances, because Stan's loose
relative-gradient stop amplifies last-bit differences.  That leaves room for a wrong line-search or update
constant that still converges.  These tests close it from three sides:

  * trajectory: the (iteration, f_k, alpha_k, n_evals) rows of the kernel (pb200_fit_trace_host) against the
    numpy oracle's (stan_lbfgs(trace=...)): identical evaluation counts and f to ~1e-12 over the first
    iterations, and agreement for as long as both take the same decisions;
  * tight-stop mode: with the loose stops off both run until the objective stalls.  On the reference's objective
    (Laplace prior: kinks) L-BFGS has no unique end point -- the two CPU oracles differ by up to 5e-4 in objective --
    so the same spread is asserted; on a near-flat prior the same loops agree to ~1e-8;
  * arbiter: restarted from the GPU's optimum, the oracle's L-BFGS stops within a few iterations (the GPU did
    not stop early or somewhere else).

and fbprophet 0.5's Newton retry (newton_kernel.cuh) against the oracle's stan_newton.
"""
import os

import numpy as np
import pytest

from oracle import prophet_oracle as po
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, synth

pytestmark = pytest.mark.gpu

NS15 = 15 * 60 * 10**9


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
def ctxs():
    """name -> context: the grouped day-table kernel (8 and 16 lanes per series), the one-warp-per-series
    kernels (day table, rotation) and the default dispatch (small batch: 4 warps per series)."""
    c = {
        "g8": _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_GROUP=8, PB200_PLAIN_GROUP=1),
        "g16": _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_GROUP=16, PB200_PLAIN_GROUP=1),
        "tab32": _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_GROUP=0),
        "rot32": _ctx_with_env(PB200_LC0_MAX=1 << 30, PB200_NO_TAB=1),
        "default": L.Context(0),
    }
    yield c
    for v in c.values():
        v.close()


def _oracle_trace(ds, y, oopts):
    rows = []
    fr = po.fit(ds, y, opts=oopts, algorithm="LBFGS", trace=rows)
    return fr, np.array(rows).reshape(-1, 4)


def _common_prefix(a, b, n):
    k = 0
    while (k < n and a[k, 3] == b[k, 3] and abs(a[k, 1] - b[k, 1]) <= 1e-10 * max(1.0, abs(a[k, 1]))
           and abs(a[k, 2] - b[k, 2]) <= 1e-6 * abs(a[k, 2])):
        k += 1
    return k


@pytest.mark.parametrize("kernel", ["g8", "g16", "tab32", "rot32", "default"])
def test_lbfgs_trajectory_matches_oracle(ctxs, kernel):
    """Every accepted iteration's f_k, step length and evaluation count.  The first iterations are compared tightly
    (any wrong Wolfe / cubic-interpolation / two-loop constant shows there: the oracle's restatements agree with
    each other to 2e-16 at that point, tests/test_oracle_c.py); after that rounding differences grow smoothly
    until a line-search decision flips, and only the length of the common prefix is reported."""
    b = synth.config3(n=12)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    cap = 512
    fb, tr = batched.fit_batch_trace_host(ctxs[kernel], opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=cap)
    vc = ctxs[kernel].last_fit_variant_counts()
    if kernel in ("g8", "g16", "tab32"):
        assert vc[3, 6] == b.n
    elif kernel == "rot32":
        assert vc[1, 6] == b.n
    frac = []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr, rows = _oracle_trace(b.ds[a:e], b.y[a:e].astype(np.float64), oopts)
        n_gpu = int(fb.meta_i32[i, 5])
        assert n_gpu >= 1 and tr[i, min(n_gpu, cap) - 1, 0] == min(n_gpu, cap)      # one row per iteration, in order
        assert np.all(tr[i, min(n_gpu, cap):, 0] == 0)
        n = min(n_gpu, len(rows), cap)
        head = min(n, 6)
        g, o = tr[i], rows
        assert np.array_equal(g[:head, 3], o[:head, 3]), (kernel, i, g[:head, 3], o[:head, 3])       # evaluations
        assert np.all(np.abs(g[:head, 1] - o[:head, 1]) <= 1e-11 * np.maximum(1.0, np.abs(o[:head, 1]))), (kernel, i)
        assert np.all(np.abs(g[:head, 2] - o[:head, 2]) <= 1e-7 * np.abs(o[:head, 2])), (kernel, i)
        k = _common_prefix(g, o, n)
        assert k >= head
        frac.append(k / n)
    print(f"{kernel}: common trajectory prefix / iterations: median {np.median(frac):.2f}, min {np.min(frac):.2f}")
    assert np.median(frac) >= 0.05


@pytest.mark.parametrize("kernel", ["g8", "g16"])
@pytest.mark.parametrize("growth", ["logistic", "linear"])
def test_lbfgs_trajectory_plain_grouped_class(ctxs, kernel, growth):
    """The grouped kernel's class WITHOUT seasonality (config #4's short ragged series, the production path of a
    large batch of them): same trajectory check, plus the status / iteration count of runs short enough to be
    identical to the end."""
    b = synth.config4(n=24)
    opts, oopts = batched.make_options(growth=growth), po.ProphetOptions(growth=growth)
    cap = 256
    fb, tr = batched.fit_batch_trace_host(ctxs[kernel], opts, b.ds, b.y, b.offsets, 0.0, 1.1, trace_cap=cap)
    vc = ctxs[kernel].last_fit_variant_counts()
    assert vc[3, 0] == b.n and vc.sum() == b.n, vc
    frac, same_end = [], 0
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr, rows = _oracle_trace(b.ds[a:e], b.y[a:e].astype(np.float64), oopts)
        n_gpu = int(fb.meta_i32[i, 5])
        n = min(n_gpu, len(rows), cap)
        head = min(n, 6)
        g, o = tr[i], rows
        assert np.array_equal(g[:head, 3], o[:head, 3]), (kernel, i, g[:head, 3], o[:head, 3])
        assert np.all(np.abs(g[:head, 1] - o[:head, 1]) <= 1e-11 * np.maximum(1.0, np.abs(o[:head, 1]))), (kernel, i)
        assert np.all(np.abs(g[:head, 2] - o[:head, 2]) <= 1e-7 * np.abs(o[:head, 2])), (kernel, i)
        k = _common_prefix(g, o, n)
        assert k >= head
        frac.append(k / n)
        if k == n and n_gpu == len(rows):
            same_end += 1
            assert fb.meta_i32[i, 4] == fr.ret
            assert abs(fb.meta_f64[i, 3] - fr.neg_logp) <= 1e-9 * max(1.0, abs(fr.neg_logp))
    print(f"plain {kernel} {growth}: common prefix / iterations median {np.median(frac):.2f}; identical to the end: {same_end}/{b.n}")
    assert np.median(frac) >= 0.05


def _tight_opts(tau=0.05, **kw):
    o = batched.make_options(algorithm="LBFGS", changepoint_prior_scale=tau, max_iter=20000, **kw)
    o.tol_rel_grad = 0.0
    o.tol_rel_obj = 0.0
    o.tol_grad = 0.0
    o.tol_param = 0.0
    o.tol_obj = 1e-13
    return o


def _tight_oopts(tau=0.05, **kw):
    return po.ProphetOptions(tol_rel_grad=0.0, tol_rel_obj=0.0, tol_grad=0.0, tol_param=0.0, tol_obj=1e-13,
                             changepoint_prior_scale=tau, max_iter=20000, **kw)


@pytest.mark.parametrize("tau", [0.05, 1e3], ids=["laplace_prior_0.05", "near_flat_prior_1e3"])
@pytest.mark.parametrize("case", ["c3", "c4", "c2"])
def test_tight_stop_mode_against_oracle(ctxs, case, tau):
    """Stan's loose stops off (tol_rel_grad = tol_rel_obj = tol_grad = tol_param = 0, tol_obj = 1e-13): both sides
    iterate until the objective stalls or the line search fails.

    What this can and cannot pin.  With the reference's Laplace prior (tau = 0.05) the objective has kinks at
    delta_s = 0 and L-BFGS does NOT have a unique end point even at tight tolerances: the two CPU restatements of the
    oracle (numpy / C, same algorithm, different summation order) end 2e-4 (config #3) .. 5e-4 (config #4) apart in
    objective and up to 0.15 apart in parameters.  So the end-point tolerance that is TRUE for this algorithm is
    5e-3 relative in the objective -- the loop itself is pinned by the trajectory test above.  With a near-flat
    prior (tau = 1e3) the kinks are negligible and both runs go to the same smooth optimum: the objectives then
    agree to ~1e-8 (median) -- four orders tighter -- which is the statement that the two optimiser loops are the
    same algorithm.  (Parameters stay weakly determined along the flat directions of 25 changepoints, so the
    objective, not delta, is compared.)"""
    if case == "c3":
        b, kw, okw, ctx = synth.config3(n=8), {}, {}, ctxs["g8"]
    elif case == "c4":
        b, kw, okw, ctx = synth.config4(n=24), {}, {}, ctxs["default"]
    else:
        b, ctx = synth.config2(n=8), ctxs["default"]
        kw = {"growth": "linear", "yearly_seasonality": True}
        okw = {"growth": "linear", "yearly_seasonality": True}
    opts, oopts = _tight_opts(tau, **kw), _tight_oopts(tau, **okw)
    fb = batched.fit_batch_host(ctx, opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    fd = batched.fit_batch_host(ctx, batched.make_options(algorithm="LBFGS", changepoint_prior_scale=tau, **kw),
                                b.ds, b.y, b.offsets, 0.0, 1.1)
    rel = []
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        fr = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), opts=oopts, algorithm="LBFGS")
        fg = fb.meta_f64[i, 3]
        rel.append(abs(fg - fr.neg_logp) / max(1.0, abs(fr.neg_logp)))
        # iterating on past Stan's default stop never raises the objective
        assert fg <= fd.meta_f64[i, 3] + 1e-9 * max(1.0, abs(fg)), (case, tau, i)
        assert fb.meta_i32[i, 5] >= fd.meta_i32[i, 5]
    rel = np.array(rel)
    print(f"{case} tau={tau}: objective rel diff GPU vs oracle median {np.median(rel):.2e} max {rel.max():.2e}")
    if tau > 1.0:
        assert np.median(rel) <= 1e-6 and rel.max() <= 2e-2, rel
    else:
        assert np.median(rel) <= 2e-3 and rel.max() <= 5e-3, rel


def test_oracle_restarted_from_the_gpu_optimum_stops_at_once(ctxs):
    """SURVEY 8c's arbiter: from theta_gpu the oracle's own L-BFGS (default Stan tolerances) terminates within a few
    iterations without lowering the objective noticeably -- the GPU stopped where Stan's rules stop."""
    b = synth.config3(n=8)
    opts, oopts = batched.make_options(), po.ProphetOptions()
    fb = batched.fit_batch_host(ctxs["g8"], opts, b.ds, b.y, b.offsets, 0.0, 1.1)
    for i in range(b.n):
        a, e = b.offsets[i], b.offsets[i + 1]
        y = b.y[a:e].astype(np.float64)
        p = po.prepare(b.ds[a:e], y, 0.0, y.max() * 1.1, oopts)
        S, K = p.S, p.K
        th = np.concatenate(([fb.params[i, 0], fb.params[i, 1]], fb.params[i, 3:3 + S], [np.log(fb.params[i, 2])],
                             fb.params[i, 3 + fb.smax:3 + fb.smax + K]))
        err, f0, _ = po.neg_logp_grad(th, p)
        assert err == 0 and abs(f0 - fb.meta_f64[i, 3]) <= 1e-9 * abs(f0)
        x, f1, it, ret, ne = po.stan_lbfgs(lambda v: po.neg_logp_grad(v, p), th, oopts)
        assert ret >= 0 and it <= 12, (i, it, ret)
        assert f0 - f1 <= 2e-4 * abs(f0), (i, f0, f1)


def test_newton_only_matches_oracle_newton(ctxs):
    """newton_kernel.cuh against oracle stan_newton on short ragged series (config #4) and on two config-#3 series.
    Newton stops on |delta lp| < 1e-8, but on this objective it zig-zags across the Laplace kinks, so the two runs
    (Jacobi vs LAPACK eigenvectors, different summation order) end up to ~2e-5 relative apart in objective
    (numpy vs C oracle: 1e-6); stated tolerance 1e-4 relative, sigma_obs 1e-3 relative."""
    for b, n_take in ((synth.config4(n=6), 6), (synth.config3(n=2), 2)):
        opts = batched.make_options(algorithm="Newton")
        fb = batched.fit_batch_host(ctxs["default"], opts, b.ds, b.y, b.offsets, 0.0, 1.1)
        for i in range(n_take):
            a, e = b.offsets[i], b.offsets[i + 1]
            fr = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), algorithm="Newton")
            assert fb.meta_i32[i, 4] == L.ST_NEWTON == fr.ret
            assert np.array_equal(fb.tchange[i, :fr.prep.S], fr.prep.t_change)
            assert abs(fb.meta_f64[i, 3] - fr.neg_logp) <= 1e-4 * max(1.0, abs(fr.neg_logp)), (i, fb.meta_f64[i, 3], fr.neg_logp)
            assert abs(fb.params[i, 2] - fr.sigma_obs) <= 1e-3 * fr.sigma_obs
            fl = po.fit(b.ds[a:e], b.y[a:e].astype(np.float64), algorithm="LBFGS")
            assert fb.meta_f64[i, 3] <= fl.neg_logp + 1e-6      # Newton's end point is below L-BFGS's loose stop


def test_line_search_failure_gets_its_newton_retry(ctxs):
    """fbprophet 0.5 fit(): a series whose L-BFGS ends in a line-search failure (PyStan's RuntimeError) is fitted
    again with Newton from the same initial point and keeps its row (reference prophet_modeler.py:65-66, 81-85).
    Failures are rare under Stan's default tolerances (1 in 500k config-#4 series, synth.CONFIG4_LSFAIL_IDS), so the
    batch also runs with the loose stops off, where L-BFGS typically ends by failing to make progress at the optimum:
    every series that is -1 with the retry off must be 60 with it on, carrying the oracle's Newton objective."""
    parts = [synth.config4(n=500_000, lo=i, hi=i + 1) for i in synth.CONFIG4_LSFAIL_IDS] + [synth.config4(n=40)]
    ds = np.concatenate([p.ds for p in parts])
    y = np.concatenate([p.y for p in parts])
    lens = np.concatenate([np.diff(p.offsets) for p in parts])
    offs = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    n = offs.size - 1
    n_fail = 0
    for conv in (False, True):
        o_off = _tight_opts() if conv else batched.make_options(algorithm="LBFGS")
        o_on = _tight_opts() if conv else batched.make_options()
        o_on.algorithm = L.ALG_LBFGS_NEWTON
        fb0 = batched.fit_batch_host(ctxs["default"], o_off, ds, y, offs, 0.0, 1.1)
        fb1 = batched.fit_batch_host(ctxs["default"], o_on, ds, y, offs, 0.0, 1.1)
        assert np.all(fb1.meta_i32[:, 4] >= 0), fb1.meta_i32[:, 4]          # no row is dropped any more
        checked = 0
        for i in range(n):
            if fb0.meta_i32[i, 4] == L.ST_LSFAIL:
                n_fail += 1
                assert fb1.meta_i32[i, 4] == L.ST_NEWTON
                assert fb1.meta_i32[i, 5] > fb0.meta_i32[i, 5] and fb1.meta_i32[i, 6] > fb0.meta_i32[i, 6]   # both runs are counted
                if checked < 4:
                    a, e = offs[i], offs[i + 1]
                    fn = po.fit(ds[a:e], y[a:e].astype(np.float64), algorithm="Newton")
                    assert abs(fb1.meta_f64[i, 3] - fn.neg_logp) <= 1e-4 * max(1.0, abs(fn.neg_logp)), (i, fb1.meta_f64[i, 3], fn.neg_logp)
                    checked += 1
            else:
                assert fb1.meta_i32[i, 4] == fb0.meta_i32[i, 4] and np.array_equal(fb1.params[i], fb0.params[i])
    assert n_fail >= 1
