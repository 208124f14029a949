"""GPU tests of the backtest's three kernels (csrc/cv_kernel.cuh, DESIGN §9) against the oracle's restatement of
fbprophet.diagnostics, beyond the one batch of test_gpu_backtest.py: cv_plan_kernel exactly on a batch past its
grid-stride loop (random series, the named cases, the golden fixture's groups with duplicate timestamps, 0- and 1-row
series, series 1 ns either side of every seasonality threshold, durations near int64's range); cv_gather_kernel bit for
bit on int32 / float32 / float64 y past its stride loop; cv_metrics_kernel over every window width with and without
intervals, and past its stride loop; the whole backtest on float y and other (horizon, period, initial) triples."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import backtest_oracle as bo  # noqa: E402
from oracle import mc_stream  # noqa: E402
from oracle import prophet_oracle as po  # noqa: E402
from test_backtest_oracle import CASES  # noqa: E402
from test_backtest_sweeps import (D, H, INT64_MAX, MINUTE, RWS, UNITS, expected_plan, random_rows,  # noqa: E402
                                  random_series)

pytestmark = pytest.mark.gpu

FLOOR, CAPM = 0.0, 1.1
# (horizon, period, initial) of the plan sweep: the job's default, period above the horizon with a 1 ns initial window,
# period equal to the horizon off every step grid, minute scale, nanosecond scale
TRIPLES = [(D, D // 2, 3 * D), (D, 3 * D // 2 + 7, 1), (6 * H + 1, 6 * H + 1, 2 * D + 3),
           (90 * MINUTE, 37 * MINUTE + 11, 5 * H), (7, 3, 1)]
DEV = {}                 # largest deviations measured, printed as the tests run


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pack(series):
    off = np.concatenate(([0], np.cumsum([s.size for s in series]))).astype(np.int64)
    ds = np.concatenate(series).astype(np.int64) if off[-1] else np.zeros(0, np.int64)
    return ds, off


def _threshold_series(rng):
    """Series 1 ns either side of (and on) the 2-, 14- and 730-day spans and the 1- and 7-day smallest steps, at
    lengths under one warp, on it, and not a multiple of it, the smallest step at a random lane."""
    out = []
    t0 = 1_500_000_000 * 10**9
    for n in (2, 5, 31, 32, 33, 45, 64, 77):
        for span in (2 * D, 14 * D, 730 * D):
            for d in (-1, 0, 1):
                s = np.linspace(0, span + d, n).astype(np.int64)
                s[-1] = span + d
                out.append(t0 + s)
        for step, base in ((D, 2 * D), (7 * D, 12 * D), (D, 12 * D)):     # 12 days: 730 days from 62 rows
            for d in (-1, 0, 1):
                steps = np.full(n - 1, base, np.int64)
                steps[rng.randint(n - 1)] = step + d
                out.append(t0 + np.concatenate(([0], np.cumsum(steps))))
    return out


def _golden_groups(gi):
    return [np.sort(gi["ds_ns"][gi["dim_id"] == d].astype(np.int64), kind="stable") for d in np.unique(gi["dim_id"])]


@pytest.fixture(scope="module")
def plan_batch(sms, golden_input):
    """More than sms * 128 series (two grid-stride rounds of the plan kernel at 8 warps per CTA and sms * 16 CTAs)."""
    rng = np.random.RandomState(11)
    series = [np.zeros(0, np.int64), np.array([1_600_000_000 * 10**9], np.int64)]
    series += [np.sort(c[0]) for c in CASES.values()] + _golden_groups(golden_input) + _threshold_series(rng)
    series.insert(len(series) // 2, np.zeros(0, np.int64))
    while len(series) < sms * 128 + 1500:
        unit = UNITS[rng.randint(len(UNITS))]
        series.append(random_series(rng, unit, (D, H, MINUTE, 7)[rng.randint(4)]))
    series.append(np.zeros(0, np.int64))
    return series


def _plan(ctx, ds, off, hz, per, ini, **switches):
    import torch
    from time_series_spark_b200 import batched
    return batched.cv_plan_device(ctx, batched.make_options(**switches), torch.from_numpy(ds).cuda(), off, hz, per, ini)


def _check_plan(plan, series, off, hz, per, ini):
    """Every series exactly: n_cutoffs, cutoffs, hist_end, win_end, err bits; returns the outcome counts."""
    from time_series_spark_b200 import _lib as L
    cut, he, we = (x.cpu().numpy() for x in (plan.cutoff, plan.hist_end, plan.win_end))
    ps = plan.pair_series.cpu().numpy()
    counts = {"err": 0, "few": 0, "cutoffs": 0}
    for i, s in enumerate(series):
        c, err = expected_plan(s, hz, per, ini)
        p0, p1 = plan.pair_off[i], plan.pair_off[i + 1]
        where = (i, s.size, hz, per, ini)
        assert int(plan.n_cutoffs[i]) == c.size and int(plan.err[i]) == err, (where, plan.n_cutoffs[i], plan.err[i], err)
        assert cut[p0:p1].tolist() == c.tolist(), where
        assert (ps[p0:p1] == i).all(), where
        assert (he[p0:p1] - off[i]).tolist() == np.searchsorted(s, c, side="right").tolist(), where
        assert (we[p0:p1] - off[i]).tolist() == np.searchsorted(s, c + hz, side="right").tolist(), where
        counts["err"] += err in (L.CV_ERR_HORIZON, L.CV_ERR_INITIAL)
        counts["few"] += err == L.CV_ERR_FEW
        counts["cutoffs"] += c.size > 0
    return counts


@pytest.mark.parametrize("triple", TRIPLES, ids=["default", "period_gt_horizon", "period_eq_horizon", "minutes", "ns"])
def test_plan_matches_oracle_past_the_stride_loop(gpu_ctx, sms, plan_batch, triple):
    assert len(plan_batch) > 8 * 16 * sms           # warps per CTA x CTAs: the stride loop runs a second round
    ds, off = _pack(plan_batch)
    plan = _plan(gpu_ctx, ds, off, *triple)
    counts = _check_plan(plan, plan_batch, off, *triple)
    assert counts["cutoffs"] > 1000 and counts["err"] > 100, counts
    print(f"plan {triple}: {counts}, {plan.n_pairs} cutoffs")


@pytest.mark.parametrize("switch", ["auto", True, False, "mixed"])
def test_plan_mask_matches_oracle(gpu_ctx, plan_batch, switch):
    sw = ("auto", True, False) if switch == "mixed" else (switch,) * 3
    names = ("yearly_seasonality", "weekly_seasonality", "daily_seasonality")
    ds, off = _pack(plan_batch)
    plan = _plan(gpu_ctx, ds, off, *TRIPLES[0], **dict(zip(names, sw)))
    opts = po.ProphetOptions(**dict(zip(names, sw)))
    want = np.array([bo.seasonality_mask(s, opts) if s.size else 0 for s in plan_batch])
    bad = np.flatnonzero(plan.mask != want)
    assert bad.size == 0, [(int(i), plan_batch[i].size, int(plan.mask[i]), int(want[i])) for i in bad[:5]]
    if switch == "auto":                           # every mask auto can give (yearly + daily without weekly: none)
        assert set(np.unique(want).tolist()) == {0, 1, 2, 3, 4, 6, 7}


@pytest.mark.parametrize("epoch", [946_684_800 * 10**9, -2_208_988_800 * 10**9], ids=["2000s", "1900s"])
def test_plan_at_durations_near_int64(gpu_ctx, epoch):
    """initial, horizon or period of ~100 000 days up to INT64_MAX: first + initial, last - horizon and prev - period
    leave int64.  The kernel must report fbprophet's plan (the oracle's Python integers), not a wrapped one."""
    series = [epoch + np.arange(0, n * D + 1, H, dtype=np.int64) for n in (1, 3, 10)]
    series += [epoch + np.array([0, 5 * D, 9 * D, 9 * D, 40 * D], np.int64), np.array([epoch], np.int64)]
    ds, off = _pack(series)
    big = (100_000 * D, 106_751 * D, INT64_MAX)
    triples = [(D, D // 2, b) for b in big] + [(b, D // 2, D) for b in big] + [(D, b, D) for b in big] + \
              [(D, b, 1) for b in big] + [(b, b, b) for b in big] + [(D, D // 2, 3 * D)]
    for t in triples:
        _check_plan(_plan(gpu_ctx, ds, off, *t), series, off, *t)


# ---- gather ---------------------------------------------------------------------------------------------------------
def _y_values(rng, n, dtype):
    """Values whose bits a conversion would change or lose: -0.0, subnormals, NaN payloads, negatives, fractions."""
    if dtype == np.int32:
        return rng.randint(-2**31, 2**31 - 1, n, dtype=np.int64).astype(np.int32)
    y = (rng.randn(n) * 10 ** rng.uniform(-3, 3, n)).astype(dtype)
    fi = np.finfo(dtype)
    special = np.array([-0.0, fi.smallest_subnormal, -fi.smallest_subnormal * 3, fi.tiny / 2, -1.5, 0.1, fi.max],
                       dtype)
    k = rng.randint(0, n, 200)
    y[k] = special[rng.randint(0, special.size, k.size)]
    ui = np.uint32 if dtype == np.float32 else np.uint64
    nan = np.array([0x7FC00123 if dtype == np.float32 else 0x7FF8000000012345], ui).view(dtype)
    y[rng.randint(0, n, 20)] = nan[0]
    return y


@pytest.mark.parametrize("dtype", [np.int32, np.float32, np.float64], ids=["int32", "float32", "float64"])
def test_gather_bit_for_bit_past_the_stride_loop(gpu_ctx, sms, dtype):
    import torch
    from time_series_spark_b200 import _lib as L
    from time_series_spark_b200 import batched
    rng = np.random.RandomState(5)
    lens = rng.randint(2, 700, 400)
    off = np.concatenate(([0], np.cumsum(lens))).astype(np.int64)
    ds = np.concatenate([t + np.sort(rng.randint(0, 10**12, n)) for t, n in zip(rng.randint(0, 10**15, lens.size), lens)])
    y = _y_values(rng, int(off[-1]), dtype)
    # pairs: a history end and a window end per (series, cutoff), in plan order
    pser = np.repeat(np.arange(lens.size), 3).astype(np.int32)
    he = off[pser] + 1 + (rng.rand(pser.size) * (lens[pser] - 1)).astype(np.int64)
    we = he + 1 + (rng.rand(pser.size) * np.minimum(off[pser + 1] - he - 1, 40)).astype(np.int64)
    we = np.minimum(we, off[pser + 1])
    he = np.minimum(he, we - 1)
    n = sms * 32 + 777                                  # entries: more than the grid's sms * 32 CTAs
    pairs = rng.randint(0, pser.size, n).astype(np.int64)
    hist = he[pairs] - off[pser[pairs]]
    fit_off = np.concatenate(([0], np.cumsum(hist))).astype(np.int64)
    hmax = int((we - he)[pairs].max())
    assert n > sms * 32 and hist.max() > 256 and (we - he)[pairs].min() < hmax
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()     # noqa: E731
    d = {k: cu(v) for k, v in dict(ds=ds, y=y, off=off, pser=pser, he=he, we=we, pairs=pairs, fit_off=fit_off).items()}
    ds_out = torch.full((int(fit_off[-1]),), -1, dtype=torch.int64, device="cuda")
    y_out = torch.full((int(fit_off[-1]),), 7, dtype=d["y"].dtype, device="cuda")
    fut = torch.full((n, hmax), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    L.check(L.load().pb200_cv_gather_device(gpu_ctx.handle, d["ds"].data_ptr(), d["y"].data_ptr(), batched._y_dtype(d["y"]),
                                            d["off"].data_ptr(), d["pser"].data_ptr(), d["he"].data_ptr(),
                                            d["we"].data_ptr(), d["pairs"].data_ptr(), n, d["fit_off"].data_ptr(), hmax,
                                            ds_out.data_ptr(), y_out.data_ptr(), fut.data_ptr()), "pb200_cv_gather_device")
    gpu_ctx.synchronize()
    src = np.concatenate([np.arange(off[pser[p]], he[p]) for p in pairs])
    assert np.array_equal(ds_out.cpu().numpy(), ds[src])
    assert y_out.cpu().numpy().tobytes() == y[src].tobytes()
    j = np.arange(hmax)[None, :]
    want_fut = ds[np.minimum(he[pairs][:, None] + j, we[pairs][:, None] - 1)]
    assert np.array_equal(fut.cpu().numpy(), want_fut)


# ---- metrics --------------------------------------------------------------------------------------------------------
def _metric_rows(rng, n_series, empty_every=7):
    """Row sets of n_series series (every empty_every-th empty, some of one row), rows shuffled so that series
    interleave; returns the per-row arrays and each series' rows in their given order."""
    parts = []
    for s in range(n_series):
        if s % empty_every == 3:
            continue
        n = 1 if s % empty_every == 5 else int(rng.choice([2, 4, 9, 10, 20, 33, 100]))
        h, y, yhat, lo, hi = random_rows(rng, n, ties=bool(s % 2), intervals=True)
        if s % 11 == 0:
            y[rng.randint(n)] = (0.0, -0.0, 5e-9, 1e-8)[s % 4]
        parts.append((np.full(n, s, np.int64), h, y, yhat, lo, hi))
    cols = [np.concatenate([p[k] for p in parts]) for k in range(6)]
    perm = rng.permutation(cols[0].size)
    return [c[perm] for c in cols]


def _metrics_device(ctx, cols, n_series, rw, intervals):
    import torch
    from time_series_spark_b200 import batched
    t = [torch.from_numpy(np.ascontiguousarray(c)).cuda() for c in cols]
    return batched.performance_metrics_device(ctx, t[0], t[1], t[2], t[3], t[4] if intervals else None,
                                              t[5] if intervals else None, n_series, rw)


def _check_metrics(got, cols, series_ids, rw, intervals):
    """Every listed series against bo.performance_metrics: horizons, coverage exact; mse, rmse, mae, mape 1e-12
    relative, MAPE NaN exactly where the oracle's is.  Returns the largest relative deviation."""
    sid, h, y, yhat, lo, hi = cols
    worst = 0.0
    for s in series_ids:
        r = sid == s
        with np.errstate(divide="ignore", invalid="ignore"):
            want = bo.performance_metrics(h[r], y[r], yhat[r], lo[r] if intervals else None, hi[r] if intervals else None, rw)
        g = got["series"] == s
        assert got["horizon"][g].tolist() == want["horizon"].tolist(), s
        if intervals:
            assert got["coverage"][g].tolist() == want["coverage"].tolist(), s
        for k in ("mse", "rmse", "mae", "mape"):
            a, b = got[k][g], want[k]
            assert np.array_equal(np.isnan(a), np.isnan(b)), (s, k)
            ok = ~np.isnan(b)
            if ok.any():
                dev = np.abs(a[ok] - b[ok]) / np.maximum(np.abs(b[ok]), 1e-300)
                worst = max(worst, float(dev.max()))
                assert dev.max() <= 1e-12, (s, k, float(dev.max()))
    return worst


@pytest.mark.parametrize("intervals", [False, True], ids=["no_intervals", "intervals"])
@pytest.mark.parametrize("rw", RWS)
def test_metrics_match_oracle(gpu_ctx, rw, intervals):
    rng = np.random.RandomState(int(rw * 1000) + intervals)
    n_series = 160
    cols = _metric_rows(rng, n_series)
    got = _metrics_device(gpu_ctx, cols, n_series, rw, intervals)
    assert (got["coverage"] is not None) == intervals
    worst = _check_metrics(got, cols, range(n_series), rw, intervals)
    assert not np.isin(got["series"], np.arange(3, n_series, 7)).any()           # empty series have no rows
    DEV["metrics"] = max(DEV.get("metrics", 0.0), worst)
    print(f"metrics rw={rw} intervals={intervals}: largest relative deviation {worst:.2e} "
          f"(running max {DEV['metrics']:.2e})")


def test_metrics_past_the_stride_loop(gpu_ctx, sms):
    """One call over more than sms * 16 CTAs x 128 threads series of 1-6 rows: series past that index match the
    oracle and are byte-identical to the same rows scored in a small call."""
    rng = np.random.RandomState(21)
    n_series = sms * 16 * 128 + 5000
    assert n_series > sms * 16 * 128
    cnt = rng.randint(1, 7, n_series)
    sid = np.repeat(np.arange(n_series), cnt).astype(np.int64)
    R = sid.size
    h = rng.randint(1, 4, R).astype(np.int64) * H
    y = rng.randn(R) * 50
    yhat = y + rng.randn(R) * 5
    lo, hi = yhat - rng.rand(R) * 8, yhat + rng.rand(R) * 8
    perm = rng.permutation(R)
    cols = [c[perm] for c in (sid, h, y, yhat, lo, hi)]
    got = _metrics_device(gpu_ctx, cols, n_series, 0.35, True)
    pick = np.sort(rng.choice(np.arange(sms * 16 * 128, n_series), 300, replace=False))
    _check_metrics(got, cols, pick, 0.35, True)
    # the same rows, in the same order, as series 0 .. 299 of a small call
    keep = np.isin(cols[0], pick)
    small = [c[keep] for c in cols]
    small[0] = np.searchsorted(pick, small[0]).astype(np.int64)
    got2 = _metrics_device(gpu_ctx, small, pick.size, 0.35, True)
    g = np.isin(got["series"], pick)
    assert np.array_equal(np.searchsorted(pick, got["series"][g]), got2["series"])
    for k in ("horizon", "mse", "rmse", "mae", "mape", "coverage"):
        assert got[k][g].tobytes() == got2[k].tobytes(), k


# ---- end to end -----------------------------------------------------------------------------------------------------
def _e2e_batch(dtype):
    """About 30 short hourly series with fractional y (one with a |y| < 1e-8 value), some with gaps longer than the
    horizon so that the closest-date branch fires."""
    rng = np.random.RandomState(31 if dtype == np.float32 else 32)
    t0 = 1_600_000_000 * 10**9
    parts = []
    for k in range(30):
        n = int(rng.randint(80, 200))
        steps = rng.randint(1, 3, n - 1).astype(np.int64) * H
        if k % 3 == 0:
            steps[n // 2] += (2 + k % 4) * D + 5 * H
        ds = t0 + k * 3 * H + np.concatenate(([0], np.cumsum(steps)))
        y = (20 + 5 * np.sin(np.arange(n) / 7.0) + rng.rand(n) * 3).astype(dtype)
        if k == 4:
            y[n - 3] = dtype(3e-9)                     # in the last held-out window
        parts.append((ds, y))
    off = np.concatenate(([0], np.cumsum([p[0].size for p in parts]))).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), off


E2E_TRIPLES = [(D, 3 * D // 2 + 7, 2 * D), (12 * H, 17 * H, 3 * D + 1)]


@pytest.mark.parametrize("triple", E2E_TRIPLES, ids=["period_gt_horizon", "period_gt_horizon_short"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["float32", "float64"])
def test_cross_validation_end_to_end(gpu_ctx, dtype, triple):
    import torch
    from time_series_spark_b200 import batched
    hz, per, ini = triple
    ds, y, off = _e2e_batch(dtype)
    opts = batched.make_options(uncertainty_samples=200)
    cap_h = np.array([float(y[a:b].max()) * CAPM for a, b in zip(off[:-1], off[1:])])
    res = batched.cross_validation_device(gpu_ctx, opts, torch.from_numpy(ds).cuda(), torch.from_numpy(y).cuda(), off,
                                          FLOOR, torch.from_numpy(cap_h).cuda(), hz, per, ini, intervals=True, seed=5,
                                          rolling_window=0.1, keep_fits=True)
    # the plan
    series = [ds[off[i]:off[i + 1]] for i in range(off.size - 1)]
    want_cut = [expected_plan(s, hz, per, ini)[0] for s in series]
    assert res.pair_cutoff.tolist() == np.concatenate(want_cut).tolist()
    assert res.pair_series.tolist() == np.repeat(np.arange(off.size - 1), [c.size for c in want_cut]).tolist()
    assert any(any((c[-1] - x) % per for x in c) for c in want_cut)             # the closest-date branch fired
    assert (res.pair_status >= 0).all()
    he = np.concatenate([np.searchsorted(s, c, side="right") for s, c in zip(series, want_cut)])
    # the fits: byte-identical to direct fits of the same histories, same dtype, forced mask, explicit cap
    f = res.fitted
    for mask in np.unique(res.pair_mask):
        sel = np.flatnonzero(res.pair_mask == mask)
        oc = batched._with_mask(opts, int(mask))
        ps = res.pair_series[sel]
        d = batched.fit_batch_host(gpu_ctx, oc, np.concatenate([ds[off[s]:off[s] + he[p]] for s, p in zip(ps, sel)]),
                                   np.concatenate([y[off[s]:off[s] + he[p]] for s, p in zip(ps, sel)]),
                                   np.concatenate(([0], np.cumsum(he[sel]))).astype(np.int64), FLOOR, 1.0,
                                   cap=cap_h[ps])
        w = d.params.shape[1]
        assert f.params[sel, :w].tobytes() == d.params.tobytes()
        for name in ("tchange", "meta_i32", "meta_i64", "meta_f64"):
            assert getattr(f, name)[sel].tobytes() == getattr(d, name).tobytes(), name
    # rows: y is the input value in float64; yhat and the intervals against the oracle
    worst_yhat = worst_iv = 0.0
    for p in range(res.pair_series.size):
        s, c = int(res.pair_series[p]), int(res.pair_cutoff[p])
        a = off[s]
        rows = np.flatnonzero((res.row_series == s) & (res.cutoff == c))
        we = int(np.searchsorted(series[s], c + hz, side="right"))
        assert res.ds[rows].tolist() == series[s][he[p]:we].tolist()
        assert res.y[rows].tobytes() == y[a + he[p]:a + we].astype(np.float64).tobytes()
        m = int(res.pair_mask[p])
        oc = po.ProphetOptions(yearly_seasonality=bool(m & 1), weekly_seasonality=bool(m & 2), daily_seasonality=bool(m & 4))
        prep = po.prepare(series[s][:he[p]], y[a:a + he[p]].astype(np.float64), FLOOR, cap_h[s], oc)
        S, smax, pr = int(f.meta_i32[p, 1]), f.smax, f.params[p]
        fr = po.FitResult(prep=prep, k=pr[0], m=pr[1], delta=pr[3:3 + S].copy(), sigma_obs=pr[2],
                          beta=pr[3 + smax:3 + smax + prep.K].copy() if prep.seasonalities else np.zeros(1),
                          theta=None, neg_logp=0.0, iters=0, n_evals=0, ret=0)
        ys = float(f.meta_f64[p, 0])
        yo = po.predict(fr, res.ds[rows], FLOOR, cap_h[s], oc)["yhat"]
        worst_yhat = max(worst_yhat, float(np.max(np.abs(yo - res.yhat[rows]))) / ys)
        if p % 9 == 0:
            dr = mc_stream.draws(f, p, res.ds[rows], FLOOR, cap_h[s], True, True, opts.uncertainty_samples, 5)
            lo, hi = mc_stream.bounds(dr, opts.interval_width)
            worst_iv = max(worst_iv, float(max(np.max(np.abs(lo - res.yhat_lower[rows])),
                                               np.max(np.abs(hi - res.yhat_upper[rows])))) / ys)
    assert worst_yhat <= 1e-12 and worst_iv <= 1e-9, (worst_yhat, worst_iv)
    # the metrics
    cols = [res.row_series, res.ds - res.cutoff, res.y, res.yhat, res.yhat_lower, res.yhat_upper]
    got = dict(res.metrics)
    worst = _check_metrics(got, cols, range(off.size - 1), 0.1, True)
    assert np.all(np.isnan(got["mape"][got["series"] == 4]))
    print(f"end to end {dtype.__name__} {triple}: yhat {worst_yhat:.2e}, intervals {worst_iv:.2e} (of y_scale), "
          f"metrics {worst:.2e} relative")


def test_job_on_golden_fixture_holds_to_oracle(tmp_path, model_input_dir, golden_input, gpu_ctx):
    """The golden fixture, duplicate timestamps included, through the backtest job: its cutoffs, held-out rows and
    metrics against the oracle, its rows byte-identical to cross_validation_device on the same packed groups."""
    import pyarrow.parquet as pq
    import torch
    from time_series_spark_b200 import batched
    from time_series_spark_b200.jobs.prophet_backtest import ProphetBacktester
    hz, per, ini = 30 * D, 15 * D, 180 * D
    cfg = {"io": {"input": model_input_dir, "metrics": str(tmp_path / "metrics"), "cv_rows": str(tmp_path / "rows")},
           "model": {"floor": 0, "cap_multiplier": CAPM},
           "backtest": {"horizon": "30 days", "period": "15 days", "initial": "180 days", "intervals": True,
                        "uncertainty_samples": 100}}
    ProphetBacktester.run(None, cfg)
    m = pq.read_table(str(tmp_path / "metrics")).to_pandas()
    r = pq.read_table(str(tmp_path / "rows")).to_pandas()
    gi = golden_input
    assert any(np.any(np.diff(np.sort(g)) == 0) for g in _golden_groups(gi))      # the fixture repeats timestamps
    for dim, g in r.groupby("dim_id"):
        sel = gi["dim_id"] == dim
        ds_sorted = np.sort(gi["ds_ns"][sel].astype(np.int64), kind="stable")
        cut = bo.generate_cutoffs(ds_sorted, hz, per, ini)
        gc = g["cutoff"].astype("int64").to_numpy()
        gd = g["ds"].astype("int64").to_numpy()
        assert np.unique(gc).tolist() == cut.tolist(), dim
        for c in cut:
            he = np.searchsorted(ds_sorted, c, side="right")
            we = np.searchsorted(ds_sorted, c + hz, side="right")
            assert gd[gc == c].tolist() == ds_sorted[he:we].tolist(), (dim, c)
        gm = m[m["dim_id"] == dim]
        want = bo.performance_metrics(gd - gc, g["y"].to_numpy(np.float64), g["yhat"].to_numpy(), g["yhat_lower"].to_numpy(),
                                      g["yhat_upper"].to_numpy(), 0.1)
        assert gm["horizon"].astype("int64").tolist() == want["horizon"].tolist(), dim
        assert gm["coverage"].tolist() == want["coverage"].tolist(), dim
        for k in ("mse", "rmse", "mae", "mape"):
            np.testing.assert_allclose(gm[k].to_numpy(), want[k], rtol=1e-12, atol=0, equal_nan=True)
    # yhat against the oracle through the fits of a direct call on the job's packing
    from time_series_spark_b200.pack import pack_groups_cuda
    frame = ProphetBacktester(cfg).read_input_dataframe(None)
    pk = pack_groups_cuda(frame.table, device="cuda:0")
    yv = pk.y.to(torch.float64)
    lens = torch.from_numpy(np.diff(pk.offsets)).cuda()
    cap = torch.segment_reduce(yv, "max", lengths=lens) * CAPM
    res = batched.cross_validation_device(gpu_ctx, batched.make_options(uncertainty_samples=100), pk.ds.contiguous(),
                                          pk.y.contiguous(), pk.offsets, FLOOR, cap, hz, per, ini, intervals=True,
                                          seed=0, rolling_window=0.1, keep_fits=True)
    assert res.ds.size == len(r)
    assert r["dim_id"].tolist() == pk.dim_id[res.row_series].tolist()
    assert r["yhat"].to_numpy().tobytes() == res.yhat.tobytes()
    assert r["y"].to_numpy(np.float64).tobytes() == res.y.tobytes()
    ds_h, y_h, cap_h = pk.ds.cpu().numpy(), yv.cpu().numpy(), cap.cpu().numpy()
    f = res.fitted
    worst = 0.0
    for p in range(0, res.pair_series.size, max(1, res.pair_series.size // 12)):
        s, c = int(res.pair_series[p]), int(res.pair_cutoff[p])
        a, b = pk.offsets[s], pk.offsets[s + 1]
        he = a + int(np.searchsorted(ds_h[a:b], c, side="right"))
        mk = int(res.pair_mask[p])
        oc = po.ProphetOptions(yearly_seasonality=bool(mk & 1), weekly_seasonality=bool(mk & 2), daily_seasonality=bool(mk & 4))
        prep = po.prepare(ds_h[a:he], y_h[a:he], FLOOR, cap_h[s], oc)
        S, smax, pr = int(f.meta_i32[p, 1]), f.smax, f.params[p]
        fr = po.FitResult(prep=prep, k=pr[0], m=pr[1], delta=pr[3:3 + S].copy(), sigma_obs=pr[2],
                          beta=pr[3 + smax:3 + smax + prep.K].copy() if prep.seasonalities else np.zeros(1),
                          theta=None, neg_logp=0.0, iters=0, n_evals=0, ret=0)
        rows = np.flatnonzero((res.row_series == s) & (res.cutoff == c))
        yo = po.predict(fr, res.ds[rows], FLOOR, cap_h[s], oc)["yhat"]
        worst = max(worst, float(np.max(np.abs(yo - res.yhat[rows]))) / float(f.meta_f64[p, 0]))
    assert worst <= 1e-12, worst
    print(f"golden fixture: {res.pair_series.size} cutoffs, {len(r)} rows, yhat deviation {worst:.2e} of y_scale")
