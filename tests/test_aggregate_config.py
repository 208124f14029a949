"""Window totals of the forecast (DESIGN §13) without a GPU: the restatement of mc_sum_kernel's windows and sums
(tests/window_oracle.window_sums) against a brute-force loop, against fbprophet's process in distribution, the two
shortcuts it replaces, and the scorer's ``forecast.aggregate`` configuration."""
import numpy as np
import pytest

import window_oracle as wo
from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
from test_mc_stream import _model
from time_series_spark_b200 import batched
from time_series_spark_b200.jobs.prophet_scorer import aggregate_rule

H_NS = 3600 * 10**9
DAY = 24 * H_NS


def _brute(d, ds, width_ns, origin_ns, width):
    """Windows by Python's floor division on exact integers, sums point by point, one draw at a time."""
    wins, sums = [], []
    for h, t in enumerate(int(x) for x in ds):
        w = (t - origin_ns) // width_ns
        if not wins or wins[-1][0] != w:
            wins.append([w, 0])
            sums.append([0.0] * d.shape[1])
        wins[-1][1] += 1
        sums[-1] = [s + float(x) for s, x in zip(sums[-1], d[h])]
    sums = np.array(sums).reshape(len(wins), d.shape[1])
    lo_p, hi_p = mcs.percentiles(width)
    return (np.array([origin_ns + w * width_ns for w, _ in wins], np.int64), np.array([c for _, c in wins], np.int64),
            np.array([np.percentile(s, lo_p) for s in sums]), np.array([np.percentile(s, hi_p) for s in sums]))


@pytest.mark.parametrize("case", [
    dict(first=3 * DAY + 5 * H_NS, step=H_NS, H=60, width=DAY, origin=0),              # partial first and last window
    dict(first=-2 * DAY - 7 * H_NS, step=H_NS, H=80, width=DAY, origin=0),             # ds before the origin
    dict(first=-5 * H_NS, step=H_NS, H=30, width=8 * H_NS, origin=3 * H_NS + 17),      # non-zero origin, crossing it
    dict(first=10 * DAY, step=H_NS, H=40, width=7 * H_NS // 2, origin=4 * DAY),        # the width does not divide the grid
    dict(first=10 * DAY, step=H_NS, H=25, width=H_NS, origin=0),                       # one point per window
    dict(first=10 * DAY, step=H_NS, H=25, width=1000 * DAY, origin=0),                 # the whole frame in one window
    dict(first=10 * DAY, step=3 * DAY, H=9, width=DAY, origin=0),                      # a grid coarser than the width
    dict(first=10 * DAY, step=H_NS, H=1, width=DAY, origin=0),
])
def test_window_sums_against_brute_force(case):
    ds = case["first"] + case["step"] * np.arange(case["H"], dtype=np.int64)
    d = np.random.RandomState(case["H"]).randn(case["H"], 37) * 10.0 + 3.0
    got = wo.window_sums(d, ds, case["width"], case["origin"], 0.8)
    ref = _brute(d, ds, case["width"], case["origin"], 0.8)
    for g, r in zip(got, ref):
        assert np.array_equal(g, r)
    assert got[1].sum() == case["H"] and np.all(got[1] > 0)
    assert np.all(np.diff(got[0]) > 0)


def test_window_sums_of_an_empty_frame():
    start, pts, lo, hi = wo.window_sums(np.zeros((0, 5)), np.zeros(0, np.int64), DAY, 0, 0.8)
    assert start.size == pts.size == lo.size == hi.size == 0


def test_window_slots_bound():
    first = np.array([10 * DAY + 5 * H_NS, -3 * DAY - 1], np.int64)
    last = first + np.array([70, 30], np.int64) * H_NS
    assert batched.window_slots(first, last, DAY, 0) == 4         # 5 h + 70 h: days 10 .. 13
    assert batched.window_slots(first, last, 1000 * DAY, -500 * DAY) == 1
    assert batched.window_slots(first[:0], last[:0], DAY, 0) == 1


def _process_draws(fr, p, oopts, fut, cap, n, seed):
    """fbprophet's sample_model / sample_predictive_trend on numpy's RNG (the process po.predict_uncertainty restates),
    keeping the draws: [H, n]."""
    rng = np.random.RandomState(seed)
    pred = po.predict(fr, fut, 0.0, cap, oopts)
    t, Tmax, S = pred["t"], pred["t"].max(), len(p.t_change)
    lam = np.mean(np.abs(fr.delta)) + 1e-8
    out = np.empty((t.size, n))
    for j in range(n):
        k = rng.poisson(S * (Tmax - 1)) if Tmax > 1 else 0
        cp_new = np.sort(1 + rng.rand(k) * (Tmax - 1))
        d_new = rng.laplace(0, lam, k)
        trend = po._piecewise_trend(t, pred["cap_scaled"], np.concatenate((fr.delta, d_new)), fr.k, fr.m,
                                    np.concatenate((p.t_change, cp_new)), p.logistic) * p.y_scale + pred["floor"]
        out[:, j] = trend * (1 + pred["multiplicative_terms"]) + pred["additive_terms"] \
            + rng.normal(0, fr.sigma_obs, t.size) * p.y_scale
    return out


@pytest.mark.parametrize("mode", ["multiplicative", "additive"])
@pytest.mark.parametrize("growth", ["logistic", "linear"])
def test_window_bounds_match_fbprophet_process_and_beat_both_shortcuts(growth, mode):
    """Daily totals of a four-day hourly frame past the history: the restated bounds agree with the sums of
    fbprophet-process draws within five Monte-Carlo standard errors; and the interval of the second day's total is narrower
    than the sum of the pointwise bounds (the noise of 24 points partly cancels) and wider than treating the points as
    independent (a simulated changepoint moves all of them together)."""
    n, w = 20_000, 0.8
    p, fr, oopts, rec = _model(growth, mode)
    fut = int(p.ds_sorted[-1]) + H_NS * np.arange(1, 97, dtype=np.int64)        # 2021-03-31 00:00 ... four whole days
    cap = 130.0
    d = mcs.draws(rec, 0, fut, 0.0, cap, growth == "logistic", mode == "multiplicative", n, 99)
    start, pts, lo, hi = wo.window_sums(d, fut, DAY, 0, w)
    assert np.array_equal(pts, [24, 24, 24, 24]) and start[0] == fut[0]
    ref = _process_draws(fr, p, oopts, fut, cap, n, 0).reshape(4, 24, n).sum(axis=1)
    mine = d.reshape(4, 24, n).sum(axis=1)
    for q, got in ((0.1, lo), (0.9, hi)):
        spread = (np.quantile(mine, q + 0.02, axis=1) - np.quantile(mine, q - 0.02, axis=1)) / 0.04
        se = np.sqrt(q * (1 - q) / n) * spread
        z = np.abs(got - np.quantile(ref, q, axis=1)) / (np.sqrt(2.0) * se)
        assert np.all(z < 5.0), (growth, mode, q, z)
    plo, phi = mcs.bounds(d, w)
    day = slice(24, 48)
    total = hi[1] - lo[1]
    assert total < 0.75 * np.sum(phi[day] - plo[day]), (total, np.sum(phi[day] - plo[day]))
    assert total > 1.25 * np.sqrt(np.sum((phi[day] - plo[day]) ** 2)), (total, np.sqrt(np.sum((phi[day] - plo[day]) ** 2)))


def _cfg(**fc):
    return {"io": {"models": "m", "forecasts": "f", "aggregates": "a"}, "forecast": {"periods": 4, "frequency": "h", **fc}}


def test_aggregate_rule_parses_fixed_widths_and_origins():
    assert aggregate_rule(_cfg()) is None
    assert aggregate_rule(_cfg(aggregate="1D")) == (DAY, 0)
    assert aggregate_rule(_cfg(aggregate="7D", aggregate_origin="1970-01-05")) == (7 * DAY, 4 * DAY)
    assert aggregate_rule(_cfg(aggregate="8h")) == (8 * H_NS, 0)
    assert aggregate_rule(_cfg(aggregate="1h", aggregate_origin="1969-12-31 06:00:00")) == (H_NS, -18 * H_NS)
    assert aggregate_rule(_cfg(aggregate="15min")) == (15 * 60 * 10**9, 0)


@pytest.mark.parametrize("spec", ["M", "1M", "Q", "MS", "A", "B", "fortnight", "", 5, "-1D", "0h"])
def test_bad_aggregate_width_is_refused(spec):
    with pytest.raises(ValueError, match="forecast.aggregate"):
        aggregate_rule(_cfg(aggregate=spec))


@pytest.mark.parametrize("origin", ["not a date", "2021-13-45", float("nan")])
def test_bad_aggregate_origin_is_refused(origin):
    with pytest.raises(ValueError, match="forecast.aggregate_origin"):
        aggregate_rule(_cfg(aggregate="1D", aggregate_origin=origin))


def test_aggregate_needs_its_output_directory_and_no_components():
    cfg = _cfg(aggregate="1D")
    del cfg["io"]["aggregates"]
    with pytest.raises(ValueError, match="io.aggregates"):
        aggregate_rule(cfg)
    with pytest.raises(ValueError, match="forecast.components"):
        aggregate_rule(_cfg(aggregate="1D", components=True))
