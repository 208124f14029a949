"""CPU tests of the backtest's reference semantics (DESIGN §9): the oracle's cutoff plan against a literal
transcription of fbprophet's generate_cutoffs loop, its performance_metrics against a brute-force reading of the
per-horizon rule, and the job's config checks."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper module next to this file
import backtest_oracle as bo  # noqa: E402
from time_series_spark_b200.jobs.prophet_backtest import backtest_spec_from_config

H = 3600 * 10**9
D = 24 * H


def literal_cutoffs(ds, horizon, period, initial):
    """fbprophet 0.5 generate_cutoffs, transcribed line by line over a plain list (no binary search)."""
    ds = [int(v) for v in ds]
    cutoff = max(ds) - horizon
    if cutoff < min(ds):
        raise ValueError("Less data than horizon.")
    result = [cutoff]
    while result[-1] is not None and result[-1] >= min(ds) + initial:
        cutoff -= period
        if not any(cutoff < d <= cutoff + horizon for d in ds):
            before = [d for d in ds if d <= cutoff]
            cutoff = (max(before) - horizon) if before else None       # NaT
        result.append(cutoff)
        if cutoff is None:
            break
    result = result[:-1]
    if not result:
        raise ValueError("Less data than horizon after initial window. Make horizon or initial shorter.")
    return list(reversed(result))


def _grid(days, step=H, start=1_600_000_000 * 10**9):
    return start + np.arange(0, days * D // step + 1, dtype=np.int64) * step


CASES = {
    "regular": (_grid(10), D, D // 2, 3 * D),
    "gap": (np.concatenate([_grid(10), _grid(10)[-1] + 6 * D + 7 * H + _grid(5) - _grid(5)[0]]), D, D // 2, 2 * D),
    "big_gap_nat": (np.array([0, 2 * D, 30 * D, 31 * D], np.int64) + 10**18, D, 10 * D, D),
    "exact_on_timestamp": (_grid(6, step=6 * H), 12 * H, 6 * H, 2 * D),
    "irregular": (np.cumsum(np.random.RandomState(3).randint(1, 9, 300)).astype(np.int64) * H, 2 * D, 17 * H, 5 * D),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_cutoffs_match_literal_loop(name):
    ds, hz, per, ini = CASES[name]
    ds = np.sort(ds)
    got = bo.generate_cutoffs(ds, hz, per, ini)
    assert got.tolist() == literal_cutoffs(ds, hz, per, ini)
    assert np.all(np.diff(got) > 0)


def test_cutoff_exactly_on_a_timestamp_keeps_that_row_in_the_history():
    ds = _grid(6, step=6 * H)
    cut = bo.generate_cutoffs(ds, 12 * H, 6 * H, 2 * D)
    assert set(cut.tolist()) <= set(ds.tolist())
    c = int(cut[0])
    assert int(np.searchsorted(ds, c, side="right")) == int(np.flatnonzero(ds == c)[0]) + 1


def test_gap_takes_the_closest_date_branch():
    ds, hz, per, ini = CASES["gap"]
    cut = bo.generate_cutoffs(np.sort(ds), hz, per, ini)
    # at least one cutoff is not on the period grid counted back from last - horizon
    last = int(ds.max()) - hz
    assert any((last - int(c)) % per for c in cut)


def test_cutoff_errors():
    ds = _grid(2)
    with pytest.raises(ValueError, match="Less data than horizon"):
        bo.generate_cutoffs(ds, 3 * D, D, D)
    with pytest.raises(ValueError, match="after initial window"):
        bo.generate_cutoffs(ds, D, D // 2, 5 * D)
    with pytest.raises(ValueError, match="Less data than horizon"):
        literal_cutoffs(ds, 3 * D, D, D)


def test_period_and_initial_defaults():
    spec = backtest_spec_from_config({"backtest": {"horizon": "1 days"}})
    assert spec["horizon"] == D and spec["period"] == D // 2 and spec["initial"] == 3 * D
    assert spec["rolling_window"] == 0.1 and spec["intervals"] is False
    ds = _grid(10, step=15 * 60 * 10**9)
    assert bo.generate_cutoffs(ds, spec["horizon"], spec["period"], spec["initial"]).tolist() == \
        literal_cutoffs(ds, D, D // 2, 3 * D)


def brute_metrics(h, y, yhat, lo, hi, rw):
    """The per-horizon rule read literally: for each distinct horizon, take the rows of that horizon and then of the
    smaller horizons nearest first, one row at a time with fractional weight for the group the window stops in."""
    n = len(h)
    w = min(n, max(1, int(rw * n)))
    hs = sorted(set(h.tolist()))
    out = []
    tiny = np.any(np.abs(y) < 1e-8)
    for k, hv in enumerate(hs):
        weights = np.zeros(n)
        need = w
        for g in range(k, -1, -1):
            idx = np.flatnonzero(h == hs[g])
            if need <= 0:
                break
            take = min(need, idx.size)
            weights[idx] = take / idx.size
            need -= take
        if need > 0:
            continue
        e = y - yhat
        with np.errstate(divide="ignore", invalid="ignore"):
            row = [hv, np.sum(weights * e * e) / w, np.sum(weights * np.abs(e)) / w,
                   np.nan if tiny else np.sum(weights * np.abs(e) / np.abs(y)) / w]
        if lo is not None:
            row.append(np.sum(weights * ((lo <= y) & (y <= hi))) / w)
        out.append(row)
    return out


def _rows(n_cut, n_h, rng, ties=True, zero_y=False):
    h = np.concatenate([np.arange(1, n_h + 1) * H for _ in range(n_cut)]).astype(np.int64)
    if not ties:
        h = h + np.arange(h.size)
    y = rng.randint(1, 50, h.size).astype(np.float64)
    if zero_y:
        y[3] = 0.0
    yhat = y + rng.randn(h.size) * 3
    lo, hi = yhat - 2, yhat + 2
    perm = rng.permutation(h.size)
    return h[perm], y[perm], yhat[perm], lo[perm], hi[perm]


@pytest.mark.parametrize("rw", [0.0, 0.1, 0.35, 1.0])
@pytest.mark.parametrize("shape", [(22, 24, True), (3, 2, True), (1, 7, False), (4, 5, False)])
@pytest.mark.parametrize("intervals", [False, True])
def test_performance_metrics_matches_brute_force(rw, shape, intervals):
    rng = np.random.RandomState(hash((rw, shape, intervals)) % 2**31)
    h, y, yhat, lo, hi = _rows(shape[0], shape[1], rng, ties=shape[2])
    got = bo.performance_metrics(h, y, yhat, lo if intervals else None, hi if intervals else None, rw)
    want = brute_metrics(h, y, yhat, lo if intervals else None, hi if intervals else None, rw)
    assert got["horizon"].tolist() == [int(r[0]) for r in want]
    np.testing.assert_allclose(got["mse"], [r[1] for r in want], rtol=1e-12)
    np.testing.assert_allclose(got["rmse"], np.sqrt([r[1] for r in want]), rtol=1e-12)
    np.testing.assert_allclose(got["mae"], [r[2] for r in want], rtol=1e-12)
    np.testing.assert_allclose(got["mape"], [r[3] for r in want], rtol=1e-12)
    if intervals:
        np.testing.assert_allclose(got["coverage"], [r[4] for r in want], rtol=1e-12)
    else:
        assert got["coverage"] is None


def test_performance_metrics_small_n_and_window_edges():
    rng = np.random.RandomState(5)
    h, y, yhat, lo, hi = _rows(1, 6, rng)        # n = 6 < 10: w = max(1, int(0.1 * 6)) = 1, one row per horizon
    got = bo.performance_metrics(h, y, yhat, rolling_window=0.1)
    assert got["horizon"].size == 6
    np.testing.assert_allclose(got["mae"], np.abs(y - yhat)[np.argsort(h)], rtol=1e-12)
    got = bo.performance_metrics(h, y, yhat, rolling_window=1.0)      # w = n: only the largest horizon has a row
    assert got["horizon"].tolist() == [int(h.max())]
    np.testing.assert_allclose(got["mae"], [np.mean(np.abs(y - yhat))], rtol=1e-12)


def test_mape_is_nan_for_a_series_with_a_zero():
    rng = np.random.RandomState(6)
    h, y, yhat, lo, hi = _rows(5, 4, rng, zero_y=True)
    with np.errstate(divide="ignore"):
        got = bo.performance_metrics(h, y, yhat, rolling_window=0.1)
    assert got["horizon"].size > 0 and np.all(np.isnan(got["mape"])) and np.all(np.isfinite(got["mae"]))


@pytest.mark.parametrize("bt, match", [
    ({}, "backtest.horizon"),
    ({"horizon": "-1 days"}, "backtest.horizon"),
    ({"horizon": "0 days"}, "backtest.horizon"),
    ({"horizon": "soon"}, "backtest.horizon"),
    ({"horizon": "1 days", "period": "0 hours"}, "backtest.period"),
    ({"horizon": "1 days", "initial": "-3 days"}, "backtest.initial"),
    ({"horizon": "1 days", "rolling_window": 1.5}, "backtest.rolling_window"),
    ({"horizon": "1 days", "rolling_window": -0.1}, "backtest.rolling_window"),
    ({"horizon": "1 days", "intervals": True, "interval_width": 1.2}, "backtest.interval_width"),
    ({"horizon": "1 days", "intervals": True, "uncertainty_samples": 1}, "backtest.uncertainty_samples"),
])
def test_config_validation(bt, match):
    with pytest.raises(ValueError, match=match):
        backtest_spec_from_config({"backtest": bt})


def test_interval_width_ignored_without_intervals():
    spec = backtest_spec_from_config({"backtest": {"horizon": "12 hours", "interval_width": 7}})
    assert spec["intervals"] is False and spec["uncertainty_samples"] == 0
