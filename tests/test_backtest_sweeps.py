"""CPU sweeps of the backtest's reference semantics (DESIGN §9): the oracle's generate_cutoffs against the literal
transcription of fbprophet's loop on thousands of seeded random small series and at durations near int64's range, and
its performance_metrics against the brute-force reading over random row sets, window widths whose ``int(rw * n)``
truncates, and the ``|y| < 1e-8`` MAPE rule at its boundary.  The generators are shared with the GPU tests of
csrc/cv_kernel.cuh (test_gpu_backtest_kernels.py)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import backtest_oracle as bo  # noqa: E402
from test_backtest_oracle import brute_metrics, literal_cutoffs  # noqa: E402

MINUTE = 60 * 10**9
H = 60 * MINUTE
D = 24 * H
UNITS = (1, MINUTE, H, D)
# 2020, 2000, 1900 and the epoch: the walk's arithmetic on either side of zero
EPOCHS = (1_600_000_000 * 10**9, 946_684_800 * 10**9, -2_208_988_800 * 10**9, 0)
INT64_MAX = 2**63 - 1
RWS = (0.0, 1e-3, 0.1, 0.29, 0.35, 0.7, 1.0)


def random_series(rng, unit, horizon, n=None):
    """A sorted history of 1-60 rows: steps of 0 (duplicate timestamps) to 3 units, in 40 % of the series one or two
    gaps longer than ``horizon``, starting near 2020, 2000, 1900 or the epoch."""
    n = int(rng.randint(1, 61)) if n is None else int(n)
    steps = rng.randint(0, 4, max(n - 1, 0)).astype(np.int64) * unit
    if n > 2 and rng.rand() < 0.4:
        for k in rng.randint(0, n - 1, rng.randint(1, 3)):
            steps[k] += horizon + int(rng.randint(1, 3 * horizon + 1, dtype=np.int64))
    t0 = EPOCHS[rng.randint(len(EPOCHS))] + int(rng.randint(0, 1000)) * unit + int(rng.randint(0, 10**6))
    return t0 + np.concatenate(([0], np.cumsum(steps))).astype(np.int64)


def random_triple(rng, unit):
    """(horizon, period, initial) on the scale of ``unit``: the period below, equal to or above the horizon and off
    the step grid, the initial window 1 ns, off-grid, or a whole number of units."""
    horizon = int(unit * rng.uniform(1, 8)) + int(rng.randint(0, 3))
    r = (0.37, 1.0, 1.6)[rng.randint(3)]
    period = horizon if r == 1.0 else max(1, int(horizon * r) + int(rng.randint(1, 4)))
    k = rng.randint(3)
    initial = 1 if k == 0 else (int(horizon * rng.uniform(0, 5)) + 1 if k == 1 else unit * int(rng.randint(1, 40)))
    return horizon, period, initial


def expected_plan(ds, horizon, period, initial):
    """(cutoffs, err bits) of one sorted series as cv_plan_kernel reports them: the oracle's cutoffs, its two
    exceptions as ERR_HORIZON / ERR_INITIAL (a 0-row series: ERR_HORIZON), ERR_FEW when a cutoff has < 2 rows."""
    if ds.size == 0:
        return np.zeros(0, np.int64), 1
    try:
        c = bo.generate_cutoffs(ds, horizon, period, initial)
    except ValueError as e:
        return np.zeros(0, np.int64), 1 if str(e) == "Less data than horizon." else 2
    few = int(np.searchsorted(ds, c, side="right").min()) < 2
    return c, 4 if few else 0


def _literal_or_error(ds, hz, per, ini, fn):
    try:
        return [int(v) for v in fn(ds, hz, per, ini)]
    except ValueError as e:
        return str(e)


def test_cutoffs_match_literal_loop_on_random_series():
    rng = np.random.RandomState(2024)
    seen = {"horizon": 0, "initial": 0, "cutoffs": 0, "closest_date": 0, "duplicates": 0, "pre_1970": 0, "one_row": 0}
    for _ in range(3000):
        unit = UNITS[rng.randint(len(UNITS))]
        hz, per, ini = random_triple(rng, unit)
        ds = random_series(rng, unit, hz)
        want = _literal_or_error(ds, hz, per, ini, literal_cutoffs)
        got = _literal_or_error(ds, hz, per, ini, bo.generate_cutoffs)
        assert got == want, (ds.tolist(), hz, per, ini)
        if isinstance(want, str):
            seen["horizon" if want == "Less data than horizon." else "initial"] += 1
        else:
            seen["cutoffs"] += 1
            seen["closest_date"] += any((want[-1] - c) % per for c in want)
        seen["duplicates"] += bool(np.any(np.diff(ds) == 0))
        seen["pre_1970"] += bool(ds[0] < 0)
        seen["one_row"] += ds.size == 1
    # every outcome and input class occurs often enough to matter
    assert min(seen.values()) >= 50, seen


@pytest.mark.parametrize("epoch", [946_684_800 * 10**9, -2_208_988_800 * 10**9])
def test_cutoffs_at_durations_near_int64(epoch):
    """Durations of ~100 000 days to INT64_MAX on 2000s and 1900s data: first + initial, last - horizon and
    prev - period leave int64; the oracle's Python integers give fbprophet's plan."""
    ds = epoch + np.arange(0, 10 * D + 1, H, dtype=np.int64)
    big = (100_000 * D, 106_751 * D, INT64_MAX)
    triples = [(D, D // 2, b) for b in big] + [(b, D // 2, D) for b in big] + [(D, b, D) for b in big] + \
              [(D, b, 1) for b in big]
    for hz, per, ini in triples:
        assert _literal_or_error(ds, hz, per, ini, bo.generate_cutoffs) == \
            _literal_or_error(ds, hz, per, ini, literal_cutoffs), (hz, per, ini)


def random_rows(rng, n, ties=True, intervals=True):
    """n held-out rows of one series: horizons (tied or distinct), fractional y / yhat of both signs, bounds that
    sometimes equal y (coverage is inclusive) or are NaN."""
    n_h = max(1, n // int(rng.randint(1, 5))) if ties else n
    h = (rng.randint(1, n_h + 1, n).astype(np.int64) * H) if ties else (rng.permutation(n).astype(np.int64) + 1) * 7
    y = rng.randn(n) * 10 ** rng.uniform(-2, 3)
    yhat = y + rng.randn(n) * np.abs(y).mean()
    if not intervals:
        return h, y, yhat, None, None
    lo, hi = yhat - rng.rand(n) * 5, yhat + rng.rand(n) * 5
    k = rng.rand(n)
    lo[k < 0.1], hi[k < 0.1] = y[k < 0.1], y[k < 0.1]                      # lo == y == hi
    lo[(k >= 0.1) & (k < 0.15)] = np.nan
    hi[(k >= 0.15) & (k < 0.2)] = np.nan
    return h, y, yhat, lo, hi


def assert_metrics_equal_brute(h, y, yhat, lo, hi, rw):
    got = bo.performance_metrics(h, y, yhat, lo, hi, rw)
    want = brute_metrics(h, y, yhat, lo, hi, rw)
    assert got["horizon"].tolist() == [int(r[0]) for r in want]
    for j, k in ((1, "mse"), (2, "mae"), (3, "mape")):
        np.testing.assert_allclose(got[k], [r[j] for r in want], rtol=1e-12, atol=0, equal_nan=True)
    np.testing.assert_allclose(got["rmse"], np.sqrt(got["mse"]), rtol=0)
    if lo is not None:
        np.testing.assert_allclose(got["coverage"], [r[4] for r in want], rtol=1e-12, atol=0)
    return got


def test_performance_metrics_matches_brute_force_on_random_rows():
    rng = np.random.RandomState(77)
    for it in range(600):
        n = int(rng.choice([1, 2, 3, 7, 10, 33, 100]))
        ties, iv = bool(rng.rand() < 0.6), bool(rng.rand() < 0.6)
        rw = RWS[it % len(RWS)]
        assert_metrics_equal_brute(*random_rows(rng, n, ties, iv), rw)


@pytest.mark.parametrize("rw, n, w", [(0.29, 100, 28), (0.7, 10, 7), (0.35, 20, 7), (1e-3, 100, 1), (0.0, 5, 1),
                                      (1.0, 9, 9)])
def test_window_width_truncation(rw, n, w):
    """w = min(n, max(1, int(rw * n))): on distinct horizons the first w - 1 have no row, so the row count pins w
    (0.29 * 100 is 28.999..., truncated to 28)."""
    rng = np.random.RandomState(n)
    h, y, yhat, lo, hi = random_rows(rng, n, ties=False)
    got = assert_metrics_equal_brute(h, y, yhat, lo, hi, rw)
    assert got["horizon"].size == n - w + 1
    last = np.argsort(h)[-w:]
    np.testing.assert_allclose(got["mae"][-1], np.abs(y - yhat)[last].mean(), rtol=1e-12)


@pytest.mark.parametrize("v, tiny", [(1e-8, False), (np.nextafter(1e-8, 0), True), (-1e-9, True), (-0.0, True),
                                     (-1e-8, False)])
def test_mape_tiny_y_boundary(v, tiny):
    rng = np.random.RandomState(9)
    h, y, yhat, lo, hi = random_rows(rng, 12, ties=True)
    y[5] = v
    with np.errstate(divide="ignore", invalid="ignore"):
        got = assert_metrics_equal_brute(h, y, yhat, lo, hi, 0.1)
    assert got["horizon"].size > 0
    assert np.all(np.isnan(got["mape"])) if tiny else np.all(np.isfinite(got["mape"]))
