"""CPU tests of the backtest's window totals (DESIGN §14): the ``backtest.aggregate`` key and the anchoring rule of
tests/window_backtest_oracle.window_rows, the reference the GPU window rows are held to."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper module next to this file
import backtest_oracle as bo  # noqa: E402
import window_backtest_oracle as wbo  # noqa: E402
from time_series_spark_b200.jobs import prophet_backtest as pb  # noqa: E402

H = 3600 * 10**9
D = 24 * H
MIN15 = 15 * 60 * 10**9


def _cfg(window_metrics=True, **bt):
    io = {"metrics": "/tmp/m"}
    if window_metrics:
        io["window_metrics"] = "/tmp/wm"
    return {"io": io, "model": {"floor": 0, "cap_multiplier": 1.1}, "backtest": {"horizon": "2 days", **bt}}


@pytest.mark.parametrize("spec,ns", [("1h", H), ("8h", 8 * H), ("1D", D), ("2 days", 2 * D), ("15min", MIN15),
                                     ("12h", 12 * H)])
def test_aggregate_widths_that_divide_the_horizon(spec, ns):
    assert pb.backtest_spec_from_config(_cfg(aggregate=spec))["aggregate"] == ns


def test_no_key_no_width():
    assert pb.backtest_spec_from_config(_cfg())["aggregate"] is None
    assert pb.backtest_spec_from_config(_cfg(window_metrics=False))["aggregate"] is None


@pytest.mark.parametrize("spec", ["7h", "5D", "3 days", "13min"])
def test_width_that_does_not_divide_the_horizon(spec):
    with pytest.raises(ValueError, match=r"backtest\.aggregate.*divide"):
        pb.backtest_spec_from_config(_cfg(aggregate=spec))


@pytest.mark.parametrize("spec", ["0h", "0D", "-1h", "-1D"])
def test_zero_or_negative_width(spec):
    with pytest.raises(ValueError, match=r"backtest\.aggregate"):
        pb.backtest_spec_from_config(_cfg(aggregate=spec))


@pytest.mark.parametrize("spec", ["M", "MS", "W-MON", "Q", "nonsense"])
def test_calendar_offsets_are_refused(spec):
    with pytest.raises(ValueError, match=r"backtest\.aggregate.*fixed-width"):
        pb.backtest_spec_from_config(_cfg(aggregate=spec))


def test_window_metrics_output_is_required():
    with pytest.raises(ValueError, match=r"backtest\.aggregate.*io\.window_metrics"):
        pb.backtest_spec_from_config(_cfg(window_metrics=False, aggregate="1D"))


def _cv_rows(ds, horizon, period, initial, rng):
    """Held-out rows of one series as cross_validation orders them (cutoff, then ds), with random y / yhat."""
    ds = np.asarray(ds, np.int64)
    parts = []
    for c in bo.generate_cutoffs(ds, horizon, period, initial):
        he, we = np.searchsorted(ds, c, side="right"), np.searchsorted(ds, c + horizon, side="right")
        parts.append((ds[he:we], np.full(we - he, c, np.int64)))
    d = np.concatenate([p[0] for p in parts])
    c = np.concatenate([p[1] for p in parts])
    return d, c, rng.normal(10, 3, d.size), rng.normal(10, 3, d.size)


def test_width_equal_to_the_horizon_gives_one_window_per_pair():
    rng = np.random.RandomState(0)
    ds = np.arange(15 * 96, dtype=np.int64) * MIN15 + 10**18 + 7 * MIN15
    d, c, y, yh = _cv_rows(ds, D, D // 2, 3 * D, rng)
    w = wbo.window_rows(d, c, y, yh, D)
    cuts = np.unique(c)
    assert w["cutoff"].tolist() == cuts.tolist() and np.all(w["horizon"] == D)
    for i, cut in enumerate(cuts):
        sel = c == cut
        s = 0.0
        for v in y[sel]:
            s = s + v
        assert w["points"][i] == sel.sum() == 96 and w["y"][i] == s


def test_width_equal_to_the_step_gives_the_cv_rows():
    rng = np.random.RandomState(1)
    ds = np.arange(10 * 24, dtype=np.int64) * H + 10**18 + 3 * MIN15      # cutoffs off the hour grid's phase
    d, c, y, yh = _cv_rows(ds, D, D // 2, 3 * D, rng)
    w = wbo.window_rows(d, c, y, yh, H)
    assert np.all(w["points"] == 1) and w["cutoff"].tolist() == c.tolist()
    assert w["horizon"].tolist() == (d - c).tolist()
    assert w["y"].tobytes() == y.tobytes() and w["yhat"].tobytes() == yh.tobytes()


def test_rows_at_window_edges_land_in_the_right_window():
    """Window j is (c + j W, c + (j + 1) W]: a row at exactly c + j W is window j - 1's last, 1 ns later window j's
    first, 1 ns earlier still window j - 1's."""
    W, c = 8 * H, 10**18
    offs = []
    for j in (1, 2):
        offs += [j * W - 1, j * W, j * W + 1]
    offs += [3 * W]                                              # the held-out span's last instant
    d = c + np.array([1] + offs, np.int64)
    w = wbo.window_rows(d, np.full(d.size, c), np.arange(d.size, dtype=np.float64), np.zeros(d.size), W)
    # windows: (c, c+W] = {1, W-1, W}; (c+W, c+2W] = {W+1, 2W-1, 2W}; (c+2W, c+3W] = {2W+1, 3W}
    assert w["horizon"].tolist() == [W, 2 * W, 3 * W]
    assert w["points"].tolist() == [3, 3, 2]
    assert w["y"].tolist() == [0.0 + 1 + 2, 0.0 + 3 + 4 + 5, 0.0 + 6 + 7]


def test_windows_emptied_by_a_gap_get_no_row():
    W, c = 4 * H, 10**18
    d = c + np.array([H, 2 * H, 17 * H, 24 * H], np.int64)      # nothing in (c+4h, c+16h]
    w = wbo.window_rows(d, np.full(d.size, c), np.ones(d.size), np.ones(d.size), W)
    assert w["horizon"].tolist() == [W, 5 * W, 6 * W]
    assert w["points"].tolist() == [2, 1, 1]
    assert w["first"].tolist() == [0, 2, 3, 4]


def test_windows_restart_at_every_cutoff():
    """Two cutoffs 12 h apart with overlapping held-out spans: each row is counted once per pair, in its own
    cutoff's windows, and the per-horizon windows line up across cutoffs."""
    rng = np.random.RandomState(2)
    ds = np.arange(6 * 24, dtype=np.int64) * H + 10**18
    d, c, y, yh = _cv_rows(ds, D, D // 2, 2 * D, rng)
    w = wbo.window_rows(d, c, y, yh, 6 * H)
    ncut = np.unique(c).size
    assert ncut >= 2 and w["cutoff"].size == 4 * ncut
    assert w["horizon"].tolist() == [6 * H, 12 * H, 18 * H, 24 * H] * ncut
    assert int(w["points"].sum()) == d.size
