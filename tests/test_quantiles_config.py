"""CPU tests of forecast quantiles (DESIGN §15): the ``forecast.quantiles`` / ``backtest.quantiles`` keys and their
columns, and the references tests/quantile_oracle.py holds the GPU to."""
import os
import sys

import numpy as np
import pyarrow as pa
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))     # the helper modules next to this file
import quantile_oracle as qo  # noqa: E402
from oracle import mc_stream as mcs  # noqa: E402
from time_series_spark_b200.frame import Frame  # noqa: E402
from time_series_spark_b200.jobs import prophet_backtest as pb  # noqa: E402
from time_series_spark_b200.jobs import prophet_scorer as ps  # noqa: E402

H = 3600 * 10**9
_EMPTY = pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32()),
                   "floor": pa.array([], pa.float32()), "cap": pa.array([], pa.float32()),
                   "model": pa.array([], pa.binary())})
BAD_LEVELS = [0.5, "0.5", True, [], [True], [0.5, False], [float("nan")], [-0.1], [1.5], [0.1, 0.10],
              [0.5, "0.9"], [0.1] * 33, {"a": 0.5}]


def _run_empty(fc):
    return ps.forecast_time_series({"forecast": {"periods": 4, "frequency": "h", **fc}}).apply_batched(
        _EMPTY, ["series_id", "dim_id"])


# ---------------------------------------------------------------------------------------------------------------------
# forecast.quantiles
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", BAD_LEVELS)
def test_scorer_refuses_bad_levels_naming_the_key(bad):
    with pytest.raises(ValueError, match=r"forecast\.quantiles"):
        ps.forecast_quantiles({"forecast": {"quantiles": bad}})
    with pytest.raises(ValueError, match=r"forecast\.quantiles"):
        _run_empty({"quantiles": bad})


def test_scorer_refuses_components_and_aggregate():
    with pytest.raises(ValueError, match=r"forecast\.quantiles.*forecast\.components"):
        ps.forecast_quantiles({"forecast": {"quantiles": [0.5], "components": True}})
    with pytest.raises(ValueError, match=r"forecast\.quantiles.*forecast\.aggregate"):
        ps.forecast_quantiles({"forecast": {"quantiles": [0.5], "aggregate": "1D"}, "io": {"aggregates": "/tmp/a"}})


def test_column_names():
    assert [ps.quantile_column(q) for q in (0.1, 0.5, 0.975, 0, 1, 0.05)] == \
        ["yhat_q0.1", "yhat_q0.5", "yhat_q0.975", "yhat_q0.0", "yhat_q1.0", "yhat_q0.05"]
    assert ps.forecast_quantiles({"forecast": {"quantiles": [0.9, 0.1, 0, 1, np.float32(0.5)]}}) == \
        [0.9, 0.1, 0.0, 1.0, float(np.float32(0.5))]
    assert ps.forecast_quantiles({"forecast": {}}) is None


@pytest.mark.parametrize("intervals", [False, True])
@pytest.mark.parametrize("levels", [None, [0.9, 0.1, 0.5]])
def test_empty_shard_schema_carries_the_quantile_columns(levels, intervals):
    out = _run_empty({"intervals": intervals, **({"quantiles": levels} if levels else {})})
    want = ["series_id", "dim_id", "ds", "yhat"] + (["yhat_lower", "yhat_upper"] if intervals else [])
    want += ["yhat_q0.9", "yhat_q0.1", "yhat_q0.5"] if levels else []
    assert out.column_names == want and out.num_rows == 0
    for c in want[4:]:
        assert out.schema.field(c).type == pa.float64()


def _forecast_frame(n=5):
    t = {"series_id": pa.array(np.arange(n, dtype=np.int32)), "dim_id": pa.array(np.ones(n, np.int32)),
         "ds": pa.array(np.arange(n, dtype=np.int64) * H + 10**18).cast(pa.timestamp("ns")),
         "yhat": pa.array(np.arange(n, dtype=np.int32)), "yhat_lower": pa.array(np.zeros(n)),
         "yhat_upper": pa.array(np.ones(n)), "yhat_q0.1": pa.array(np.full(n, 0.25)), "yhat_q0.9": pa.array(np.full(n, 0.75))}
    return Frame(pa.table(t))


def test_convert_forecasts_passes_the_quantile_columns_and_the_gpu_writer_refuses_them():
    f = _forecast_frame()
    conv = ps.ProphetScorer.convert_forecasts(f)
    assert conv.table.column_names == ["created_timestamp", "series_id", "dim_id", "forecast_date", "forecast_timestamp",
                                       "forecast_quantity", "yhat_lower", "yhat_upper", "yhat_q0.1", "yhat_q0.9"]
    assert conv.table["yhat_q0.9"].equals(f.table["yhat_q0.9"])
    assert "standard six" in ps._gpu_writer_refusal(conv, big_only=False)


# ---------------------------------------------------------------------------------------------------------------------
# backtest.quantiles
# ---------------------------------------------------------------------------------------------------------------------
def _cfg(quantile_metrics=True, **bt):
    io = {"metrics": "/tmp/m"}
    if quantile_metrics:
        io["quantile_metrics"] = "/tmp/qm"
    return {"io": io, "model": {"floor": 0, "cap_multiplier": 1.1}, "backtest": {"horizon": "2 days", **bt}}


@pytest.mark.parametrize("bad", BAD_LEVELS)
def test_backtest_refuses_bad_levels_naming_the_key(bad):
    with pytest.raises(ValueError, match=r"backtest\.quantiles"):
        pb.backtest_spec_from_config(_cfg(quantiles=bad))


def test_backtest_needs_its_output_and_refuses_aggregate():
    with pytest.raises(ValueError, match=r"backtest\.quantiles.*io\.quantile_metrics"):
        pb.backtest_spec_from_config(_cfg(quantile_metrics=False, quantiles=[0.5]))
    cfg = _cfg(quantiles=[0.5], aggregate="1D")
    cfg["io"]["window_metrics"] = "/tmp/wm"
    with pytest.raises(ValueError, match=r"backtest\.quantiles.*backtest\.aggregate"):
        pb.backtest_spec_from_config(cfg)


def test_backtest_spec_with_and_without_the_key():
    base = pb.backtest_spec_from_config(_cfg())
    assert base["quantiles"] is None and base["uncertainty_samples"] == 0
    spec = pb.backtest_spec_from_config(_cfg(quantiles=[0.9, 0.1], uncertainty_samples=300, seed=4))
    assert spec["quantiles"] == [0.9, 0.1] and spec["uncertainty_samples"] == 300 and spec["seed"] == 4
    assert spec["intervals"] is False and spec["interval_width"] == 0.8
    assert {k: v for k, v in spec.items() if k not in ("quantiles", "uncertainty_samples", "seed")} == \
        {k: v for k, v in base.items() if k not in ("quantiles", "uncertainty_samples", "seed")}
    with pytest.raises(ValueError, match=r"backtest\.uncertainty_samples"):
        pb.backtest_spec_from_config(_cfg(quantiles=[0.5], uncertainty_samples=1))


# ---------------------------------------------------------------------------------------------------------------------
# the references
# ---------------------------------------------------------------------------------------------------------------------
def _draws(seed, n=1000, H_=12):
    rng = np.random.RandomState(seed)
    d = rng.normal(50, 10, (H_, n))
    d[3] = 7.0                                                # a constant point
    d[4, : n // 2] = d[4, 0]                                  # many ties
    return d


@pytest.mark.parametrize("n", [2, 3, 1000, 1024])
@pytest.mark.parametrize("w", [0.0, 0.5, 0.8, 0.95, 1.0])
def test_quantiles_at_the_bound_percentiles_are_the_bounds(n, w):
    d = _draws(n, n)
    lo, hi = mcs.bounds(d, w)
    q = qo.quantiles(d, mcs.percentiles(w))
    scale = np.max(np.abs(d))
    assert np.max(np.abs(q[0] - lo)) <= 1e-12 * scale and np.max(np.abs(q[1] - hi)) <= 1e-12 * scale


def test_quantiles_at_arbitrary_levels_are_numpy_linear():
    d = _draws(1)
    pct = [0.0, 100.0, 50.0, 12.345, 99.9, 0.05, 50.0, 33.3333]
    q = qo.quantiles(d, pct)
    ref = np.percentile(d, pct, axis=1, method="linear")
    assert q.shape == (len(pct), d.shape[0])
    assert np.max(np.abs(q - ref)) <= 1e-12 * np.max(np.abs(d))


def _brute(horizon, y, yq, lv, rw):
    """Literal reading of the rule for one level: sort by horizon (stable), per distinct horizon the mean over w rows,
    all of the horizon's, then smaller horizons nearest first, the last group contributing its mean times the rows it
    still needs; no row where fewer than w rows lie at or below the horizon."""
    n = len(y)
    w = min(n, max(1, int(rw * n)))
    loss = [max(lv * (a - b), (lv - 1.0) * (a - b)) for a, b in zip(y, yq)]
    below = [1.0 if a <= b else 0.0 for a, b in zip(y, yq)]
    hs = sorted(set(int(h) for h in horizon))
    out = {"horizon": [], "pinball": [], "share_below": []}
    for k, h in enumerate(hs):
        need, sp, sb = w, 0.0, 0.0
        for g in range(k, -1, -1):
            idx = [i for i in range(n) if horizon[i] == hs[g]]
            c = len(idx)
            take = min(need, c)
            sp += sum(loss[i] for i in idx) / c * take
            sb += sum(below[i] for i in idx) / c * take
            need -= take
            if need == 0:
                break
        if need > 0:
            continue
        out["horizon"].append(h)
        out["pinball"].append(sp / w)
        out["share_below"].append(sb / w)
    return out


@pytest.mark.parametrize("rw", [0.0, 1e-3, 0.1, 0.35, 1.0])
@pytest.mark.parametrize("seed", range(6))
def test_quantile_metrics_against_brute_force(rw, seed):
    rng = np.random.RandomState(seed)
    n = 1 if seed == 0 else int(rng.randint(2, 60))
    horizon = rng.randint(1, 6, n).astype(np.int64) * H
    y = np.round(rng.normal(0, 3, n), 1)
    levels = [0.1, 0.5, 0.9, 0.0, 1.0]
    yq = np.stack([np.round(y + rng.normal(0, 2, n), 1) for _ in levels])
    yq[:, ::3] = y[::3]                                                      # ties
    got = qo.quantile_metrics(horizon, y, yq, levels, rw)
    for q, lv in enumerate(levels):
        ref = _brute(horizon, y, yq[q], lv, rw)
        assert got[q]["horizon"].tolist() == ref["horizon"]
        np.testing.assert_allclose(got[q]["pinball"], ref["pinball"], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(got[q]["share_below"], ref["share_below"], rtol=1e-12, atol=1e-15)
        # no horizon group split by the window (w rows end exactly at a group boundary): the share is exact
        w = min(n, max(1, int(rw * n)))
        counts = {h: int(np.sum(horizon == h)) for h in set(horizon.tolist())}
        hs = sorted(counts)
        for k, h in enumerate(got[q]["horizon"]):
            kk = hs.index(h)
            cum = np.cumsum([counts[x] for x in hs[kk::-1]])
            if w in cum.tolist():
                rows = np.isin(horizon, hs[kk - int(np.searchsorted(cum, w)):kk + 1])
                assert got[q]["share_below"][k] == np.sum(y[rows] <= yq[q][rows]) / w
