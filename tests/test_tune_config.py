"""CPU tests of the tuning job's configuration (jobs/prophet_tuner.py: the ``tune`` section) and of its tuning table."""
import itertools

import numpy as np
import pytest

from time_series_spark_b200 import batched
from time_series_spark_b200.jobs import prophet_tuner as pt


def _cfg(**tune):
    return {"model": {"floor": 0, "cap_multiplier": 1.1}, "backtest": {"horizon": "1 days"}, "tune": tune}


def test_defaults_are_the_documented_grid():
    spec = pt.tune_spec_from_config({"model": {}})
    assert spec["metric"] == "rmse"
    assert spec["grid"] == list(itertools.product([0.001, 0.01, 0.1, 0.5], [0.01, 0.1, 1.0, 10.0]))
    assert pt.tune_spec_from_config(_cfg()) == spec


def test_grid_order_and_metric():
    spec = pt.tune_spec_from_config(_cfg(changepoint_prior_scale=[0.5, 0.05], seasonality_prior_scale=[1, 3.0], metric="mape"))
    assert spec["grid"] == [(0.5, 1.0), (0.5, 3.0), (0.05, 1.0), (0.05, 3.0)]
    assert spec["metric"] == "mape"
    for m in ("mse", "rmse", "mae"):
        assert pt.tune_spec_from_config(_cfg(metric=m))["metric"] == m


@pytest.mark.parametrize("key", ["changepoint_prior_scale", "seasonality_prior_scale"])
@pytest.mark.parametrize("value", [[], "0.1", 0.1, None, ["a"], [0.1, "x"], [True], [0.1, 0.0], [-1.0], [float("nan")],
                                   [float("inf")]])
def test_bad_scale_lists_name_the_key(key, value):
    with pytest.raises(ValueError, match=f"tune.{key}"):
        pt.tune_spec_from_config(_cfg(**{key: value}))


@pytest.mark.parametrize("metric", ["coverage", "smape", "RMSE", None, 1])
def test_bad_metric_names_the_key(metric):
    with pytest.raises(ValueError, match="tune.metric"):
        pt.tune_spec_from_config(_cfg(metric=metric))


def test_tuning_table_rows_and_fallback():
    grid = np.array([(0.01, 0.1), (0.01, 10.0), (0.5, 0.1)])
    scores = np.array([[3.0, 2.0, 2.0], [np.nan, 1.0, 5.0], [np.inf, np.nan, 1.0]])
    eligible = np.array([[True, True, True], [False, False, False], [False, False, True]])
    res = batched.TuneResult(grid, scores, eligible, np.array([1, -1, 2]), None, None, None)
    t = pt.tuning_table(np.array([7, 8, 9]), np.array([1, 2, 3]), res, "rmse", (0.05, 10.0))
    assert t.schema.names == ["series_id", "dim_id", "changepoint_prior_scale", "seasonality_prior_scale", "rmse", "selected"]
    assert t["series_id"].to_pylist() == [7, 7, 7, 8, 8, 8, 8, 9, 9, 9]
    assert t["dim_id"].to_pylist() == [1, 1, 1, 2, 2, 2, 2, 3, 3, 3]
    assert t["changepoint_prior_scale"].to_pylist() == [0.01, 0.01, 0.5, 0.01, 0.01, 0.5, 0.05, 0.01, 0.01, 0.5]
    assert t["seasonality_prior_scale"].to_pylist() == [0.1, 10.0, 0.1, 0.1, 10.0, 0.1, 10.0, 0.1, 10.0, 0.1]
    r = t["rmse"].to_numpy(zero_copy_only=False)
    assert r[:3].tolist() == [3.0, 2.0, 2.0] and np.isnan(r[3:9]).all() and r[9] == 1.0
    assert t["selected"].to_pylist() == [False, True, False, False, False, False, True, False, False, True]
