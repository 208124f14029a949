"""The modeler's ``insample`` section (DESIGN §16) on the CPU: its keys, defaults and refusals, and the in-sample
reference (tests/insample_oracle.py) on the golden fixture."""
import os
import sys

import numpy as np
import pandas as pd
import pytest
import yaml

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import insample_oracle as io_  # noqa: E402
from oracle import mc_stream as mcs  # noqa: E402
from oracle import prophet_oracle as po  # noqa: E402
from time_series_spark_b200.jobs import prophet_modeler as pm  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(insample, fitted="/tmp/fitted"):
    io = {"input": "in", "models": "models"}
    if fitted:
        io["fitted"] = fitted
    cfg = {"io": io, "model": {"floor": 0, "cap_multiplier": 1.1}}
    if insample is not ...:
        cfg["insample"] = insample
    return cfg


def test_without_the_section_there_is_nothing_to_do():
    assert pm.insample_options(_cfg(..., fitted=None)) is None
    assert pm.insample_options(_cfg(...)) is None


def test_defaults():
    assert pm.insample_options(_cfg({"interval_width": 0.99})) == {
        "interval_width": 0.99, "uncertainty_samples": 1000, "seed": 0, "refit": False}
    got = pm.insample_options(_cfg({"interval_width": 1, "uncertainty_samples": 2, "seed": 7, "refit": True}, fitted=None))
    assert got == {"interval_width": 1.0, "uncertainty_samples": 2, "seed": 7, "refit": True}
    assert pm.insample_options(_cfg({"interval_width": 0, "uncertainty_samples": 1024}))["uncertainty_samples"] == 1024


@pytest.mark.parametrize("sec,key", [
    ({}, "insample.interval_width"),
    ({"uncertainty_samples": 1000}, "insample.interval_width"),
    ({"interval_width": -0.01}, "insample.interval_width"),
    ({"interval_width": 1.5}, "insample.interval_width"),
    ({"interval_width": float("nan")}, "insample.interval_width"),
    ({"interval_width": "0.9"}, "insample.interval_width"),
    ({"interval_width": True}, "insample.interval_width"),
    ({"interval_width": 0.9, "uncertainty_samples": 1}, "insample.uncertainty_samples"),
    ({"interval_width": 0.9, "uncertainty_samples": 1025}, "insample.uncertainty_samples"),
    ({"interval_width": 0.9, "uncertainty_samples": 100.0}, "insample.uncertainty_samples"),
    ({"interval_width": 0.9, "seed": -1}, "insample.seed"),
    ({"interval_width": 0.9, "refit": "yes"}, "insample.refit"),
    ({"interval_width": 0.9, "width": 0.5}, "insample.width"),
    ({"interval_width": 0.9, "outlier_rule": "iqr"}, "insample.outlier_rule"),
    (None, "insample"),
    ([0.9], "insample"),
])
def test_refusals_name_the_key(sec, key):
    with pytest.raises(ValueError, match=key.replace(".", r"\.")):
        pm.insample_options(_cfg(sec))


def test_a_section_that_would_write_nothing_is_refused():
    with pytest.raises(ValueError, match=r"io\.fitted or insample\.refit"):
        pm.insample_options(_cfg({"interval_width": 0.9}, fitted=None))
    with pytest.raises(ValueError, match=r"io\.fitted or insample\.refit"):
        pm.insample_options(_cfg({"interval_width": 0.9, "refit": False}, fitted=None))


def test_example_config_parses():
    with open(os.path.join(ROOT, "config", "example_insample_modeler_app_config.yaml")) as f:
        cfg = yaml.safe_load(f)
    assert pm.insample_options(cfg) == {"interval_width": 0.99, "uncertainty_samples": 1000, "seed": 0, "refit": False}


def test_fitted_schema_keeps_the_input_y_type():
    import pyarrow as pa
    s = pm.fitted_schema(pa.int32())
    assert s.names == ["series_id", "dim_id", "ds", "y", "yhat", "yhat_lower", "yhat_upper", "outlier"]
    assert [str(t) for t in s.types] == ["int32", "int32", "timestamp[ns]", "int32", "double", "double", "double", "bool"]
    assert pm.fitted_schema(pa.float32()).field("y").type == pa.float32()


def test_null_rows_last_ds_per_group():
    import pyarrow as pa
    t = pa.table({"series_id": pa.array([1, 1, 1, 2, 2], pa.int32()), "dim_id": pa.array([5, 5, 5, 5, 6], pa.int32()),
                  "ds": pa.array(np.array([10, 30, 20, 40, 50], "datetime64[s]")),
                  "y": pa.array([1.0, None, np.nan, 3.0, None])})
    got = pm.null_rows_last_ds(t, np.array([1, 2, 2], np.int32), np.array([5, 5, 6], np.int32))
    lo = np.iinfo(np.int64).min
    assert got.tolist() == [30 * 10**9, lo, 50 * 10**9]
    assert pm.null_rows_last_ds(t.slice(3, 1), np.array([2], np.int32), np.array([5], np.int32)).tolist() == [lo]


def test_insample_report_line():
    assert pm.insample_report(816, 12, 2, 0) == ("In-sample: 816 rows predicted, 12 flagged as outliers in 2 series; "
                                                 "0 series refitted without them")


def _golden_fits(gi, go):
    """The golden fixture's groups with the oracle's stored optimum: (dims, ds, y, FitResult, record)."""
    out = []
    lay_smax, lay_kmax = 25, 34
    for dim in (91, 155):
        sel = gi["dim_id"] == dim
        order = np.argsort(gi["ds_ns"][sel], kind="stable")
        ds, y = gi["ds_ns"][sel][order], gi["y"][sel][order]
        p = po.prepare(ds, y.astype(np.float64), 0.0, float(go[f"d{dim}_cap"]), po.ProphetOptions())
        fr = po.FitResult(prep=p, k=float(go[f"d{dim}_k"]), m=float(go[f"d{dim}_m"]), delta=go[f"d{dim}_delta"],
                          sigma_obs=float(go[f"d{dim}_sigma_obs"]), beta=go[f"d{dim}_beta"], theta=None, neg_logp=0.0,
                          iters=0, n_evals=0, ret=0)
        rec = mcs.record(p, fr.k, fr.m, fr.sigma_obs, fr.delta, fr.beta, lay_smax, lay_kmax)
        out.append((dim, ds, y, fr, rec))
    return out


def test_oracle_filtered_batch_is_a_pandas_filter_of_the_input(golden_input, golden_oracle):
    """On the golden fixture: the oracle's in-sample yhat is the fixture's, and the batch without the rows the oracle
    flags (80 % interval, 200 draws) is the input with those rows deleted."""
    fits = _golden_fits(golden_input, golden_oracle)
    stack = mcs.stack([f[4] for f in fits], 25, 34)
    ds_all, y_all, yh_all, lo_all, hi_all, offsets = [], [], [], [], [], [0]
    for i, (dim, ds, y, fr, _) in enumerate(fits):
        yh = io_.yhat(fr, ds, 0.0, fr.prep.cap_value)
        ref = golden_oracle[f"d{dim}_yhat_insample"]
        assert yh.shape == ref.shape and np.max(np.abs(yh - ref)) <= 1e-9 * fr.prep.y_scale
        lo, hi = io_.bounds(stack, i, ds, 0.0, fr.prep.cap_value, True, True, 200, 0.8, 3)
        assert np.all(lo <= hi)
        ds_all.append(ds); y_all.append(y); yh_all.append(yh); lo_all.append(lo); hi_all.append(hi)
        offsets.append(offsets[-1] + ds.size)
    ds_c, y_c = np.concatenate(ds_all), np.concatenate(y_all)
    flag = io_.flags(y_c, np.concatenate(lo_all), np.concatenate(hi_all))
    assert 0 < flag.sum() < flag.size                    # the premise: some rows are flagged, most are not
    kept, off, ds_k, y_k = io_.kept_batch(ds_c, y_c, offsets, flag)
    df = pd.DataFrame({"dim_id": np.repeat([91, 155], np.diff(offsets)), "ds": ds_c, "y": y_c, "outlier": flag})
    want = df[~df["outlier"]]
    assert np.array_equal(ds_k, want["ds"].to_numpy()) and np.array_equal(y_k, want["y"].to_numpy())
    assert y_k.dtype == y_c.dtype
    assert kept.tolist() == want.groupby("dim_id").size().loc[[91, 155]].tolist()
    assert off.tolist() == [0, int(kept[0]), int(kept.sum())]


def test_oracle_flags_never_on_a_nan_bound():
    y = np.array([1, 5, 9], np.int32)
    assert io_.flags(y, np.array([np.nan, 6.0, np.nan]), np.array([0.0, np.nan, np.nan])).tolist() == [True, True, False]
