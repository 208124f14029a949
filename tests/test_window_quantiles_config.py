"""Quantiles of window and period totals (DESIGN §21) without a GPU: the jobs' keys, their refusals (each names its key
and comes before any GPU context), the io.aggregates / window outputs' columns and empty-shard schemas, configs
without the keys left as they were, the library's declarations, and the CPU reference the GPU tests hold the planes to.
"""
import os
import re

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

import quantile_oracle as qo
import window_oracle as wo
import period_oracle as pdo
import window_quantile_oracle as wqo
from oracle import mc_stream as mcs
from oracle import prophet_oracle as po
import test_lib_prototypes as tlp
from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched
from time_series_spark_b200.jobs import prophet_backtest as pb
from time_series_spark_b200.jobs import prophet_scorer as ps

H_NS = 3600 * 10**9
DAY = 24 * H_NS


def _window_quantile_declarations():
    path = os.path.join(os.path.dirname(tlp.HEADER), "prophet_b200_window_quantiles.h")
    with open(path) as f:
        text = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return {name: (tlp._c_kind(ret), [tlp._c_kind(q) for q in " ".join(params.split()).split(",")])
            for ret, name, params in tlp.DECL.findall(text)}


def test_window_quantile_header_matches_the_library():
    """include/prophet_b200_window_quantiles.h declares the five entry points, each its sums twin's arguments plus
    n_q, h_percentiles and d_sum_quantiles; the library exports them with ctypes prototypes of the same kinds."""
    decl = _window_quantile_declarations()
    assert sorted(decl) == sorted(L.WINDOW_QUANTILE_EXPORTS) and not set(decl) & set(tlp.DECLARATIONS)
    lib = L.load()
    for name, (ret, params) in decl.items():
        twin = name.replace("_quantiles", "")
        assert ret == "int32" and params == tlp.DECLARATIONS[twin][1] + ["int32", "pointer", "pointer"], name
        f = getattr(lib, name)
        assert [tlp._ctypes_kind(t) for t in f.argtypes] == params and tlp._ctypes_kind(f.restype) == ret, name


# ---------------------------------------------------------------------------------------------------------------------
# refusals: each names its key, and none needs a GPU context
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def no_gpu(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("a GPU context was requested")
    monkeypatch.setattr(ps, "get_context", refuse)
    monkeypatch.setattr(pb, "get_context", refuse)
    monkeypatch.setattr(L.Context, "__init__", refuse)
    monkeypatch.setattr(ps.pdist, "init_process_group", refuse)


def _scorer_cfg(**fc):
    return {"io": {"models": "m", "forecasts": "f", "aggregates": "a"},
            "forecast": {"periods": 4, "frequency": "h", **fc}}


SCORER_BAD = [
    (dict(aggregate_quantiles=[0.5]), r"forecast\.aggregate_quantiles needs forecast\.aggregate"),
    (dict(aggregate="1D", aggregate_quantiles=0.5), r"forecast\.aggregate_quantiles must be a list"),
    (dict(aggregate="1D", aggregate_quantiles=[]), r"forecast\.aggregate_quantiles must be a list"),
    (dict(aggregate="1D", aggregate_quantiles=[0.5] * 33), r"forecast\.aggregate_quantiles must be a list"),
    (dict(aggregate="1D", aggregate_quantiles=[1.5]), r"forecast\.aggregate_quantiles must hold levels"),
    (dict(aggregate="1D", aggregate_quantiles=[-0.1]), r"forecast\.aggregate_quantiles must hold levels"),
    (dict(aggregate="1D", aggregate_quantiles=[float("nan")]), r"forecast\.aggregate_quantiles must hold levels"),
    (dict(aggregate="1D", aggregate_quantiles=[True]), r"forecast\.aggregate_quantiles must hold levels"),
    (dict(aggregate="1D", aggregate_quantiles=["0.5"]), r"forecast\.aggregate_quantiles must hold levels"),
    (dict(aggregate_period="M", aggregate_quantiles=[0.5, 0.5]), r"forecast\.aggregate_quantiles names a level twice"),
]


@pytest.mark.parametrize("fc,match", SCORER_BAD)
def test_scorer_refusals_name_the_key_before_any_gpu_context(no_gpu, fc, match):
    cfg = _scorer_cfg(**fc)
    with pytest.raises(ValueError, match=match):
        ps.aggregate_quantiles(cfg)
    with pytest.raises(ValueError, match=match):
        ps.ProphetScorer.score(None, cfg)


def test_scorer_keeps_refusing_quantiles_with_the_aggregate_keys(no_gpu):
    for fc in (dict(aggregate="1D", quantiles=[0.5], aggregate_quantiles=[0.5]),
               dict(aggregate_period="M", quantiles=[0.5], aggregate_quantiles=[0.5])):
        with pytest.raises(ValueError, match=r"forecast\.(quantiles|aggregate_period) cannot be combined"):
            ps.ProphetScorer.score(None, _scorer_cfg(**fc))


def test_scorer_accepts_either_aggregate_key():
    assert ps.aggregate_quantiles(_scorer_cfg(aggregate="1D", aggregate_quantiles=[0.9, 0.1, 1])) == [0.9, 0.1, 1.0]
    assert ps.aggregate_quantiles(_scorer_cfg(aggregate_period="Q", aggregate_quantiles=[0.5])) == [0.5]
    assert ps.aggregate_quantiles(_scorer_cfg(aggregate="1D")) is None


def _bt_cfg(io_extra=True, **bt):
    io = {"input": "i", "metrics": "m", "window_metrics": "wm"}
    if io_extra:
        io["window_quantile_metrics"] = "wq"
    return {"io": io, "model": {"floor": 0, "cap_multiplier": 1.1},
            "backtest": {"horizon": "1 days", **bt}}


BACKTEST_BAD = [
    (_bt_cfg(intervals=True, aggregate_quantiles=[0.5]), r"backtest\.aggregate_quantiles needs backtest\.aggregate"),
    (_bt_cfg(aggregate="8h", aggregate_quantiles=[0.5]), r"backtest\.aggregate_quantiles needs backtest\.intervals"),
    (_bt_cfg(io_extra=False, aggregate="8h", intervals=True, aggregate_quantiles=[0.5]),
     r"backtest\.aggregate_quantiles needs io\.window_quantile_metrics"),
    (_bt_cfg(aggregate="8h", intervals=True, aggregate_quantiles=[]), r"backtest\.aggregate_quantiles must be a list"),
    (_bt_cfg(aggregate="8h", intervals=True, aggregate_quantiles=[0.5] * 33),
     r"backtest\.aggregate_quantiles must be a list"),
    (_bt_cfg(aggregate="8h", intervals=True, aggregate_quantiles=[2]), r"backtest\.aggregate_quantiles must hold levels"),
    (_bt_cfg(aggregate="8h", intervals=True, aggregate_quantiles=[0.1, 0.1]),
     r"backtest\.aggregate_quantiles names a level twice"),
]


@pytest.mark.parametrize("cfg,match", BACKTEST_BAD)
def test_backtest_refusals_name_the_key_before_any_gpu_context(no_gpu, cfg, match):
    with pytest.raises(ValueError, match=match):
        pb.backtest_spec_from_config(cfg)
    tbl = pa.table({"series_id": pa.array([1], pa.int32()), "dim_id": pa.array([1], pa.int32()),
                    "ds": pa.array([0], pa.timestamp("ns")), "y": pa.array([1.0])})
    with pytest.raises(ValueError, match=match):
        pb.ProphetBacktester(cfg).backtest(tbl)


def test_backtest_regressors_refuse_the_aggregate_first(no_gpu):
    cfg = _bt_cfg(aggregate="8h", intervals=True, aggregate_quantiles=[0.5])
    cfg["model"]["regressors"] = [{"name": "promo"}]
    tbl = pa.table({"series_id": pa.array([1], pa.int32()), "dim_id": pa.array([1], pa.int32()),
                    "ds": pa.array([0], pa.timestamp("ns")), "y": pa.array([1.0])})
    with pytest.raises(ValueError, match=r"backtest\.aggregate is not available with model\.regressors"):
        pb.ProphetBacktester(cfg).backtest(tbl)


def test_backtest_spec_carries_the_levels():
    spec = pb.backtest_spec_from_config(_bt_cfg(aggregate="8h", intervals=True, aggregate_quantiles=[0.9, 0.1]))
    assert spec["aggregate_quantiles"] == [0.9, 0.1] and spec["aggregate"] == 8 * H_NS


@pytest.mark.parametrize("bt", [{}, dict(aggregate="8h"), dict(aggregate="8h", intervals=True),
                                dict(quantiles=[0.5], intervals=True), dict(intervals=True, uncertainty_samples=10)])
def test_backtest_specs_without_the_key_are_unchanged(bt):
    cfg = _bt_cfg(**bt)
    cfg["io"]["quantile_metrics"] = "q"
    spec = pb.backtest_spec_from_config(cfg)
    assert list(spec) == ["horizon", "period", "initial", "rolling_window", "intervals", "uncertainty_samples",
                          "interval_width", "seed", "aggregate", "quantiles"]


def test_batched_refuses_bad_levels_before_the_library():
    for lv in ([], [0.5] * 33, [1.5], [float("nan")], [[0.5]]):
        with pytest.raises(ValueError, match="levels must be 1 to 32 fractions"):
            batched.predict_sums_host(None, None, None, None, None, None, DAY, levels=lv)
        with pytest.raises(ValueError, match="levels must be 1 to 32 fractions"):
            batched.predict_period_sums_host(None, None, None, None, None, None, 1, 0, levels=lv)


def test_cross_validation_refuses_window_quantiles_without_their_inputs():
    import torch
    ds, y = torch.zeros(4, dtype=torch.int64), torch.zeros(4)
    off = np.array([0, 4])
    for opts, kw in ((batched.make_options(), dict(intervals=True)),
                     (batched.make_options(), dict(aggregate_ns=DAY)),
                     (batched.make_options(uncertainty_samples=0), dict(aggregate_ns=DAY, intervals=True))):
        with pytest.raises(ValueError, match="window_quantiles need aggregate_ns, intervals"):
            batched.cross_validation_device(None, opts, ds, y, off, 0.0, None, DAY, DAY, DAY,
                                            window_quantiles=[0.5], **kw)
    with pytest.raises(ValueError, match="levels must be"):
        batched.cross_validation_device(None, batched.make_options(), ds, y, off, 0.0, None, DAY, DAY, DAY,
                                        intervals=True, aggregate_ns=DAY, window_quantiles=[1.5])


# ---------------------------------------------------------------------------------------------------------------------
# columns and schemas
# ---------------------------------------------------------------------------------------------------------------------
def test_aggregate_schema_and_columns():
    assert ps.aggregate_schema().equals(ps.AGGREGATE_SCHEMA)
    assert ps.aggregate_schema(None).equals(ps.AGGREGATE_SCHEMA)
    s = ps.aggregate_schema([0.9, 0.1, 0.975])
    assert s.names == ps.AGGREGATE_SCHEMA.names + ["yhat_q0.9", "yhat_q0.1", "yhat_q0.975"]
    assert all(s.field(n).type == pa.float64() for n in s.names[-3:])
    # aggregate_table of a WindowQuantiles: the planes gathered to the window rows, after yhat_upper
    n, wmax = 3, 4
    nw = np.array([2, 4, 1], np.int32)
    ok = np.array([True, True, False])
    rng = np.random.RandomState(0)
    f = lambda dt: rng.randint(0, 100, (n, wmax)).astype(dt)                                     # noqa: E731
    qs = rng.randn(2, n, wmax)
    ws = batched.WindowQuantiles(nw, f(np.int64), f(np.int32), f(np.float64), f(np.int64), f(np.float64), f(np.float64),
                                 np.array([0.9, 0.1]), qs)
    t = ps.aggregate_table(np.arange(n, dtype=np.int32), np.ones(n, np.int32), ok, ws)
    assert t.schema.equals(ps.aggregate_schema([0.9, 0.1]))
    keep = (np.arange(wmax)[None, :] < nw[:, None]) & ok[:, None]
    assert t.num_rows == 6
    assert t["yhat_q0.9"].to_numpy().tolist() == qs[0][keep].tolist()
    assert t["yhat_q0.1"].to_numpy().tolist() == qs[1][keep].tolist()
    plain = ps.aggregate_table(np.arange(n, dtype=np.int32), np.ones(n, np.int32), ok,
                               batched.WindowSums(*(getattr(ws, fl.name) for fl in batched.fields(batched.WindowSums))))
    assert plain.schema.equals(ps.AGGREGATE_SCHEMA) and t.select(plain.column_names).equals(plain)


@pytest.mark.parametrize("fc", [dict(aggregate="1D"), dict(aggregate_period="M"), dict(aggregate_period="W-SUN")])
def test_scorer_empty_shard_aggregates_schema(fc):
    empty = pa.table({"series_id": pa.array([], pa.int32()), "dim_id": pa.array([], pa.int32()),
                      "floor": pa.array([], pa.float32()), "cap": pa.array([], pa.float32()),
                      "model": pa.array([], pa.binary())})
    op = ps.forecast_time_series(_scorer_cfg(**fc))
    op.apply_batched(empty, ["series_id", "dim_id"])
    assert op.aggregates.num_rows == 0 and op.aggregates.schema.equals(ps.AGGREGATE_SCHEMA)
    op = ps.forecast_time_series(_scorer_cfg(aggregate_quantiles=[0.5, 0.05], **fc))
    op.apply_batched(empty, ["series_id", "dim_id"])
    assert op.aggregates.num_rows == 0 and op.aggregates.schema.equals(ps.aggregate_schema([0.5, 0.05]))


def test_window_output_tables_carry_the_levels():
    levels = [0.1, 0.5]
    w = batched.CvWindows(8 * H_NS, np.array([0, 0, 1]), np.array([5, 5, 7]), np.array([8, 16, 8]) * H_NS,
                          np.array([2, 3, 1], np.int32), np.zeros(3), np.ones(3), np.zeros(3), np.ones(3),
                          {"series": np.array([0, 1]), "horizon": np.array([8, 8]) * H_NS, "mse": np.zeros(2),
                           "rmse": np.zeros(2), "mae": np.zeros(2), "mape": np.zeros(2), "coverage": np.ones(2)},
                          yhat_q=np.arange(6.0).reshape(2, 3),
                          quantile_metrics={"series": np.array([0, 0, 1, 1]), "horizon": np.array([8, 8, 8, 8]) * H_NS,
                                            "level": np.array(levels * 2), "pinball": np.arange(4.0),
                                            "share_below": np.arange(4.0) / 4})
    res = batched.CvResult(np.array([0, 1]), np.array([5, 7]), np.array([0, -1]), np.zeros(2, np.int64),
                           *(np.zeros(0, np.int64),) * 3, np.zeros(0), np.zeros(0), None, None, windows=w)
    _, rows = pb.assemble_window_outputs(np.array([10, 11], np.int32), np.array([1, 1], np.int32), res, True, levels)
    assert rows.column_names[-2:] == ["yhat_q0.1", "yhat_q0.5"] and rows.num_rows == 2   # series 1's fit failed
    assert rows["yhat_q0.5"].to_pylist() == [3.0, 4.0]
    _, plain = pb.assemble_window_outputs(np.array([10, 11], np.int32), np.array([1, 1], np.int32), res, True)
    assert plain.column_names == rows.column_names[:-2]
    t = pb.window_quantile_metrics_table(np.array([10, 11], np.int32), np.array([1, 1], np.int32), res)
    assert t.schema.equals(pb.QUANTILE_METRICS_SCHEMA) and t.num_rows == 2
    assert t["quantile"].to_pylist() == levels and t["pinball_loss"].to_pylist() == [0.0, 1.0]


# ---------------------------------------------------------------------------------------------------------------------
# the CPU reference of the planes
# ---------------------------------------------------------------------------------------------------------------------
def _draws(growth, mode, fut, n, seed=5):
    rng = np.random.RandomState(3)
    ds = np.datetime64("2021-03-01", "ns").astype(np.int64) + H_NS * np.arange(720, dtype=np.int64)
    y = 100 + 10 * rng.rand(ds.size)
    p = po.prepare(ds, y, 0.0, 130.0, po.ProphetOptions(growth=growth, seasonality_mode=mode))
    delta = 0.5 * rng.laplace(size=p.S)
    beta = 0.05 * rng.randn(p.K)
    k, m = (0.8, -0.2) if growth == "logistic" else (0.1, 0.7)
    rec = mcs.stack([mcs.record(p, k, m, 0.02, delta, beta, 25, 14)], 25, 14)
    return mcs.draws(rec, 0, fut, 0.0, 130.0, growth == "logistic", mode == "multiplicative", n, seed)


@pytest.mark.parametrize("growth,mode", [("logistic", "multiplicative"), ("linear", "additive")])
@pytest.mark.parametrize("n", [2, 3, 200])
def test_reference_planes_at_the_bounds_are_the_window_bounds(growth, mode, n):
    last = np.datetime64("2021-03-30T23:00", "ns").astype(np.int64)
    fut = last + H_NS * np.arange(1, 61, dtype=np.int64)
    d = _draws(growth, mode, fut, n)
    for w in (0.0, 0.8, 1.0):
        pct = mcs.percentiles(w)
        pl = wqo.window_quantiles(d, fut, 8 * H_NS, 5 * H_NS, pct)
        _, _, lo, hi = wo.window_sums(d, fut, 8 * H_NS, 5 * H_NS, w)
        np.testing.assert_allclose(pl[0], lo, rtol=1e-13, atol=0)
        np.testing.assert_allclose(pl[1], hi, rtol=1e-13, atol=0)
    fut_m = np.datetime64("2021-03-31", "ns").astype(np.int64) + DAY * np.arange(1, 80, dtype=np.int64)
    dm = _draws(growth, mode, fut_m, n)
    pl = wqo.period_quantiles(dm, fut_m, "M", mcs.percentiles(0.8))
    _, _, lo, hi = pdo.period_sums(dm, fut_m, "M", 0.8)
    np.testing.assert_allclose(pl, np.stack([lo, hi]), rtol=1e-13, atol=0)


def test_reference_one_point_windows_are_the_pointwise_planes():
    last = np.datetime64("2021-03-30T23:00", "ns").astype(np.int64)
    fut = last + H_NS * np.arange(1, 41, dtype=np.int64)
    d = _draws("logistic", "multiplicative", fut, 100)
    pct = [0.0, 2.5, 50.0, 97.5, 100.0, 33.3, 50.0]
    assert wqo.window_quantiles(d, fut, H_NS, 0, pct).tobytes() == qo.quantiles(d, pct).tobytes()
    # a frame of month starts: every calendar month holds one point
    ms = pd.date_range("2021-04-01", periods=12, freq="MS").values.astype("datetime64[ns]").astype(np.int64)
    dm = _draws("linear", "additive", ms, 50)
    assert wqo.period_quantiles(dm, ms, "M", pct).tobytes() == qo.quantiles(dm, pct).tobytes()


def test_example_configs_pass_their_checks():
    import os
    import yaml
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "config")
    with open(os.path.join(root, "example_window_quantile_scorer_app_config.yaml")) as f:
        cfg = yaml.safe_load(f)
    assert ps.aggregate_quantiles(cfg) == [0.5, 0.9, 0.95] and ps.aggregate_rule(cfg) == (DAY, 0)
    with open(os.path.join(root, "example_window_quantile_backtest_app_config.yaml")) as f:
        spec = pb.backtest_spec_from_config(yaml.safe_load(f))
    assert spec["aggregate_quantiles"] == [0.5, 0.9, 0.95] and spec["aggregate"] == DAY and spec["intervals"]


# ---------------------------------------------------------------------------------------------------------------------
# the wrappers' library calls with levels: the sums call's, through the _quantiles twin with three more arguments
# ---------------------------------------------------------------------------------------------------------------------
def _sums_cases():
    from test_batched_calls import CASES
    return {k: v for k, v in CASES.items() if "sums" in k}


@pytest.mark.parametrize("case", sorted(_sums_cases()))
def test_levels_select_the_quantile_twin(monkeypatch, case):
    from test_batched_calls import _run
    fn, inputs = _sums_cases()[case]
    levels = [0.9, 0.1, 0.5]
    ev0, d0, _, _ = _run(monkeypatch, fn, inputs)
    entries = [e[0] for e in ev0 if not isinstance(e, str) and "sums" in e[0]]
    peek = {}
    if entries:
        twin = entries[0].replace("_host", "_quantiles_host").replace("_device", "_quantiles_device")
        peek = {twin: (len(ev0[[e[0] if not isinstance(e, str) else e for e in ev0].index(entries[0])][1]) + 1, (3,))}
    ev1, d1, rec, _ = _run(monkeypatch, fn, dict(inputs, levels=levels), peek)
    if not isinstance(d0, dict):                     # an argument error: the same one, and no call
        assert d1 == d0 and ev1 == ev0
        return
    assert len(ev1) == len(ev0)
    for a, b in zip(ev0, ev1):
        if isinstance(a, str) or "sums" not in a[0]:
            assert a == b
            continue
        planes = "[1].quantiles" if a[1][-1] == "[1].upper" else a[1][-1]      # an empty output has no role
        assert b[0] == twin and b[1] == a[1] + (3, "tmp", planes), (a, b)
    assert [list(v) for v in rec.raw] == [[90.0, 10.0, 50.0]]
    wmax = d0["[1].start"][2][1]
    kind = d0["[1].lower"][0]
    n = d0["[1].n_windows"][2][0]
    assert d1 == dict(d0, **{"[1].levels": ("np", "float64", (3,)),
                             "[1].quantiles": (kind, "float64" if kind == "np" else "torch.float64", (3, n, wmax))})
