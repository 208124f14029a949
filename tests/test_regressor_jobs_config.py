"""Extra regressors in the jobs without a GPU (DESIGN §20): the modeler's YAML keys and their errors, the input and
future-value readers, the version-4 model record, and every refusal raising before a GPU context is made."""
import os

import numpy as np
import pyarrow as pa
import pytest

from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, model_record
from time_series_spark_b200.jobs import prophet_backtest as pb
from time_series_spark_b200.jobs import prophet_modeler as pm
from time_series_spark_b200.jobs import prophet_scorer as ps
from time_series_spark_b200.jobs import prophet_tuner as pt

REGS = [{"name": "promo"}, {"name": "price", "standardize": True, "prior_scale": 0.5}]
MONTHLY = dict(name="monthly", period=30.5, fourier_order=5)


def _fitted(opts, n=4, seed=0, reg=True):
    lay = L.get_layout(opts)
    rng = np.random.RandomState(seed)
    R = batched.n_regressors(opts)
    return batched.FittedBatch(rng.rand(n, lay.pstride), rng.rand(n, lay.smax), rng.randint(0, 99, (n, 8)).astype(np.int32),
                               rng.randint(0, 2**40, (n, 2)), rng.rand(n, 4), lay.smax, lay.kmax,
                               reg_scale=rng.rand(n, R, 2) if reg and R else None)


def _concat(*cols):
    return pa.chunked_array([c for col in cols for c in (col.chunks if isinstance(col, pa.ChunkedArray) else [col])])


def _models(*parts):
    cols = [model_record.encode(_fitted(o, n=k, seed=j), np.zeros(k, np.int64), o) for j, (o, k) in enumerate(parts)]
    n = sum(k for _, k in parts)
    return pa.table({"series_id": pa.array(np.arange(n), pa.int32()), "dim_id": pa.array(np.zeros(n), pa.int32()),
                     "floor": pa.array(np.zeros(n), pa.float32()), "cap": pa.array(np.full(n, 9.0), pa.float32()),
                     "model": _concat(*cols)})


def test_options_are_make_regressor_options():
    o = pm.options_from_config({"model": {"regressors": REGS, "holidays_prior_scale": 4.0, "seasonalities": [MONTHLY],
                                          "growth": "linear", "n_changepoints": 5}})
    want = batched.make_regressor_options(regressors=REGS, holidays_prior_scale=4.0, seasonalities=[MONTHLY],
                                          growth="linear", n_changepoints=5)
    assert bytes(o)[:C_SIZE_V3_HEAD] == bytes(want)[:C_SIZE_V3_HEAD]
    assert batched.n_regressors(o) == 2 and o.holidays_prior_scale == 4.0
    assert [(o.regressors[i].name, o.regressors[i].prior_scale, o.regressors[i].standardize) for i in range(2)] == \
        [(b"promo", 0.0, L.STD_AUTO), (b"price", 0.5, 1)]


# the bytes of pb200_options_v3 before its pointers (the seasonality table pointer sits inside the v2 part)
C_SIZE_V3_HEAD = L.OptionsV2.seasonalities.offset


@pytest.mark.parametrize("model", [{}, {"regressors": []}, {"holidays_prior_scale": 3.0},
                                   {"regressors": [], "seasonalities": [MONTHLY]}])
def test_without_regressors_the_options_are_the_parents(model):
    rest = {k: v for k, v in model.items() if k not in ("regressors", "holidays_prior_scale")}
    a, b = pm.options_from_config({"model": model}), pm.options_from_config({"model": rest})
    assert type(a) is type(b) and batched.seasonality_table(a) == batched.seasonality_table(b)
    # the bytes up to the table pointer (a v1 options has none)
    assert bytes(a)[:C_SIZE_V3_HEAD] == bytes(b)[:C_SIZE_V3_HEAD]


@pytest.mark.parametrize("model, match", [
    ({"regressors": "promo"}, r"model\.regressors must be a list"),
    ({"regressors": [{"name": "a"}, {"prior_scale": 1}]}, r"model\.regressors\[1\]\.name is required"),
    ({"regressors": [{"name": "a"}, {"name": "b", "standardize": "yes"}]}, r"model\.regressors\[1\]\.standardize"),
    ({"regressors": [{"name": "a", "prior_scale": 0}]}, r"model\.regressors\[0\]\.prior_scale"),
    ({"regressors": [{"name": "a", "colour": 1}]}, r"model\.regressors\[0\]: unknown"),
    ({"regressors": [{"name": "a", "mode": "additive"}]}, r"model\.regressors\[0\]\.mode.*model\.seasonality_mode"),
    ({"regressors": [{"name": "a"}, {"name": "a"}]}, r"model\.regressors\[1\]\.name: regressor 'a' is added twice"),
    ({"regressors": [{"name": "monthly"}], "seasonalities": [MONTHLY]}, r"model\.regressors\[0\]\.name.*seasonality"),
    ({"regressors": [{"name": "a"}], "holidays_prior_scale": 0}, r"model\.holidays_prior_scale"),
    ({"regressors": [{"name": f"r{i}"} for i in range(17)]}, r"model\.regressors: at most 16"),
    ({"regressors": [{"name": "y"}]}, r"model\.regressors\[0\]\.name: 'y' is reserved"),
    ({"regressors": [{"name": "ds"}]}, r"model\.regressors\[0\]\.name: 'ds' is reserved"),
])
def test_yaml_errors_name_the_key(model, match):
    with pytest.raises(ValueError, match=match):
        pm.options_from_config({"model": model})


@pytest.mark.parametrize("name", ["series_id", "dim_id", "start_time", "quantity"])
def test_names_of_input_columns_are_refused(name):
    with pytest.raises(ValueError, match=r"model\.regressors\[1\]\.name: .* column of the modeler's input"):
        pm.options_from_config({"model": {"regressors": [{"name": "promo"}, {"name": name}]}})


def test_input_reader_takes_the_regressor_columns(tmp_path):
    for sid, lines in ((7, ["1,2020-01-01 00:00:00,5,1,2.5", "1,2020-01-01 00:15:00,,0,", "2,2020-01-01 00:00:00,3,,9"]),
                       (8, ["1,2020-01-02 00:00:00,4,1,1e3"])):
        d = tmp_path / "input" / f"series_id={sid}"
        os.makedirs(d)
        (d / "part.csv").write_text("\n".join(lines) + "\n")
    cfg = {"io": {"input": str(tmp_path / "input")}, "model": {"regressors": REGS}}
    t = pm.ProphetModeler(cfg).read_input_dataframe().table.sort_by([("series_id", "ascending"), ("dim_id", "ascending"),
                                                                    ("ds", "ascending")])
    assert t.column_names == ["series_id", "dim_id", "ds", "y", "promo", "price"]
    assert t.schema.field("promo").type == pa.float64() and t.schema.field("price").type == pa.float64()
    assert t["y"].to_pylist() == [5, None, 3, 4]
    assert t["promo"].to_pylist() == [1.0, 0.0, None, 1.0]
    assert t["price"].to_pylist() == [2.5, None, 9.0, 1000.0]


def test_future_reader_filters_the_series(tmp_path):
    for sid in (3, 4, 5):
        d = tmp_path / "fut" / f"series_id={sid}"
        os.makedirs(d)
        (d / "part.csv").write_text(f"0,2021-03-01 00:00:00,1,{sid}.5\n0,2021-03-01 01:00:00,,7\n")
    t = ps.read_future_regressors(str(tmp_path / "fut"), ["promo", "price"], np.array([5, 3, 5]))
    t = t.sort_by([("series_id", "ascending"), ("ds", "ascending")])
    assert t.column_names == ["series_id", "dim_id", "ds", "promo", "price"]
    assert t["series_id"].to_pylist() == [3, 3, 5, 5]
    assert t["promo"].to_pylist() == [1.0, None, 1.0, None]
    assert t["price"].to_pylist() == [3.5, 7.0, 5.5, 7.0]


@pytest.mark.parametrize("kw", [dict(regressors=REGS), dict(regressors=[{"name": "t"}], seasonalities=[MONTHLY],
                                                            yearly_seasonality=False, holidays_prior_scale=2.0,
                                                            growth="linear", seasonality_mode="additive",
                                                            n_changepoints=3)])
def test_v4_round_trip_rebuilds_the_fit_options(kw):
    o = batched.make_regressor_options(**kw)
    fb = _fitted(o, n=5)
    col = model_record.encode(fb, np.arange(5, dtype=np.int64), o)
    assert {int.from_bytes(b[4:6], "little") for b in col.to_pylist()} == {4}
    d, last, info = model_record.decode(col)
    assert last.tolist() == list(range(5))
    for f in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64", "reg_scale"):
        assert getattr(d, f).tobytes() == getattr(fb, f).tobytes(), f
    assert info["holidays_prior_scale"] == kw.get("holidays_prior_scale", 10.0)
    assert [r["name"] for r in info["regressors"]] == [r["name"] for r in kw["regressors"]]
    o2 = model_record.regressor_options(info)
    assert bytes(o2)[:C_SIZE_V3_HEAD] == bytes(o)[:C_SIZE_V3_HEAD]
    assert batched.seasonality_table(o2) == batched.seasonality_table(o)
    assert model_record._regressor_spec(o2) == model_record._regressor_spec(o)
    assert _concat(model_record.encode(d, last, o2)).to_pylist() == col.to_pylist()


def test_v1_and_v2_bytes_do_not_change():
    # the version-1 and version-2 layouts, written out field by field
    for o, tail in ((batched.make_options(), 0), (batched.make_table_options(seasonalities=[MONTHLY]), 16 + 36 * 8)):
        fb = _fitted(o, n=3)
        blob = _concat(model_record.encode(fb, np.arange(3, dtype=np.int64), o)).to_pylist()
        assert {int.from_bytes(b[4:6], "little") for b in blob} == {1 if not tail else 2}
        pstride = 3 + fb.smax + fb.kmax
        assert len(blob[0]) == 4 + 2 + 2 + 4 + 4 + 16 + 32 + 16 + 8 + 32 + 8 * pstride + 8 * fb.smax + tail
        assert blob[1][-tail - 8 * fb.smax - 8 * pstride:len(blob[1]) - tail - 8 * fb.smax] == fb.params[1].tobytes()


def test_encode_refuses_a_fit_without_its_scales():
    o = batched.make_regressor_options(regressors=REGS)
    with pytest.raises(ValueError, match="reg_scale"):
        model_record.encode(_fitted(o, reg=False), np.zeros(4, np.int64), o)
    fb = _fitted(o)
    fb.reg_scale = fb.reg_scale[:, :1]
    with pytest.raises(ValueError, match="reg_scale has shape"):
        model_record.encode(fb, np.zeros(4, np.int64), o)


def test_decode_refuses_mixed_classes_and_specs():
    v4 = batched.make_regressor_options(regressors=REGS)
    v1 = batched.make_options()
    v2 = batched.make_table_options(seasonalities=[MONTHLY])
    for other in (v1, v2):
        for a, b in ((v4, other), (other, v4)):
            with pytest.raises(ValueError, match="version-4 model records with records of another version"):
                model_record.decode(_models((a, 2), (b, 2))["model"])
    # the v1 / v2 mix keeps its message
    with pytest.raises(ValueError, match="version-1 and version-2 model records in one table"):
        model_record.decode(_models((v1, 2), (v2, 2))["model"])
    spec = batched.make_regressor_options(regressors=[REGS[0], dict(REGS[1], standardize="auto")])
    with pytest.raises(ValueError, match="different regressors"):
        model_record.check_one_class(_models((v4, 2), (spec, 2))["model"])
    hps = batched.make_regressor_options(regressors=REGS, holidays_prior_scale=3.0)
    with pytest.raises(ValueError, match="different regressors"):
        model_record.decode(_models((v4, 2), (hps, 2))["model"])
    tab = batched.make_regressor_options(regressors=REGS, seasonalities=[MONTHLY])
    with pytest.raises(ValueError, match="different seasonality tables"):
        model_record.check_one_class(_models((v4, 2), (tab, 2))["model"])
    # other layouts (n_changepoints) of one spec are one class
    model_record.check_one_class(_models((v4, 2), (batched.make_regressor_options(regressors=REGS, n_changepoints=3), 2))
                                 ["model"])


class _NoGpu(Exception):
    pass


@pytest.fixture
def no_context(monkeypatch):
    """Any attempt to make a GPU context fails the test: the refusals must come first."""
    def boom(*a, **k):
        raise _NoGpu("a GPU context was requested")
    for mod in (pm, ps, pb, pt):
        monkeypatch.setattr(mod, "get_context", boom)
    return boom


def _input_table():
    return pa.table({"series_id": pa.array([1, 1], pa.int32()), "dim_id": pa.array([0, 0], pa.int32()),
                     "ds": pa.array([0, 10**9], pa.timestamp("ns")), "y": pa.array([1, 2], pa.int32()),
                     "promo": pa.array([0.0, 1.0]), "price": pa.array([1.0, 2.0])})


def test_modeler_refusals_come_first(no_context):
    base = {"model": {"floor": 0, "cap_multiplier": 1.1, "regressors": REGS}}
    cfg = dict(base, io={"warm_start": "/nonexistent/models", "models": "/nonexistent/out"})
    with pytest.raises(ValueError, match=r"io\.warm_start .*model\.regressors"):
        pm.model_time_series(cfg).apply_batched(_input_table(), ["series_id", "dim_id"])
    cfg["insample"] = {"interval_width": 0.8, "refit": True}
    with pytest.raises(ValueError, match=r"io\.warm_start .*model\.regressors.*insample\.refit"):
        pm.model_time_series(cfg).apply_batched(_input_table(), ["series_id", "dim_id"])
    cfg = dict(base, io={"fitted": "/nonexistent/f"}, insample={"interval_width": 0.8})
    with pytest.raises(ValueError, match=r"insample is not available with model\.regressors"):
        pm.model_time_series(cfg).apply_batched(_input_table(), ["series_id", "dim_id"])
    cfg = {"model": {"floor": 0, "cap_multiplier": 1.1, "regressors": [{"name": "a", "standardize": 2}]}}
    with pytest.raises(ValueError, match=r"model\.regressors\[0\]\.standardize"):
        pm.model_time_series(cfg).apply_batched(_input_table(), ["series_id", "dim_id"])


def test_tuner_and_backtest_modes_refuse_regressors(no_context):
    cfg = {"model": {"floor": 0, "cap_multiplier": 1.1, "regressors": REGS}, "backtest": {"horizon": "1 days"},
           "io": {}}
    with pytest.raises(ValueError, match=r"model\.regressors: the tuner"):
        pt.ProphetTuner(cfg).tune(None)
    for bt, io, key in (({"aggregate": "6h"}, {"window_metrics": "/w"}, "aggregate"),
                        ({"quantiles": [0.5]}, {"quantile_metrics": "/q"}, "quantiles")):
        c = dict(cfg, backtest=dict({"horizon": "1 days"}, **bt), io=io)
        with pytest.raises(ValueError, match=rf"backtest\.{key} is not available with model\.regressors"):
            pb.ProphetBacktester(c).backtest(_input_table())


def test_plan_options_are_the_v2_part():
    o = batched.make_regressor_options(regressors=REGS, seasonalities=[MONTHLY])
    p = batched.plan_options(o)
    assert type(p) is L.OptionsV2 and p.abi_version == L.ABI_VERSION_TABLE
    assert batched.seasonality_table(p) == batched.seasonality_table(o) and batched.n_regressors(p) == 0
    assert bytes(p)[:C_SIZE_V3_HEAD] == bytes(o)[:C_SIZE_V3_HEAD].replace(b"\x03", b"\x02", 1)
    d = batched.make_options()
    assert batched.plan_options(d) is d


class _Prophet05:
    """fbprophet 0.5's handling of extra regressors, step by step in pandas: add_regressor's entry, initialize_scales,
    setup_dataframe's standardisation and prophet_copy's deep copy of extra_regressors."""

    def __init__(self, standardize):
        self.extra_regressors = {f"r{i}": {"standardize": s, "mu": 0.0, "std": 1.0} for i, s in enumerate(standardize)}

    def initialize_scales(self, df):
        for name, props in self.extra_regressors.items():
            standardize = props["standardize"]
            n_vals = len(df[name].unique())
            if n_vals < 2:
                standardize = False
            if standardize == "auto":
                standardize = set(df[name].unique()) != {1, 0}
            if standardize:
                props["mu"] = df[name].mean()
                props["std"] = df[name].std()

    def setup_dataframe(self, df):
        df = df.copy()
        for name, props in self.extra_regressors.items():
            df[name] = (df[name] - props["mu"]) / props["std"]
        return df

    def prophet_copy(self):
        import copy
        m = _Prophet05([])
        m.extra_regressors = copy.deepcopy(self.extra_regressors)
        return m


def test_prophet_copy_scales_are_the_host_rule():
    import pandas as pd
    rng = np.random.RandomState(5)
    T, cut = 200, 120
    cols = {
        "flag": ((np.arange(T) // 7) % 2).astype(float),                              # binary: never standardised
        "price": np.where(np.arange(T) < cut, 4.0, 4.0 + rng.rand(T)),                 # constant before the cutoff
        "forced": np.where(np.arange(T) < cut, 2.5, rng.rand(T)),                      # standardize: true, constant prefix
        "temp": 10 + rng.randn(T),                                                     # standardised at both
        "one": np.where(np.arange(T) < cut, 0.0, 1.0),                                 # 0/1 overall, one value before
    }
    stdz = ["auto", "auto", True, "auto", "auto"]
    df = pd.DataFrame({f"r{i}": v for i, v in enumerate(cols.values())})
    m = _Prophet05(stdz)
    m.initialize_scales(df)
    history = m.setup_dataframe(df)
    full = np.array([[m.extra_regressors[f"r{i}"]["mu"], m.extra_regressors[f"r{i}"]["std"]] for i in range(5)])
    mc = m.prophet_copy()
    mc.initialize_scales(history.iloc[:cut])
    want = np.array([[mc.extra_regressors[f"r{i}"]["mu"], mc.extra_regressors[f"r{i}"]["std"]] for i in range(5)])
    x = np.stack(list(cols.values()))
    # the library's restatement: the full scales from x, z from them, the cutoff's scales from z with the copy
    fs = batched.regressor_scales(x, [0, T], stdz)[0]
    np.testing.assert_allclose(fs, full, rtol=1e-13, atol=0)
    z = (x - fs[:, :1]) / fs[:, 1:]
    got = batched.regressor_scales(z[:, :cut], [0, cut], stdz, copy=fs[None])[0]
    kept = [0, 1, 2, 4]                                      # not standardised at the cutoff: the copied full scales
    assert (got[kept] == fs[kept]).all()
    assert got[1, 1] != 1.0 and (got[[0, 4]] == [0.0, 1.0]).all()
    np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-15)
    # the constant-before-cutoff price is fitted on ((x - mu_full) / std_full - mu_full) / std_full
    zz = (z[1, :cut] - got[1, 0]) / got[1, 1]
    np.testing.assert_allclose(zz, ((cols["price"][:cut] - full[1, 0]) / full[1, 1] - full[1, 0]) / full[1, 1], rtol=1e-14)


@pytest.mark.parametrize("fc, io, match", [
    ({"components": True}, {"future_regressors": "/x"}, r"forecast\.components is not available"),
    ({"aggregate": "1D"}, {"future_regressors": "/x", "aggregates": "/a"}, r"forecast\.aggregate is not available"),
    ({"aggregate_period": "M"}, {"future_regressors": "/x", "aggregates": "/a"},
     r"forecast\.aggregate_period is not available"),
    ({"quantiles": [0.5]}, {"future_regressors": "/x"}, r"forecast\.quantiles is not available"),
    ({}, {}, r"io\.future_regressors is required"),
])
def test_scorer_refusals_come_first(no_context, fc, io, match):
    models = _models((batched.make_regressor_options(regressors=REGS), 3))
    op = ps.forecast_time_series({"io": io, "forecast": dict({"periods": 3, "frequency": "D"}, **fc)})
    with pytest.raises(ValueError, match=match):
        op.apply_batched(models, ["series_id", "dim_id"])


def test_scorer_refuses_future_values_for_other_models(no_context):
    for o in (batched.make_options(), batched.make_table_options(seasonalities=[MONTHLY])):
        op = ps.forecast_time_series({"io": {"future_regressors": "/x"}, "forecast": {"periods": 3, "frequency": "D"}})
        with pytest.raises(ValueError, match=r"io\.future_regressors is given, but the models have no extra regressors"):
            op.apply_batched(_models((o, 2)), ["series_id", "dim_id"])


def test_every_rank_refuses_what_the_whole_table_refuses(no_context):
    import time_series_spark_b200.dist as pdist
    v4 = batched.make_regressor_options(regressors=REGS)
    spec = batched.make_regressor_options(regressors=REGS[:1])
    op = ps.forecast_time_series({"io": {"future_regressors": "/x"}, "forecast": {"periods": 3, "frequency": "D"}})
    orig = pdist.world
    try:
        for rank in (0, 1):
            pdist.world = lambda: (rank, 2, rank)
            with pytest.raises(ValueError, match="different regressors"):
                op.apply_batched(_models((v4, 3), (spec, 3)), ["series_id", "dim_id"])
            with pytest.raises(ValueError, match="version-4 model records with records of another version"):
                op.apply_batched(_models((v4, 3), (batched.make_options(), 3)), ["series_id", "dim_id"])
    finally:
        pdist.world = orig


def test_example_configs_are_ones_the_jobs_take():
    import yaml
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "config")
    with open(os.path.join(root, "example_regressors_modeler_app_config.yaml")) as f:
        cfg = yaml.safe_load(f)
    o = pm.options_from_config(cfg)
    assert batched.n_regressors(o) == len(cfg["model"]["regressors"]) >= 2
    with open(os.path.join(root, "example_regressors_scorer_app_config.yaml")) as f:
        sc = yaml.safe_load(f)
    assert sc["io"]["future_regressors"] and sc["io"]["models"] == cfg["io"]["models"]
    ps.refuse_regressor_modes(sc, True)
    with open(os.path.join(root, "example_regressors_backtest_app_config.yaml")) as f:
        bt = yaml.safe_load(f)
    assert batched.n_regressors(pm.options_from_config(bt)) == 2
    spec = pb.backtest_spec_from_config(bt)
    assert spec["aggregate"] is None and spec["quantiles"] is None
