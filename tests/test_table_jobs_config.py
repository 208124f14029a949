"""Seasonality tables in the jobs without a GPU (DESIGN §18): the version-2 model record, the modeler's YAML keys and
their errors, the warm-start and tuner refusals, the scorer's component columns and the backtest's prophet_copy
options."""
import numpy as np
import pyarrow as pa
import pytest

from time_series_spark_b200 import _lib as L
from time_series_spark_b200 import batched, model_record
from time_series_spark_b200.jobs import prophet_modeler as pm
from time_series_spark_b200.jobs import prophet_scorer as ps
from time_series_spark_b200.jobs import prophet_tuner as pt

MONTHLY = dict(name="monthly", period=30.5, fourier_order=5)
TABLE = dict(seasonalities=[MONTHLY, dict(name="weekly", period=7, fourier_order=2, prior_scale=0.5)],
             yearly_seasonality=12)


def _fitted(opts, n=4, seed=0):
    lay = L.get_layout(opts)
    rng = np.random.RandomState(seed)
    return batched.FittedBatch(rng.rand(n, lay.pstride), rng.rand(n, lay.smax), rng.randint(0, 99, (n, 8)).astype(np.int32),
                               rng.randint(0, 2**40, (n, 2)), rng.rand(n, 4), lay.smax, lay.kmax)


def _parent_v1_bytes(fitted, last_ds, opts) -> bytes:
    """The version-1 encoder as it stood before version 2: the record layout written out."""
    smax, kmax = fitted.smax, fitted.kmax
    dt = np.dtype([("magic", "S4"), ("version", "<u2"), ("flags", "<u2"), ("smax", "<i4"), ("kmax", "<i4"),
                   ("switches", "<i4", (4,)), ("meta_i32", "<i4", (8,)), ("meta_i64", "<i8", (2,)), ("last_ds", "<i8"),
                   ("meta_f64", "<f8", (4,)), ("params", "<f8", (3 + smax + kmax,)), ("tchange", "<f8", (smax,))])
    rec = np.zeros(fitted.n, dt)
    rec["magic"], rec["version"] = b"PB2M", 1
    rec["flags"] = (1 if opts.growth == 1 else 0) | (2 if opts.multiplicative else 0)
    rec["smax"], rec["kmax"] = smax, kmax
    rec["switches"] = [opts.yearly, opts.weekly, opts.daily, opts.n_changepoints]
    rec["meta_i32"], rec["meta_i64"], rec["meta_f64"] = fitted.meta_i32, fitted.meta_i64, fitted.meta_f64
    rec["last_ds"] = last_ds
    rec["params"], rec["tchange"] = fitted.params, fitted.tchange
    return rec.tobytes()


def _blob_bytes(arr) -> bytes:
    return b"".join(arr.to_pylist())


@pytest.mark.parametrize("kw", [dict(TABLE), dict(yearly_seasonality=20),
                                dict(seasonalities=[MONTHLY], weekly_seasonality=False, daily_seasonality=8,
                                     growth="linear", seasonality_mode="additive", n_changepoints=3),
                                dict(seasonalities=[dict(name="yearly", period=365.25, fourier_order=3)])])
def test_v2_round_trip_rebuilds_the_fit_options(kw):
    opts = batched.make_table_options(**kw)
    fb = _fitted(opts)
    last = np.arange(fb.n, dtype=np.int64) * 7
    col = model_record.encode(fb, last, opts)
    assert np.frombuffer(col.buffers()[2], "<u2", count=1, offset=4)[0] == 2
    got, last2, info = model_record.decode(col)
    assert info["table"] is not None
    for f in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64"):
        assert np.array_equal(getattr(got, f), getattr(fb, f))
    assert np.array_equal(last2, last)
    rebuilt = model_record.table_options(info)
    a, b = L.get_layout(rebuilt), L.get_layout(opts)
    assert (a.smax, a.kmax, a.pstride) == (b.smax, b.kmax, b.pstride)
    assert batched.component_names(rebuilt) == batched.component_names(opts)
    assert batched.seasonality_table(rebuilt) == batched.seasonality_table(opts)
    assert (rebuilt.growth, rebuilt.multiplicative, rebuilt.n_changepoints) == \
        (opts.growth, opts.multiplicative, opts.n_changepoints)
    # the record of the rebuilt options is the same bytes
    assert _blob_bytes(model_record.encode(fb, last, rebuilt)) == _blob_bytes(col)


@pytest.mark.parametrize("opts", [
    batched.make_options(), batched.make_options(growth="linear", yearly_seasonality=True, daily_seasonality=False),
    batched.make_table_options(yearly_seasonality=10), batched.make_table_options(yearly_seasonality=True),
    batched.make_table_options(weekly_seasonality=3, daily_seasonality=0, seasonalities=[])])
def test_v1_options_and_restated_tables_write_the_parent_bytes(opts):
    fb = _fitted(batched.make_options())
    last = np.array([5, 6, 7, 8], np.int64)
    col = model_record.encode(fb, last, opts)
    assert model_record.record_dtype(fb.smax, fb.kmax).itemsize == len(col[0].as_py())
    assert _blob_bytes(col) == _parent_v1_bytes(fb, last, opts)
    assert "table" not in model_record.decode(col)[2]


def test_restating_config_is_the_switch_config():
    a = pm.options_from_config({"model": {"yearly_seasonality": 10}})
    b = pm.options_from_config({"model": {"yearly_seasonality": True}})
    assert type(a) is L.Options and bytes(a) == bytes(b)
    assert bytes(pm.options_from_config({"model": {"seasonalities": []}})) == bytes(pm.options_from_config({}))


def _concat(*cols):
    return pa.chunked_array([c for col in cols for c in (col.chunks if isinstance(col, pa.ChunkedArray) else [col])])


def test_decode_refusals():
    t = batched.make_table_options(**TABLE)
    v2 = model_record.encode(_fitted(t), np.zeros(4, np.int64), t)
    d = batched.make_options()
    v1 = model_record.encode(_fitted(d), np.zeros(4, np.int64), d)
    with pytest.raises(ValueError, match="version-1 and version-2 model records in one table"):
        model_record.decode(_concat(v1, v2))
    with pytest.raises(ValueError, match="version-1 and version-2 model records in one table"):
        model_record.decode(_concat(v2, v1))
    other = batched.make_table_options(seasonalities=[dict(MONTHLY, period=30.4375), TABLE["seasonalities"][1]],
                                       yearly_seasonality=12)
    v2b = model_record.encode(_fitted(other), np.zeros(4, np.int64), other)
    with pytest.raises(ValueError, match="different seasonality tables"):
        model_record.decode(_concat(v2, v2b))
    raw = bytearray(_blob_bytes(v2))
    raw[4:6] = (3).to_bytes(2, "little")
    bad = pa.array([bytes(raw[:len(v2[0].as_py())])], pa.binary())
    with pytest.raises(ValueError, match="version 3 is unknown"):
        model_record.decode(bad)


def test_encode_refuses_what_it_cannot_represent():
    o = batched.make_table_options(**TABLE)
    o.yearly = L.SEAS_AUTO              # an order under an AUTO switch: make_table_options cannot say that
    with pytest.raises(ValueError, match="no model record"):
        model_record.encode(_fitted(o), np.zeros(4, np.int64), o)
    o = batched.make_table_options(**TABLE)
    with pytest.raises(ValueError, match="layout"):
        model_record.encode(_fitted(batched.make_options()), np.zeros(4, np.int64), o)


@pytest.mark.parametrize("model, match", [
    ({"seasonalities": [MONTHLY, dict(name="q", period=91.3, fourier_order=0)]},
     r"model\.seasonalities\[1\]\.fourier_order"),
    ({"seasonalities": [dict(name="q", period=-1, fourier_order=2)]}, r"model\.seasonalities\[0\]\.period"),
    ({"seasonalities": [dict(period=3, fourier_order=2)]}, r"model\.seasonalities\[0\]\.name is required"),
    ({"seasonalities": [dict(name="q", period=3, fourier_order=2, colour=1)]}, r"model\.seasonalities\[0\]: unknown"),
    ({"seasonalities": [dict(name="q", period=3, fourier_order=2, prior_scale=0)]},
     r"model\.seasonalities\[0\]\.prior_scale"),
    ({"seasonalities": [dict(name="q", period=3, fourier_order=2, mode="additive")]},
     r"model\.seasonalities\[0\]\.mode.*model\.seasonality_mode"),
    ({"seasonalities": [dict(name="weekly", period=7, fourier_order=2)], "weekly_seasonality": True},
     r"model\.seasonalities\[0\]\.name: 'weekly' replaces the built-in only when model\.weekly_seasonality is 'auto'"),
    ({"seasonalities": [dict(name=f"s{i}", period=2 + i, fourier_order=1) for i in range(9)]},
     r"model\.seasonalities: at most 8"),
    ({"seasonalities": "monthly"}, r"model\.seasonalities must be a list"),
    ({"yearly_seasonality": -2}, r"model\.yearly_seasonality must be >= 0"),
    ({"daily_seasonality": "sometimes", "seasonalities": []}, r"model\.daily_seasonality must be 'auto'"),
    ({"yearly_seasonality": 40}, r"model\.yearly_seasonality: .*K = 94"),
    ({"yearly_seasonality": 25, "seasonalities": [dict(name="q", period=3, fourier_order=2)]},
     r"model\.yearly_seasonality / model\.seasonalities: .*K = 68"),
])
def test_yaml_errors_name_the_key(model, match):
    with pytest.raises(ValueError, match=match):
        pm.options_from_config({"model": model})


@pytest.mark.parametrize("name", ["series_id", "dim_id", "ds", "yhat", "created_timestamp", "forecast_date",
                                  "forecast_timestamp", "forecast_quantity", "yhat_q0.5", "yhat_q"])
def test_names_of_forecast_columns_are_refused(name):
    with pytest.raises(ValueError, match=r"model\.seasonalities\[1\]\.name"):
        pm.options_from_config({"model": {"seasonalities": [MONTHLY, dict(name=name, period=3, fourier_order=1)]}})


def test_warm_start_is_refused_for_a_table():
    cfg = {"model": {"floor": 0, "cap_multiplier": 1.1, "seasonalities": [MONTHLY]},
           "io": {"warm_start": "/nonexistent/models", "models": "/nonexistent/out"}}
    with pytest.raises(ValueError, match=r"io\.warm_start .*model\.seasonalities"):
        pm.model_time_series(cfg).apply_batched(pa.table({"series_id": pa.array([], pa.int32())}), ["series_id", "dim_id"])
    cfg["insample"] = {"interval_width": 0.8, "refit": True}
    with pytest.raises(ValueError, match=r"io\.warm_start .*insample\.refit"):
        pm.model_time_series(cfg).apply_batched(pa.table({"series_id": pa.array([], pa.int32())}), ["series_id", "dim_id"])
    # the default model's warm start, and a restating table's, are not refused
    pm.refuse_table_warm_start(cfg, pm.options_from_config({"model": {"yearly_seasonality": 10}}))
    pm.refuse_table_warm_start(cfg, pm.options_from_config({}))


@pytest.mark.parametrize("model, key", [({"seasonalities": [MONTHLY]}, "model.seasonalities"),
                                        ({"daily_seasonality": 10}, "model.daily_seasonality")])
def test_tuner_refuses_a_table(model, key):
    cfg = {"model": dict(model, floor=0, cap_multiplier=1.1), "backtest": {"horizon": "1 days"}, "io": {}}
    with pytest.raises(ValueError, match=key.replace(".", r"\.") + ": the tuner"):
        pt.ProphetTuner(cfg).tune(None)     # refused before the input is touched


def test_scorer_component_columns_and_order():
    opts = batched.make_table_options(seasonalities=[MONTHLY, dict(name="weekly", period=7, fourier_order=2),
                                                     dict(name="quarterly", period=91.3, fourier_order=2)],
                                      yearly_seasonality=12, daily_seasonality=False)
    names = batched.component_names(opts)
    assert ps.custom_component_names(opts) == ("monthly", "quarterly")
    tab = batched.seasonality_table(opts)
    assert [e[0] for e in tab] == ["monthly", "weekly", "quarterly", "yearly"]
    n, h = 3, 2
    res = batched.ForecastBatch(None, np.zeros((n, h)), None, None, None,
                                np.arange(len(names) * n * h, dtype=np.float64).reshape(len(names), n, h),
                                np.zeros((n, h)), np.ones((n, h)), names=names)
    mask = batched.table_mask(tab, np.array([0, 1, 7]))         # yearly off, on, on; weekly custom: always on
    cols = ps.component_columns(res, mask, h, True, tab)
    assert list(cols) == list(ps.COMPONENT_COLUMNS) + ["monthly", "quarterly", "trend_lower", "trend_upper"]
    assert cols["yearly"].null_count == h and not cols["yearly"][0].is_valid and cols["yearly"][2].is_valid
    assert cols["weekly"].null_count == 0
    assert cols["daily"].null_count == n * h                     # no entry of that name
    assert cols["monthly"].to_pylist() == res.component("monthly").reshape(-1).tolist()
    fields = ps._component_fields(True, ps.custom_component_names(opts))
    assert [f.name for f in fields] == list(cols)
    # convert_forecasts keeps them, after the built-ins' columns and before trend_lower / trend_upper
    frame = {"series_id": pa.array([1] * (n * h), pa.int32()), "dim_id": pa.array([0] * (n * h), pa.int32()),
             "ds": pa.array(np.arange(n * h), pa.int64()).cast(pa.timestamp("ns")),
             "yhat": pa.array([0] * (n * h), pa.int32())}
    frame.update(cols)
    out = ps.ProphetScorer.convert_forecasts(ps.Frame(pa.table(frame))).table
    assert out.column_names == ["created_timestamp", "series_id", "dim_id", "forecast_date", "forecast_timestamp",
                                "forecast_quantity"] + list(cols)


def test_empty_shard_has_the_custom_columns():
    opts = batched.make_table_options(seasonalities=[MONTHLY])
    col = model_record.encode(_fitted(opts, n=2), np.zeros(2, np.int64), opts)
    models = pa.table({"series_id": pa.array([1, 2], pa.int32()), "dim_id": pa.array([0, 0], pa.int32()),
                       "floor": pa.array([0, 0], pa.float32()), "cap": pa.array([9, 9], pa.float32()), "model": col})
    op = ps.forecast_time_series({"forecast": {"periods": 3, "frequency": "D", "components": True, "intervals": True}})
    import time_series_spark_b200.dist as pdist
    orig = pdist.world
    try:
        pdist.world = lambda: (1, 3, 1)          # rank 1 of 3 over 2 models: an empty shard
        out = op.apply_batched(models, ["series_id", "dim_id"])
    finally:
        pdist.world = orig
    assert out.num_rows == 0
    assert out.column_names == ["series_id", "dim_id", "ds", "yhat", "yhat_lower", "yhat_upper"] + \
        list(ps.COMPONENT_COLUMNS) + ["monthly", "trend_lower", "trend_upper"]


def test_with_mask_gives_prophet_copy_tables():
    # every custom entry kept, a built-in forced by the full history's mask, a custom 'weekly' under AUTO left alone
    opts = batched.make_table_options(seasonalities=[MONTHLY, dict(name="weekly", period=7, fourier_order=2)],
                                      yearly_seasonality=12)
    for mask in range(8):
        o = batched._with_mask(opts, mask)
        assert o.abi_version == L.ABI_VERSION_TABLE and o.weekly == L.SEAS_AUTO
        assert (o.yearly, o.daily) == (int(mask & 1 != 0), int(mask & 4 != 0))
        assert (o.yearly_order, o.weekly_order, o.daily_order) == (12, 0, 0)
        want = [e for e in batched.seasonality_table(opts) if e[3] == 0 or mask & e[3]]
        assert batched.seasonality_table(o) == want
        L.get_layout(o)                         # the library takes it
        # the cutoff table's entries are the full table's active ones, so the packed columns agree
        full = batched.table_mask(batched.seasonality_table(opts), mask)
        assert [e for j, e in enumerate(batched.seasonality_table(opts)) if full >> j & 1] == want
    # the copy owns its entries and leaves the original alone
    o = batched._with_mask(opts, 0)
    del opts
    assert [o.seasonalities[i].name for i in range(o.n_seasonalities)] == [b"monthly", b"weekly"]
    # forcing a built-in that a custom entry replaces is what the library refuses
    opts = batched.make_table_options(seasonalities=[dict(name="weekly", period=7, fourier_order=2)])
    bad = batched.copy_options(opts)
    bad.weekly = 1
    with pytest.raises(ValueError, match="replaces the built-in only when"):
        L.get_layout(bad)
    # v1 options: the switches forced, nothing else
    o = batched._with_mask(batched.make_options(), 5)
    assert type(o) is L.Options and (o.yearly, o.weekly, o.daily) == (1, 0, 1)


@pytest.mark.parametrize("kw", [dict(yearly_seasonality=20), dict(yearly_seasonality=20, weekly_seasonality=False),
                                dict(daily_seasonality=10, yearly_seasonality=False), dict(TABLE),
                                dict(seasonalities=[dict(name="weekly", period=7, fourier_order=3)])])
def test_cutoff_tables_stay_tables_within_the_full_layout(kw):
    # the plan's mask has a forced-on built-in's bit set and a forced-off one's clear; under every such mask the cutoff
    # options are still a table (a custom entry is always on, an int order forces its built-in on) and no wider than
    # the full layout, with the full table's active entries in order
    opts = batched.make_table_options(**kw)
    full, tab = L.get_layout(opts), batched.seasonality_table(opts)
    sw = (opts.yearly, opts.weekly, opts.daily)
    for mask in range(8):
        if any((s == 1 and not mask & bit) or (s == 0 and mask & bit) for s, bit in zip(sw, (1, 2, 4))):
            continue
        o = batched._with_mask(opts, mask)
        assert batched.is_table(o)
        assert L.get_layout(o).pstride <= full.pstride
        m = int(batched.table_mask(tab, mask))
        assert batched.seasonality_table(o) == [e for j, e in enumerate(tab) if m >> j & 1]


def test_example_config_is_one_the_library_takes():
    import os
    import yaml
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "config", "example_seasonalities_modeler_app_config.yaml")) as f:
        cfg = yaml.safe_load(f)
    opts = pm.options_from_config(cfg)
    assert batched.is_table(opts)
    lay = L.get_layout(opts)
    assert lay.kmax == 60 and lay.pstride == 88            # as the file's comment says
    assert ps.custom_component_names(opts) == ("monthly", "quarterly")


def test_warm_start_from_a_table_job_is_refused():
    # a default-model job whose io.warm_start is a table job's models: the records' mask and betas are the table's
    t = batched.make_table_options(seasonalities=[dict(name="weekly", period=7, fourier_order=3)])
    assert L.get_layout(t).kmax == L.get_layout(batched.make_options()).kmax    # same layout, other columns
    models = pa.table({"series_id": pa.array([1, 2], pa.int32()), "dim_id": pa.array([0, 0], pa.int32()),
                       "model": model_record.encode(_fitted(t, n=2), np.zeros(2, np.int64), t)})
    with pytest.raises(ValueError, match=r"io\.warm_start holds models fitted with a seasonality table"):
        pm.warm_start_init(models, batched.make_options(), np.array([1, 2]), np.array([0, 0]))


def _models(*parts):
    cols = [model_record.encode(_fitted(o, n=k, seed=j), np.zeros(k, np.int64), o) for j, (o, k) in enumerate(parts)]
    n = sum(k for _, k in parts)
    return pa.table({"series_id": pa.array(np.arange(n), pa.int32()), "dim_id": pa.array(np.zeros(n), pa.int32()),
                     "floor": pa.array(np.zeros(n), pa.float32()), "cap": pa.array(np.full(n, 9.0), pa.float32()),
                     "model": _concat(*cols)})


@pytest.mark.parametrize("components", [False, True])
def test_every_rank_refuses_a_table_of_two_model_classes(components):
    import time_series_spark_b200.dist as pdist
    t = batched.make_table_options(**TABLE)
    other = batched.make_table_options(seasonalities=[MONTHLY], n_changepoints=3)
    op = ps.forecast_time_series({"forecast": {"periods": 3, "frequency": "D", "components": components}})
    orig = pdist.world
    try:
        for models, match in ((_models((batched.make_options(), 3), (t, 3)), "version-1 and version-2"),
                              (_models((t, 3), (other, 3)), "different seasonality tables")):
            for rank in (0, 1):     # rank 0's shard holds one class only: the refusal is the whole table's
                pdist.world = lambda: (rank, 2, rank)
                with pytest.raises(ValueError, match=match):
                    op.apply_batched(models, ["series_id", "dim_id"])
    finally:
        pdist.world = orig
    # one table of differing layouts (n_changepoints) is one model class
    model_record.check_one_class(_models((t, 2), (batched.make_table_options(**TABLE, n_changepoints=3), 2))["model"])


def _random_tables(k):
    rng = np.random.RandomState(11)
    names = ["monthly", "quarterly", "yearly", "weekly", "daily", "hourly"]
    periods = {"monthly": 30.5, "quarterly": 91.3, "yearly": 365.25, "weekly": 7.0, "daily": 1.0, "hourly": 1 / 24}
    out = []
    while len(out) < k:
        kw = {}
        for key, dflt in (("yearly_seasonality", 10), ("weekly_seasonality", 3), ("daily_seasonality", 4)):
            kw[key] = ["auto", True, False, 0, dflt, int(rng.randint(1, 8))][rng.randint(6)]
        pick = rng.choice(names, rng.randint(0, 4), replace=False)
        kw["seasonalities"] = [dict(name=str(nm), period=periods[nm], fourier_order=int(rng.randint(1, 5))) for nm in pick]
        kw["n_changepoints"] = 5
        try:
            out.append(batched.make_table_options(**kw))
        except ValueError:
            pass
    return out


def test_host_table_is_the_librarys():
    # seasonality_table restates the library's normalisation; held here to what the library reports of it: the
    # Fourier column count of the whole table (pb200_get_layout's kmax), the custom component planes
    # (pb200_component_count and their names) and whether it is the default model
    seen_v1 = seen_table = 0
    for o in _random_tables(300):
        tab = batched.seasonality_table(o)
        lay = L.get_layout(o)
        v1 = L.Options.from_buffer_copy(o)
        v1.abi_version = L.ABI_VERSION
        if tab is None:
            seen_v1 += 1
            assert lay.kmax == L.get_layout(v1).kmax
            assert batched.component_names(o) == L.COMPONENTS
            continue
        seen_table += 1
        assert lay.kmax == sum(2 * e[2] for e in tab)
        assert batched.component_names(o)[L.N_COMPONENTS:] == tuple(
            e[0] for e in tab if e[3] == 0 and e[0] not in ("yearly", "weekly", "daily"))
        assert len({e[0] for e in tab}) == len(tab)
        kinds = [e[3] for e in tab]
        assert kinds == sorted(kinds, key=lambda k: (k != 0, k))      # the customs as added, then yearly, weekly, daily
    assert seen_v1 > 10 and seen_table > 100
