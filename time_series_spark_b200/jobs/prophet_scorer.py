"""H100 drop-in for the reference's src/jobs/prophet_scorer.py.

Same names and contracts -- ``forecast_time_series(config)``, ``extract_date``,
``ProphetScorer(config).read_model_dataframe / convert_forecasts / write_forecasts``,
``ProphetScorer.score`` -- same YAML keys (``io.models``, ``io.forecasts``,
``forecast.periods``, ``forecast.frequency``), same models-table input and forecast CSV
output ``(created_timestamp, series_id, dim_id, forecast_date, forecast_timestamp,
forecast_quantity)``.  The per-model ``make_future_dataframe`` / ``predict`` / int-cast /
floor-clamp body (reference :35-102) is one batched GPU call over all models.

Optional keys beyond the reference: ``forecast.intervals`` (default false: the reference
computes yhat_lower/yhat_upper inside Prophet.predict and drops them at :86; set true to get
``yhat_lower``/``yhat_upper`` columns), ``forecast.uncertainty_samples`` (1000),
``forecast.interval_width`` (0.8), ``forecast.seed``, ``forecast.components`` (default false; true adds fbprophet's
component columns ``trend, yearly, weekly, daily, multiplicative_terms, additive_terms``, and ``trend_lower`` /
``trend_upper`` with intervals -- DESIGN §12), ``forecast.aggregate`` (a fixed-width duration such as ``'1D'``: also
write, to ``io.aggregates``, the forecast total of every such window of every model with the interval of the total from
the joint draws -- DESIGN §13), ``forecast.aggregate_origin`` (where window 0 starts, default 1970-01-01),
``forecast.aggregate_period`` (a pandas period alias such as ``'M'``, ``'Q-NOV'``, ``'Y'`` or ``'W-SUN'``: the same
``io.aggregates`` table over calendar months, quarters, years or weeks -- DESIGN §17),
``forecast.aggregate_quantiles`` (with ``forecast.aggregate`` or ``forecast.aggregate_period``, a list of 1 to 32 levels
in [0, 1]: one float64 column ``yhat_q<level>`` per level in ``io.aggregates``, after ``yhat_upper``, the percentile
100 level of the window total's ``uncertainty_samples`` draws -- DESIGN §21) and
``forecast.quantiles`` (a list of 1 to 32 levels in [0, 1]: one float64 column ``yhat_q<level>`` per level, the
percentile 100 level of the point's ``uncertainty_samples`` draws -- DESIGN §15).

Models with a seasonality table (version-2 records, written by the modeler from ``model.seasonalities`` or an int
built-in order -- DESIGN §18) are scored with the table the record carries; no scorer key is needed, and every mode
above serves them.  With ``forecast.components`` each custom seasonality not named like a built-in adds one float64
column of its name after ``additive_terms`` (in table order); a custom ``yearly`` / ``weekly`` / ``daily`` fills that
built-in's column, which is null where the model's entry of that name is inactive.

Models with extra regressors (version-4 records, written by the modeler from ``model.regressors`` -- DESIGN §20) need
``io.future_regressors``: the regressors' values on the forecast grid, as hive dirs ``series_id=<id>/`` of header-less
CSV ``dim_id,timestamp,<one value per regressor in the record's order>``.  Each rank reads the series_ids of its own
models.  The values are joined onto every model's grid on the GPU by exact timestamp; rows off the grid are ignored.  A
grid point without a row, a NaN value on one and a repeated ``(series_id, dim_id, timestamp)`` raise ValueError before
any predict, naming the regressor or the row.  Point forecasts and ``forecast.intervals`` serve such models;
``forecast.components``, ``forecast.aggregate``, ``forecast.aggregate_period`` and ``forecast.quantiles`` are refused
with them, and ``io.future_regressors`` is refused for models without regressors.
"""
from __future__ import annotations

import logging
import os
from datetime import datetime, timezone

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.csv as pacsv
import pyarrow.dataset as pads

from .. import _lib as L
from .. import batched, model_record
from .. import dist as pdist
from ..frame import Frame
from .prophet_modeler import get_context

FORECAST_SCHEMA = pa.schema([   # reference prophet_scorer.py:27-32
    pa.field("series_id", pa.int32(), True),
    pa.field("dim_id", pa.int32(), True),
    pa.field("ds", pa.timestamp("ns"), True),
    pa.field("yhat", pa.int32(), True),
])


# fbprophet's component columns of Prophet.predict, in the frame's order; a seasonal column is null on the rows of a model
# that has no such seasonality (fbprophet would have no such column for it)
COMPONENT_COLUMNS = ("trend", "yearly", "weekly", "daily", "multiplicative_terms", "additive_terms")
_SEASONAL_BIT = {"yearly": 1, "weekly": 2, "daily": 4}


def _want_components(fc) -> bool:
    v = fc.get("components", False)
    if not isinstance(v, (bool, np.bool_)):
        raise ValueError(f"forecast.components must be true or false (got {v!r})")
    return bool(v)


def quantile_levels(section: dict, key: str):
    """``<section>.quantiles`` checked (``key`` is its full name for the messages): None without it, else the list of
    levels, 1 to 32 numbers in [0, 1], whose column names ``quantile_column`` are distinct."""
    v = section.get("quantiles")
    if v is None:
        return None
    if not isinstance(v, (list, tuple)) or not 1 <= len(v) <= batched.QUANTILES_MAX:
        raise ValueError(f"{key} must be a list of 1 to {batched.QUANTILES_MAX} levels in [0, 1] (got {v!r})")
    levels = []
    for q in v:
        if isinstance(q, (bool, np.bool_)) or not isinstance(q, (int, float, np.integer, np.floating)) or \
                not 0.0 <= float(q) <= 1.0:
            raise ValueError(f"{key} must hold levels in [0, 1] (got {q!r})")
        levels.append(float(q))
    names = [quantile_column(q) for q in levels]
    if len(set(names)) != len(names):
        raise ValueError(f"{key} names a level twice (columns {names})")
    return levels


def quantile_column(q: float) -> str:
    """The forecast column of level q: yhat_q0.1, yhat_q0.5, yhat_q0.975."""
    return "yhat_q" + repr(float(q))


def _component_fields(intervals: bool, custom=()):
    names = COMPONENT_COLUMNS + tuple(custom) + (("trend_lower", "trend_upper") if intervals else ())
    return [pa.field(n, pa.float64()) for n in names]


def custom_component_names(opts) -> tuple:
    """The component columns a seasonality table adds to COMPONENT_COLUMNS: one per custom entry not named like a
    built-in, in table order (batched.component_names past the six planes)."""
    return tuple(batched.component_names(opts)[L.N_COMPONENTS:])


def component_columns(res: "batched.ForecastBatch", mask: np.ndarray, periods: int, intervals: bool, table=None) -> dict:
    """The component columns of one shard's forecast frame, one row per (model, period), from a components predict
    (``res``) and the models' seasonality masks (meta_i32[:, 3]).  With a seasonality table (``table``:
    batched.seasonality_table) the mask is the table mask: a built-in's column is null where the entry of its name (the
    built-in's own, or a custom entry replacing it) is inactive or absent, and each custom entry not named like a
    built-in adds its column after additive_terms."""
    mask = np.asarray(mask)
    cols = {}
    entry = {e[0]: j for j, e in enumerate(table or ())}
    for name in COMPONENT_COLUMNS:
        v = np.ascontiguousarray(res.component(name)).reshape(-1)
        absent = None
        if name in _SEASONAL_BIT:
            if table is None:
                off = (mask & _SEASONAL_BIT[name]) == 0
            elif name in entry:
                off = ((mask >> entry[name]) & 1) == 0
            else:
                off = np.ones(mask.shape, bool)
            absent = np.repeat(off, periods)
        cols[name] = pa.array(v, pa.float64(), mask=absent)
    for name in res.names[L.N_COMPONENTS:]:
        cols[name] = pa.array(np.ascontiguousarray(res.component(name)).reshape(-1), pa.float64())
    if intervals:
        cols["trend_lower"] = pa.array(res.trend_lower.reshape(-1), pa.float64())
        cols["trend_upper"] = pa.array(res.trend_upper.reshape(-1), pa.float64())
    return cols


AGGREGATE_SCHEMA = pa.schema([
    pa.field("series_id", pa.int32()), pa.field("dim_id", pa.int32()), pa.field("window_start", pa.timestamp("ns")),
    pa.field("window_points", pa.int32()), pa.field("forecast_quantity", pa.int64()), pa.field("yhat", pa.float64()),
    pa.field("yhat_lower", pa.float64()), pa.field("yhat_upper", pa.float64()),
])


def forecast_quantiles(config):
    """``forecast.quantiles`` checked (quantile_levels), or None; it does not combine with forecast.components or
    forecast.aggregate."""
    fc = config.get("forecast", {}) or {}
    levels = quantile_levels(fc, "forecast.quantiles")
    if levels is not None and _want_components(fc):
        raise ValueError("forecast.quantiles cannot be combined with forecast.components")
    if levels is not None and fc.get("aggregate") is not None:
        raise ValueError("forecast.quantiles cannot be combined with forecast.aggregate")
    return levels


def aggregate_rule(config):
    """``forecast.aggregate`` / ``forecast.aggregate_origin`` as (width_ns, origin_ns), or None without the key.  The
    width is a fixed-width pandas duration ('1D', '7D', '8h'); calendar offsets ('M') have no fixed width and are refused."""
    import pandas as pd
    fc = config.get("forecast", {}) or {}
    if fc.get("aggregate") is None:
        return None
    spec = fc["aggregate"]
    try:
        off = _to_offset(spec)
        width = int(7 * 86400 * 10**9 * off.n if isinstance(off, pd.offsets.Week) and off.weekday is None else off.nanos)
    except Exception:
        raise ValueError(f"forecast.aggregate must be a fixed-width duration such as '1D', '7D' or '8h' (got {spec!r}; "
                         "calendar offsets such as 'M' have no fixed width)") from None
    if width <= 0:
        raise ValueError(f"forecast.aggregate must be a positive duration (got {spec!r})")
    try:
        origin = pd.Timestamp(fc.get("aggregate_origin", "1970-01-01"))
        if origin is pd.NaT:
            raise ValueError("NaT")
        if origin.tzinfo is not None:
            origin = origin.tz_convert("UTC").tz_localize(None)
        origin_ns = int(origin.value)
    except Exception:
        raise ValueError(f"forecast.aggregate_origin must be a timestamp (got {fc.get('aggregate_origin')!r})") from None
    if not (config.get("io", {}) or {}).get("aggregates"):
        raise ValueError("forecast.aggregate needs io.aggregates, the directory the window totals are written to")
    if _want_components(fc):
        raise ValueError("forecast.aggregate cannot be combined with forecast.components")
    return width, origin_ns


def aggregate_period(config):
    """``forecast.aggregate_period``, a pandas period alias ('M', 'Q-NOV', 'Y', 'W-SUN'), as batched.period_rule's tuple,
    or None without the key.  It writes io.aggregates as forecast.aggregate does, so it needs io.aggregates and combines
    with none of forecast.aggregate, forecast.aggregate_origin, forecast.components and forecast.quantiles."""
    fc = config.get("forecast", {}) or {}
    spec = fc.get("aggregate_period")
    if spec is None:
        return None
    for other in ("aggregate", "aggregate_origin", "quantiles"):
        if fc.get(other) is not None:
            raise ValueError(f"forecast.aggregate_period cannot be combined with forecast.{other}")
    if _want_components(fc):
        raise ValueError("forecast.aggregate_period cannot be combined with forecast.components")
    if not (config.get("io", {}) or {}).get("aggregates"):
        raise ValueError("forecast.aggregate_period needs io.aggregates, the directory the period totals are written to")
    try:
        return batched.period_rule(spec)
    except ValueError as e:
        raise ValueError(f"forecast.aggregate_period: {e}") from None


def aggregate_quantiles(config):
    """``forecast.aggregate_quantiles`` checked as quantile_levels checks forecast.quantiles, or None without it.  The
    levels describe the window totals of io.aggregates, so the key needs forecast.aggregate or
    forecast.aggregate_period."""
    fc = config.get("forecast", {}) or {}
    levels = quantile_levels({"quantiles": fc.get("aggregate_quantiles")}, "forecast.aggregate_quantiles")
    if levels is not None and fc.get("aggregate") is None and fc.get("aggregate_period") is None:
        raise ValueError("forecast.aggregate_quantiles needs forecast.aggregate or forecast.aggregate_period: its levels "
                         "are quantiles of the window totals")
    return levels


def aggregate_schema(levels=None) -> pa.Schema:
    """io.aggregates' schema: AGGREGATE_SCHEMA, then one float64 column quantile_column(q) per level of
    forecast.aggregate_quantiles."""
    schema = AGGREGATE_SCHEMA
    for q in levels or ():
        schema = schema.append(pa.field(quantile_column(q), pa.float64()))
    return schema


def aggregate_table(sid, did, ok, ws: "batched.WindowSums") -> pa.Table:
    """One row per (model, window) of the models that have a forecast, from a shard's WindowSums (a WindowQuantiles
    adds its levels' columns after yhat_upper)."""
    wmax = ws.start.shape[1]
    keep = (np.arange(wmax)[None, :] < ws.n_windows[:, None]) & ok[:, None]
    rows = np.nonzero(keep)[0]
    quant = {}
    if isinstance(ws, batched.WindowQuantiles):
        quant = {quantile_column(q): pa.array(ws.quantiles[j][keep], pa.float64()) for j, q in enumerate(ws.levels)}
    return pa.table({
        "series_id": pa.array(sid[rows], pa.int32()),
        "dim_id": pa.array(did[rows], pa.int32()),
        "window_start": pa.array(ws.start[keep], pa.int64()).cast(pa.timestamp("ns")),
        "window_points": pa.array(ws.points[keep], pa.int32()),
        "forecast_quantity": pa.array(ws.quantity_sum[keep], pa.int64()),
        "yhat": pa.array(ws.yhat_sum[keep], pa.float64()),
        "yhat_lower": pa.array(ws.lower[keep], pa.float64()),
        "yhat_upper": pa.array(ws.upper[keep], pa.float64()),
        **quant,
    })


# pandas 0.25 (the reference's pin) offset aliases that later pandas renamed
_LEGACY_ALIASES = {"H": "h", "T": "min", "S": "s", "L": "ms", "U": "us", "N": "ns", "M": "ME", "BM": "BME",
                   "Q": "QE", "BQ": "BQE", "A": "YE", "Y": "YE", "BA": "BYE", "BY": "BYE", "AS": "YS", "BAS": "BYS"}


def _to_offset(frequency):
    import re
    import pandas as pd
    try:
        return pd.tseries.frequencies.to_offset(frequency)
    except ValueError:
        m = re.fullmatch(r"(-?\d*)([A-Za-z]+)(-.*)?", str(frequency))
        if not m or m.group(2) not in _LEGACY_ALIASES:
            raise
        return pd.tseries.frequencies.to_offset(f"{m.group(1)}{_LEGACY_ALIASES[m.group(2)]}{m.group(3) or ''}")


def frequency_to_future(last_ds_ns: np.ndarray, periods: int, frequency) -> np.ndarray:
    """Prophet.make_future_dataframe(periods, freq, include_history=False) for every model
    (reference :57-66): ``date_range(start=last, periods=periods+1, freq)``, keep ``> last``,
    first ``periods``.  'W' is replaced by ``pd.offsets.Week()`` so weeks stay on the last
    date's weekday (:59-62).  Fixed-width frequencies are pure int64 arithmetic; calendar
    frequencies (e.g. 'M') go through pandas once per distinct last date."""
    import pandas as pd
    last = np.asarray(last_ds_ns, dtype=np.int64)
    if isinstance(frequency, str) and frequency == "W":
        frequency = pd.offsets.Week()
    off = _to_offset(frequency)
    nanos = None
    if isinstance(off, pd.offsets.Week) and off.weekday is None:
        nanos = 7 * 86400 * 10**9 * off.n
    else:
        try:
            nanos = int(off.nanos)
        except Exception:
            nanos = None
    if nanos is not None:
        return batched.make_future(last, periods, nanos)
    out = np.empty((last.size, periods), np.int64)
    uniq, inv = np.unique(last, return_inverse=True)
    for u_i, u in enumerate(uniq):
        ld = pd.Timestamp(int(u))
        dates = pd.date_range(start=ld, periods=periods + 1, freq=off)
        dates = dates[dates > ld][:periods]
        if len(dates) != periods:
            raise ValueError("could not build the future frame for frequency %r" % (frequency,))
        out[inv == u_i] = dates.values.astype("datetime64[ns]").astype(np.int64)[None, :]
    return out


def refuse_regressor_modes(config, regressors: bool) -> None:
    """The scorer's keys that do not go with the models' class: with extra regressors (version-4 records) the modes
    without regressor values (components, window and period totals, quantiles) and a missing io.future_regressors;
    without them an io.future_regressors, which would be ignored.  Each raises ValueError naming the key."""
    fc = config.get("forecast", {}) or {}
    path = (config.get("io", {}) or {}).get("future_regressors")
    if not regressors:
        if path:
            raise ValueError("io.future_regressors is given, but the models have no extra regressors (they are not "
                             "version-4 records)")
        return
    for key in ("aggregate", "aggregate_period", "quantiles"):
        if fc.get(key) is not None:
            raise ValueError(f"forecast.{key} is not available for models with extra regressors (model.regressors)")
    if _want_components(fc):
        raise ValueError("forecast.components is not available for models with extra regressors (model.regressors)")
    if not path:
        raise ValueError("io.future_regressors is required: the models have extra regressors (model.regressors), "
                         "whose values on the forecast grid it holds")


def read_future_regressors(path: str, names, series_id) -> pa.Table:
    """The rows of io.future_regressors (hive dirs ``series_id=<id>/``, header-less CSV ``dim_id,timestamp,<values>``)
    whose series_id is one of ``series_id``: columns series_id, dim_id, ds and one float64 column per name (an empty
    field is null)."""
    part = pads.partitioning(pa.schema([("series_id", pa.int32())]), flavor="hive")
    cols = ["dim_id", "ds"] + list(names)
    types = dict({"dim_id": pa.int32(), "ds": pa.timestamp("ns")}, **{n: pa.float64() for n in names})
    fmt = pads.CsvFileFormat(read_options=pacsv.ReadOptions(column_names=cols),
                             convert_options=pacsv.ConvertOptions(
                                 column_types=types, timestamp_parsers=["%Y-%m-%d %H:%M:%S", pacsv.ISO8601]))
    dset = pads.dataset(path, format=fmt, partitioning=part, exclude_invalid_files=False, ignore_prefixes=[".", "_"])
    sids = pa.array(np.unique(np.asarray(series_id, dtype=np.int32)), pa.int32())
    return dset.to_table(columns=["series_id"] + cols, filter=pc.field("series_id").isin(sids))


def _at(sid, did, i, ts) -> str:
    return f"series_id {int(sid[i])}, dim_id {int(did[i])}, ds {np.datetime64(int(ts), 'ns')}"


def future_regressor_values(ctx, table: pa.Table, names, sid, did, future_ds, ok):
    """The future values ``[R, n, H]`` (a CUDA tensor) of the models ``(sid, did)`` on their grids ``future_ds`` (a CUDA
    int64 tensor ``[n, H]``) from the rows of io.future_regressors in ``table``: packed on the GPU, matched to the models
    on the host and joined by pb200_join_future_regressors_device.  Raises ValueError, naming the row, for a repeated
    (series_id, dim_id, timestamp), and -- over the models ``ok`` -- naming the regressor, the first model and
    timestamp and the count, for a grid point without a row or with a NaN value (fbprophet: "Found NaN in column")."""
    import torch
    from ..pack import pack_groups_cuda
    from .prophet_modeler import _group_keys
    dev = future_ds.device
    pk = pack_groups_cuda(table, device=dev, y_col=None, reg_cols=list(names))
    if pk.ds.numel() > 1:
        starts = torch.zeros(pk.ds.numel(), dtype=torch.bool, device=dev)
        starts[torch.from_numpy(pk.offsets[:-1]).to(dev)] = True
        dup = (pk.ds[1:] == pk.ds[:-1]) & ~starts[1:]
        if bool(dup.any()):
            r = int(torch.nonzero(dup)[0, 0]) + 1
            g = int(np.searchsorted(pk.offsets, r, side="right") - 1)
            raise ValueError("io.future_regressors holds more than one row for "
                             f"{_at(pk.series_id, pk.dim_id, g, pk.ds[r].item())} ({int(dup.sum())} repeated row(s) in all)")
    gkey = _group_keys(pk.series_id, pk.dim_id)
    mkey = _group_keys(sid, did)
    order = np.argsort(gkey, kind="stable")
    group = np.full(mkey.size, -1, np.int64)
    if gkey.size:
        pos = np.minimum(np.searchsorted(gkey[order], mkey), gkey.size - 1)
        hit = gkey[order][pos] == mkey
        group[hit] = order[pos[hit]]
    fut, missing, first = batched.join_future_regressors_device(
        ctx, pk.ds.contiguous(), pk.offsets, pk.regressors.contiguous(), torch.from_numpy(group).to(dev),
        future_ds.contiguous())
    missing = missing.cpu().numpy()
    bad = (missing > 0) & ok
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError(f"Found NaN in column {names[0]}: io.future_regressors has no row for {int(missing[bad].sum())} "
                         f"forecast point(s) of {int(bad.sum())} model(s) (first: "
                         f"{_at(sid, did, i, first[i].item())})")
    okd = torch.from_numpy(ok).to(dev)
    for r, name in enumerate(names):
        nan = torch.isnan(fut[r]) & okd[:, None]
        if bool(nan.any()):
            i, h = (int(v) for v in torch.nonzero(nan)[0])
            raise ValueError(f"Found NaN in column {name}: io.future_regressors holds NaN for {int(nan.sum())} forecast "
                             f"point(s) (first: {_at(sid, did, i, future_ds[i, h].item())})")
    return fut


class _ForecastTimeSeriesOp:
    """Batched GROUPED_MAP operator over the models table."""

    def __init__(self, config):
        self.config = config
        self.aggregates = None      # with forecast.aggregate: the window totals of the last apply_batched (this rank's models)

    def apply_batched(self, table: pa.Table, keys) -> pa.Table:
        if list(keys) != ["series_id", "dim_id"]:
            raise ValueError("forecast_time_series groups by ('series_id', 'dim_id')")
        fc = self.config["forecast"]
        want_intervals = bool(fc.get("intervals", False))
        # forecast.aggregate_period: weeks are a fixed-width rule, months / quarters / years the calendar call
        period = aggregate_period(self.config)
        rule = period[1:] if period and period[0] == "fixed" else aggregate_rule(self.config)
        months = period[1:] if period and period[0] == "months" else None
        alevels = aggregate_quantiles(self.config)
        self.aggregates = aggregate_schema(alevels).empty_table() if rule or months else None
        levels = forecast_quantiles(self.config)
        if want_intervals or rule or months or levels:
            width = float(fc.get("interval_width", 0.8))
            if not 0.0 <= width <= 1.0:     # fbprophet refuses it too (numpy's percentile range check); NaN fails here
                raise ValueError(f"forecast.interval_width must be in [0, 1] (got {fc.get('interval_width')!r})")
        want_components = _want_components(fc)
        # every rank scores a shard of the whole table, so the model class (version 1, or version 2 with one seasonality
        # table) is checked over all of it, and a table's custom component columns come from its first model: every
        # rank's frame (an empty shard's too) then has the same columns
        rank, ws, _ = pdist.world()
        custom = ()
        if table.num_rows:
            valid = table["model"].filter(pc.is_valid(table["model"]))
            if len(valid):
                if ws > 1:
                    model_record.check_one_class(valid)
                _, _, info0 = model_record.decode(valid.slice(0, 1))
                # a version-4 record's refusals come before any GPU work, on every rank
                refuse_regressor_modes(self.config, "regressors" in info0)
                if want_components and "table" in info0:
                    custom = custom_component_names(model_record.table_options(info0))
        if ws > 1 and table.num_rows:      # shard the model rows across ranks (equal horizon => equal work)
            lo, hi = pdist.shard_bounds(np.arange(table.num_rows + 1, dtype=np.int64), ws)[rank]
            table = table.slice(lo, hi - lo)
        # every rank must hand back the same columns (an empty shard too): the optional gather issues one
        # collective per column
        empty_schema = FORECAST_SCHEMA
        if want_intervals:
            empty_schema = empty_schema.append(pa.field("yhat_lower", pa.float64())).append(pa.field("yhat_upper", pa.float64()))
        for q in levels or ():
            empty_schema = empty_schema.append(pa.field(quantile_column(q), pa.float64()))
        if want_components:
            for f in _component_fields(want_intervals, custom):
                empty_schema = empty_schema.append(f)
        if table.num_rows == 0:
            return empty_schema.empty_table()
        # model is None -> "no model found", empty frame for that group (reference :51-55)
        mcol = table["model"]
        if mcol.null_count:
            nulls = table.filter(pc.is_null(mcol))
            for sid, did in zip(nulls["series_id"].to_pylist(), nulls["dim_id"].to_pylist()):
                print(f"For series_id: {sid}, dim_id: {did}, no model found")
            table = table.filter(pc.is_valid(mcol))
            if table.num_rows == 0:
                return empty_schema.empty_table()
        fitted, last_ds, info = model_record.decode(table["model"])
        mc = dict(interval_width=fc.get("interval_width", 0.8),
                  uncertainty_samples=fc.get("uncertainty_samples", 1000) if want_intervals or rule or months or levels else 0)
        if "regressors" in info:     # a version-4 record: the fit's table and regressors (DESIGN §20)
            opts = model_record.regressor_options(info, **mc)
        elif "table" in info:        # a version-2 record: the fit's seasonality table (DESIGN §18)
            opts = model_record.table_options(info, **mc)
        else:
            opts = batched.make_options(growth="logistic" if info["logistic"] else "linear",
                                        seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
                                        n_changepoints=info["n_changepoints"], **mc)
            opts.yearly, opts.weekly, opts.daily = info["yearly"], info["weekly"], info["daily"]
        # reference :46-47: floor / cap are read back from the FLOAT32 columns of the models table
        floor = table["floor"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.float64)
        cap = table["cap"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.float64)
        periods = int(fc["periods"])
        future = frequency_to_future(last_ds, periods, fc["frequency"])
        ctx = get_context()
        sid = table["series_id"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.int32)
        did = table["dim_id"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.int32)
        ok = fitted.meta_i32[:, 4] >= 0
        if "regressors" in info:
            res = self._predict_regressors(ctx, opts, info, fitted, future, floor, cap, sid, did, ok, want_intervals)
        elif rule:
            res, sums = batched.predict_sums_host(ctx, opts, fitted, future, floor, cap, rule[0], rule[1],
                                                  seed=int(fc.get("seed", 0)), intervals=want_intervals, levels=alevels)
            self.aggregates = aggregate_table(sid, did, ok, sums)
        elif months:
            res, sums = batched.predict_period_sums_host(ctx, opts, fitted, future, floor, cap, months[0], months[1],
                                                         seed=int(fc.get("seed", 0)), intervals=want_intervals,
                                                         levels=alevels)
            self.aggregates = aggregate_table(sid, did, ok, sums)
        elif levels:
            res = batched.predict_quantiles_host(ctx, opts, fitted, future, floor, cap, levels, seed=int(fc.get("seed", 0)),
                                                 intervals=want_intervals)
        else:
            res = batched.predict_batch_host(ctx, opts, fitted, future, floor, cap, seed=int(fc.get("seed", 0)),
                                             intervals=want_intervals, components=want_components)
        # "Negative forecast values found" log line (reference :76-79)
        neg = np.flatnonzero(ok & (np.trunc(res.yhat).min(axis=1) < floor))
        for i in neg[:100]:
            print(f"Negative forecast values found for series_id: {int(sid[i])}, dim_id: {int(did[i])}")
        cols = {
            "series_id": pa.array(np.repeat(sid, periods), pa.int32()),
            "dim_id": pa.array(np.repeat(did, periods), pa.int32()),
            "ds": pa.array(future.reshape(-1), pa.int64()).cast(pa.timestamp("ns")),
            "yhat": pa.array(res.yhat_int.reshape(-1), pa.int32()),
        }
        if want_intervals:
            cols["yhat_lower"] = pa.array(res.yhat_lower.reshape(-1), pa.float64())
            cols["yhat_upper"] = pa.array(res.yhat_upper.reshape(-1), pa.float64())
        for q, lv in enumerate(levels or ()):
            cols[quantile_column(lv)] = pa.array(res.quantiles[q].reshape(-1), pa.float64())
        if want_components:
            cols.update(component_columns(res, fitted.meta_i32[:, 3], periods, want_intervals,
                                          batched.seasonality_table(opts)))
        out = pa.table(cols)
        if not ok.all():
            out = out.filter(pa.array(np.repeat(ok, periods)))
        return out

    def _predict_regressors(self, ctx, opts, info, fitted, future, floor, cap, sid, did, ok, intervals):
        """Point forecasts (and intervals) of version-4 models: io.future_regressors joined onto the grids on the GPU,
        then pb200_predict_regressors_device with each record's (mu, std); the result on the host."""
        import torch
        torch.cuda.set_device(ctx.device)
        dev = torch.device("cuda", ctx.device)
        names = [r["name"] for r in info["regressors"]]
        tab = read_future_regressors(self.config["io"]["future_regressors"], names, sid)
        fut = torch.from_numpy(np.ascontiguousarray(future)).to(dev)
        freg = future_regressor_values(ctx, tab, names, sid, did, fut, ok)
        fd = batched.FittedBatch(*(torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (
            fitted.params, fitted.tchange, fitted.meta_i32, fitted.meta_i64, fitted.meta_f64)), fitted.smax, fitted.kmax,
            reg_scale=torch.from_numpy(np.ascontiguousarray(fitted.reg_scale)).to(dev))
        res = batched.predict_batch_device(ctx, opts, fd, fut, torch.from_numpy(floor).to(dev),
                                           torch.from_numpy(cap).to(dev), seed=int(self.config["forecast"].get("seed", 0)),
                                           intervals=intervals, regressors=freg)
        host = lambda t: None if t is None else t.cpu().numpy()  # noqa: E731
        return batched.ForecastBatch(future, host(res.yhat), host(res.yhat_lower), host(res.yhat_upper),
                                     host(res.yhat_int))

    def __call__(self, pdf):
        tbl = pa.Table.from_pandas(pdf, preserve_index=False)
        return self.apply_batched(tbl, ["series_id", "dim_id"]).to_pandas()


def forecast_time_series(config):
    """Forecast using trained time series model (series_id, dim_id) -- reference :18-104."""
    return _ForecastTimeSeriesOp(config)


def extract_date(datetimestamp: datetime):
    """reference :107-108."""
    return datetimestamp.date().strftime("%Y-%m-%d")


_ROWS_PER_PART = 1 << 20


def _strftime_via_dictionary(ts, fmt: str):
    """``pc.strftime`` costs 0.5-0.9 us per VALUE (seconds for millions of forecast rows, which the GPU computes in milliseconds), and a
    forecast frame repeats few distinct timestamps -- every model's horizon is the same handful of grid points.  Format the
    distinct values only and expand through the dictionary indices (a 20 ns per row memcpy).  Falls back to the direct call
    when most values are distinct."""
    chunks = ts.chunks if isinstance(ts, pa.ChunkedArray) else [ts]
    out = []
    for ch in chunks:
        if len(ch) == 0:
            out.append(pc.strftime(ch, format=fmt))
            continue
        enc = ch.dictionary_encode()
        if len(enc.dictionary) * 4 > len(ch):
            out.append(pc.strftime(ch, format=fmt))
        else:
            out.append(pa.DictionaryArray.from_arrays(enc.indices, pc.strftime(enc.dictionary, format=fmt)).cast(pa.string()))
    return pa.chunked_array(out, pa.string()) if isinstance(ts, pa.ChunkedArray) else out[0]


_GPU_ROWS_PER_PART = 4 << 20
_CSV_HEADER = b'"created_timestamp","series_id","dim_id","forecast_date","forecast_timestamp","forecast_quantity"\n'


def _gpu_writer_refusal(output_df: Frame, big_only: bool):
    """None if the frame can go through the GPU row formatter (csrc/csv_kernel.cuh), else the reason it cannot."""
    src = getattr(output_df, "forecast_source", None)
    if src is None:
        return "not the direct result of convert_forecasts"
    created, t = src
    if output_df.table.column_names != ["created_timestamp", "series_id", "dim_id", "forecast_date", "forecast_timestamp",
                                        "forecast_quantity"] or output_df.table.num_rows != t.num_rows:
        return "columns other than the standard six (interval columns keep the Arrow writer)"
    if big_only and t.num_rows <= _ROWS_PER_PART:
        return "small frame"
    if len(created.encode()) > 64:
        return "created_timestamp longer than 64 bytes"
    for c in ("series_id", "dim_id", "yhat"):
        if not pa.types.is_integer(t[c].type) or t[c].null_count:
            return f"column {c} is not a null-free integer column"
    if not pa.types.is_timestamp(t["ds"].type) or t["ds"].null_count:
        return "ds is not a null-free timestamp column"
    if t.num_rows and pc.min(pc.cast(t["ds"], pa.int64())).as_py() < 0:
        return "timestamps before 1970"
    try:
        import torch
        if not torch.cuda.is_available():
            return "no CUDA device"
    except Exception:
        return "no CUDA device"
    return None


def _write_forecasts_gpu(output_df: Frame, out: str, rank: int):
    """Part files of at most _GPU_ROWS_PER_PART rows: columns up through pack's pinned ring, rows formatted by
    pb200_forecast_csv_*_device, text back through two pinned buffers, file writes on a thread so that the GPU formats
    part k + 1 while part k goes to disk.  Byte for byte the Arrow writer's output (tests/test_gpu_jobs.py)."""
    import torch
    from concurrent.futures import ThreadPoolExecutor
    from ..pack import _device_column
    created, t = output_df.forecast_source
    ctx = get_context()
    torch.cuda.set_device(ctx.device)
    dev = torch.device("cuda", ctx.device)
    n = t.num_rows
    unit = t["ds"].type.unit
    mult = {"s": 10**9, "ms": 10**6, "us": 10**3, "ns": 1}[unit]
    bounds = list(range(0, n, _GPU_ROWS_PER_PART)) + [n]
    single = len(bounds) == 2
    host = [None, None]
    pending = [None, None]

    def dump(path, buf, nbytes):
        with open(path, "wb") as f:
            f.write(_CSV_HEADER)
            f.write(memoryview(buf.numpy())[:nbytes])

    with ThreadPoolExecutor(max_workers=2) as pool:
        for k in range(len(bounds) - 1):
            a, m = bounds[k], bounds[k + 1] - bounds[k]
            sid = _device_column(t["series_id"].slice(a, m), pa.int32(), dev)
            did = _device_column(t["dim_id"].slice(a, m), pa.int32(), dev)
            qty = _device_column(t["yhat"].slice(a, m), pa.int32(), dev)
            ds = _device_column(t["ds"].slice(a, m), pa.int64(), dev)
            if mult != 1:
                ds *= mult
            text = batched.forecast_csv_device(ctx, sid, did, ds, qty, created.encode())
            nbytes = int(text.numel())
            b = k & 1
            if pending[b] is not None:
                pending[b].result()                                    # the buffer's previous part is on disk
            if host[b] is None or host[b].numel() < nbytes:
                host[b] = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
            host[b][:nbytes].copy_(text)
            torch.cuda.current_stream(dev).synchronize()
            name = f"part-{rank:05d}.csv" if single else f"part-{rank:05d}-{k:04d}.csv"
            pending[b] = pool.submit(dump, os.path.join(out, name), host[b], nbytes)
        for p in pending:
            if p is not None:
                p.result()


class ProphetScorer:
    """Forecast quantities using trained models (reference :114-165)."""

    def __init__(self, config, logger=None):
        self.logger = logger or logging.getLogger(self.__class__.__name__)
        self.config = config

    def read_model_dataframe(self, spark=None) -> Frame:
        pdist.size_host_pools()             # pyarrow threads = this rank's share of the lease, not os.cpu_count()
        dset = pads.dataset(self.config["io"]["models"], format="parquet")
        return Frame(dset.to_table())

    @staticmethod
    def convert_forecasts(forecast_df: Frame) -> Frame:
        """reference :131-145; the per-row Python date UDF becomes one vectorised strftime."""
        created_timestamp = datetime.now(timezone.utc).replace(microsecond=0).isoformat()
        t = forecast_df.table
        n = t.num_rows
        ds = t["ds"]
        cols = {
            "created_timestamp": pa.array([created_timestamp] * n, pa.string()) if n < 1024 else
            pa.DictionaryArray.from_arrays(pa.array(np.zeros(n, np.int32)), pa.array([created_timestamp])).cast(pa.string()),
            "series_id": t["series_id"],
            "dim_id": t["dim_id"],
            "forecast_date": _strftime_via_dictionary(ds, "%Y-%m-%d"),
            "forecast_timestamp": ds,
            "forecast_quantity": t["yhat"],
        }
        quants = tuple(c for c in t.column_names if c.startswith("yhat_q"))
        known = {"series_id", "dim_id", "ds", "yhat", "yhat_lower", "yhat_upper", "trend_lower", "trend_upper",
                 *quants, *COMPONENT_COLUMNS}
        custom = tuple(c for c in t.column_names if c not in known)   # a seasonality table's component columns
        for extra in ("yhat_lower", "yhat_upper") + quants + COMPONENT_COLUMNS + custom + ("trend_lower", "trend_upper"):
            if extra in t.column_names:
                cols[extra] = t[extra]
        out = Frame(pa.table(cols))
        # what the frame was made from: lets write_forecasts format the rows on the GPU instead of from these columns
        out.forecast_source = (created_timestamp, t)
        return out

    def write_forecasts(self, output_df: Frame):
        """CSV with header, mode='overwrite' (reference :147-150); a directory of part files."""
        out = self.config["io"]["forecasts"]
        rank = pdist.world()[0]
        pdist.prepare_output_dir(out)
        t = output_df.table
        writer = (self.config.get("forecast", {}) or {}).get("writer", "auto")      # auto | gpu | arrow
        if writer not in ("auto", "gpu", "arrow"):
            raise ValueError("forecast.writer must be 'auto', 'gpu' or 'arrow'")
        if writer != "arrow":
            why = _gpu_writer_refusal(output_df, big_only=(writer == "auto"))
            if why is None:
                return _write_forecasts_gpu(output_df, out, rank)
            if writer == "gpu":
                raise ValueError("forecast.writer = 'gpu' cannot write this frame: " + why)
        if "forecast_timestamp" in t.column_names and pa.types.is_timestamp(t["forecast_timestamp"].type):
            # Spark's CSV writer prints timestamps as yyyy-MM-dd'T'HH:mm:ss.SSSXXX by default, e.g.
            # 2019-01-01T00:00:05.000Z.  Arrow's %S prints the fraction at the column's unit, so the column is
            # cast to milliseconds first (a timestamp[ns] column would print nine digits).
            i = t.column_names.index("forecast_timestamp")
            ms = pc.cast(t["forecast_timestamp"], pa.timestamp("ms"), safe=False)
            t = t.set_column(i, "forecast_timestamp", _strftime_via_dictionary(ms, "%Y-%m-%dT%H:%M:%SZ"))
        wo = pacsv.WriteOptions(include_header=True, quoting_style="needed")
        n = t.num_rows
        if n <= _ROWS_PER_PART:
            pacsv.write_csv(t, os.path.join(out, f"part-{rank:05d}.csv"), write_options=wo)
            return
        # a big frame goes out as several part files written concurrently (Spark's output is a directory of part files
        # too; pyarrow's CSV writer releases the GIL): config #5's 67 M rows are ~5 GB of text
        from concurrent.futures import ThreadPoolExecutor
        bounds = list(range(0, n, _ROWS_PER_PART)) + [n]
        def write(k):
            pacsv.write_csv(t.slice(bounds[k], bounds[k + 1] - bounds[k]),
                            os.path.join(out, f"part-{rank:05d}-{k:04d}.csv"), write_options=wo)
        with ThreadPoolExecutor(max_workers=max(1, pdist.size_host_pools())) as pool:
            list(pool.map(write, range(len(bounds) - 1)))

    def write_aggregates(self, aggregates: pa.Table, created_timestamp: str):
        """The window totals of forecast.aggregate as CSV with header under io.aggregates: one part file per rank,
        ``created_timestamp, series_id, dim_id, window_start, window_points, forecast_quantity, yhat, yhat_lower,
        yhat_upper[, yhat_q<level>...]``; window_start printed like forecast_timestamp."""
        out = self.config["io"]["aggregates"]
        rank = pdist.world()[0]
        pdist.prepare_output_dir(out)
        t = aggregates
        ms = pc.cast(t["window_start"], pa.timestamp("ms"), safe=False)
        t = t.set_column(t.column_names.index("window_start"), "window_start",
                         _strftime_via_dictionary(ms, "%Y-%m-%dT%H:%M:%SZ"))
        t = t.add_column(0, "created_timestamp", pa.array([created_timestamp] * t.num_rows, pa.string()))
        pacsv.write_csv(t, os.path.join(out, f"part-{rank:05d}.csv"),
                        write_options=pacsv.WriteOptions(include_header=True, quoting_style="needed"))

    @staticmethod
    def score(spark_session, config):
        aggregate_period(config)            # a bad forecast.aggregate_period, forecast.aggregate or forecast.quantiles
        aggregate_rule(config)              # fails before anything is read
        forecast_quantiles(config)
        aggregate_quantiles(config)
        pdist.init_process_group()          # no-op unless launched by torchrun with WORLD_SIZE > 1
        scorer = ProphetScorer(config)
        model_df = scorer.read_model_dataframe(spark_session)
        op = forecast_time_series(scorer.config)
        forecast_df = model_df.groupby("series_id", "dim_id").apply(op)
        if op.aggregates is not None:       # per-rank part files; forecast.gather below is for the forecast frame only
            scorer.write_aggregates(op.aggregates, datetime.now(timezone.utc).replace(microsecond=0).isoformat())
        if config["forecast"].get("gather", False) and pdist.world()[1] > 1:
            # optional: one NCCL gather of the final forecast frame to rank 0 (the only collective on
            # the path); default is one part file per rank, like Spark's output directory
            t = forecast_df.table
            cols = [np.ascontiguousarray(t[c].combine_chunks().to_numpy(zero_copy_only=False)) for c in t.column_names]
            cols = [c.astype("datetime64[ns]").astype(np.int64) if c.dtype.kind == "M" else c for c in cols]
            got = pdist.gather_rows(cols, dst=0)
            if got is None:
                pdist.prepare_output_dir(scorer.config["io"]["forecasts"])
                return
            # a seasonal component column's nulls travel as NaN (the rows of failed models, the only NaN ones, are gone)
            arrays = [pa.array(a, pa.int64()).cast(pa.timestamp("ns")) if n == "ds" else
                      pa.array(a, from_pandas=n in _SEASONAL_BIT) for n, a in zip(t.column_names, got)]
            forecast_df = Frame(pa.table(dict(zip(t.column_names, arrays))).cast(t.schema))
        converted_df = scorer.convert_forecasts(forecast_df)
        scorer.write_forecasts(converted_df)
