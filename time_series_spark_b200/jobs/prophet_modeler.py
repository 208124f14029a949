"""H100 drop-in for the reference's src/jobs/prophet_modeler.py.

Same names and contracts -- ``MODEL_INPUT_SCHEMA``, ``model_time_series(config)``,
``ProphetModeler(config).read_input_dataframe / persist_models``, ``ProphetModeler.model`` --
same YAML keys (``io.input``, ``io.models``, ``model.floor``, ``model.cap_multiplier``), same
header-less hive-partitioned CSV input and the same 5-column models table
``(series_id, dim_id, floor float32, cap float32, model binary)``.  What changes is the
engine: ``groupby('series_id','dim_id').apply(model_time_series(config))`` is ONE batched GPU
call over all groups (libprophet_b200.so) instead of one fbprophet/Stan fit per Spark task.
There is no Spark and no CPU fallback; ``spark`` arguments are accepted and ignored.

Optional keys beyond the reference (defaults reproduce prophet_modeler.py:65 exactly):
``model.growth``, ``model.seasonality_mode``, ``model.yearly_seasonality``,
``model.weekly_seasonality``, ``model.daily_seasonality``, ``model.n_changepoints``,
``model.changepoint_range``, ``model.changepoint_prior_scale``, ``model.seasonality_prior_scale``.

Seasonality tables (DESIGN §18): ``model.yearly_seasonality`` / ``weekly_seasonality`` / ``daily_seasonality`` also take
an int Fourier order (> 0 forces the built-in on at that order, 0 is off), and ``model.seasonalities`` is a list of
fbprophet ``add_seasonality`` calls in the order they are made: ``{name, period (days), fourier_order, prior_scale?
(default model.seasonality_prior_scale), mode? (must be model.seasonality_mode)}``.  With either key the options come
from ``batched.make_table_options`` and every error names the YAML key.  A custom name that is a column of the scorer's
frames (series_id, dim_id, ds, yhat, created_timestamp, forecast_date, forecast_timestamp, forecast_quantity, yhat_q...)
is refused here, since the scorer writes one component column per custom seasonality.  The models table then holds
version-2 records, which carry the table to the scorer; a table that restates the defaults (``yearly_seasonality: 10``)
is the default model and writes the same version-1 bytes as ``yearly_seasonality: true``.  ``io.warm_start`` (and so
``insample.refit`` with a warm start) is refused for a table; ``insample`` without it serves table models unchanged.

Extra regressors (DESIGN §20): ``model.regressors`` is a list of fbprophet ``add_regressor`` calls in the order they are
made, ``{name, prior_scale? (default model.holidays_prior_scale, 10.0), standardize? ('auto', true, false), mode? (must be
model.seasonality_mode)}``.  With it, regressor r is header-less CSV column 4 + r of the input (after ``quantity``), read
as float64; an empty field is null (NaN).  The options come from ``batched.make_regressor_options`` and every error names
the YAML key; a name that is a column of the input or the internal frame (series_id, dim_id, start_time, quantity, ds, y)
is refused.  Rows whose y is null are dropped before the values are looked at, as fbprophet fits on
``df[df['y'].notnull()]``; a NaN value on a kept row fails the job with fbprophet's ``ValueError("Found NaN in column
<name>")``.  The models table then holds version-4 records, which carry each series' standardisation (mu, std) and the
regressors to the scorer.  ``io.warm_start`` and the ``insample`` section are refused with regressors; the backtest takes them (DESIGN §20).  Without
``model.regressors`` (or with an empty list) the job reads, fits and writes what it did before.

``io.warm_start`` (optional): the path of a previous models table, for a job re-run on a schedule over the same groups
plus new rows (fbprophet's "updating fitted models", ``m.fit(df, init=stan_init(m_old))``).  Every group starts its
fit from its row of that table when the row's changepoint count and seasonalities are those of the new history
(DESIGN §11), else from fbprophet's cold start; one line reports how many were warm, how many cold and why, and
how many table rows matched no input group.  The table must have been fitted with the job's growth, seasonality mode,
seasonality switches and ``n_changepoints``.  It may be ``io.models`` itself: the old table is read before it is
replaced.  Without the key the job is the cold fit it has always been.

``insample`` (optional section): fbprophet's in-sample predict, ``m.predict()`` with no frame, for every fitted group
(DESIGN §16).  ``insample.interval_width`` (required, in [0, 1]) decides what counts as an outlier: a history row whose
y lies outside its ``yhat_lower`` / ``yhat_upper``, from ``insample.uncertainty_samples`` draws (default 1000, in
[2, 1024]) keyed by ``insample.seed`` (default 0).  ``io.fitted`` (optional) receives one parquet part file per rank with
one row per history row of every group that got a model, in the packed order: ``series_id, dim_id, ds, y`` (y in the
input column's type), ``yhat, yhat_lower, yhat_upper`` (float64) and ``outlier`` (bool).  ``insample.refit: true``
(default false) drops the flagged rows and fits again on the device, with the same options and ``io.warm_start``:
``io.models`` then holds the models a plain run gives on the input without those rows (a group left with fewer than 2
rows raises), while ``io.fitted`` still describes the first fit, the one the flags come from.  The section needs
``io.fitted`` or ``refit: true``; one line reports the rows predicted and flagged and the series flagged and refitted.
Without the section the job is what it was.
"""
from __future__ import annotations

import glob
import logging
import os
import time

import numpy as np
import pyarrow as pa
import pyarrow.csv as pacsv
import pyarrow.dataset as pads
import pyarrow.parquet as pq

from .. import _lib as L
from .. import batched, model_record
from .. import dist as pdist
from ..frame import Frame
from ..pack import pack_groups, pack_groups_cuda

# reference prophet_modeler.py:12-17 (Spark StructType -> Arrow)
MODEL_INPUT_SCHEMA = pa.schema([
    pa.field("series_id", pa.int32(), True),
    pa.field("dim_id", pa.int32(), True),
    pa.field("start_time", pa.timestamp("ns"), True),
    pa.field("quantity", pa.int32(), True),
])

# reference prophet_modeler.py:32-38
MODEL_OUTPUT_SCHEMA = pa.schema([
    pa.field("series_id", pa.int32(), True),
    pa.field("dim_id", pa.int32(), True),
    pa.field("floor", pa.float32(), True),
    pa.field("cap", pa.float32(), True),
    pa.field("model", pa.binary(), True),
])

_contexts = {}


def get_context(device=None) -> L.Context:
    """One pb200 context per (process, device); LOCAL_RANK picks the device under torchrun."""
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0"))
    if device not in _contexts:
        _contexts[device] = L.Context(device)
    return _contexts[device]


_BUILTIN_KEYS = ("yearly_seasonality", "weekly_seasonality", "daily_seasonality")

# columns of the scorer's frames a custom seasonality's component column must not shadow: the internal frame's and the
# written CSV's (convert_forecasts); names starting with yhat_q are the quantile columns
SCORER_COLUMNS = frozenset(["series_id", "dim_id", "ds", "yhat", "created_timestamp", "forecast_date",
                            "forecast_timestamp", "forecast_quantity"])


def table_keys(config) -> list:
    """The ``model.*`` keys that make the job's model a seasonality table: ``model.seasonalities`` and the built-in
    switches given as an int order."""
    m = config.get("model", {}) or {}
    keys = [f"model.{k}" for k in _BUILTIN_KEYS
            if isinstance(m.get(k), (int, np.integer)) and not isinstance(m.get(k), (bool, np.bool_))]
    return keys + (["model.seasonalities"] if "seasonalities" in m else [])


def _model_key_error(e: ValueError, keys) -> ValueError:
    """make_table_options' (or make_regressor_options') message with each key it names spelled as its YAML key
    (model.<key>); a message that names none (the library's limits) is prefixed with the table's keys."""
    import re
    msg = str(e)
    named = re.sub(r"(?<![\w.])(seasonalities(?=[\[:])|regressors(?=[\[:])|yearly_seasonality|weekly_seasonality|"
                   r"daily_seasonality|seasonality_mode|holidays_prior_scale)", r"model.\1", msg)
    return ValueError(named if named != msg else f"{' / '.join(keys)}: {msg}")


# columns of the modeler's input and internal frames a regressor's column must not be named like (fbprophet's
# validate_column_name refuses ds and y itself)
INPUT_COLUMNS = frozenset(["series_id", "dim_id", "start_time", "quantity"])


def regressor_keys(config) -> list:
    """The ``model.*`` keys of extra regressors the config gives: ``model.regressors``, ``model.holidays_prior_scale``."""
    m = config.get("model", {}) or {}
    return [f"model.{k}" for k in ("regressors", "holidays_prior_scale") if k in m]


def regressor_names(config) -> list:
    """The names of ``model.regressors`` in order (the input's extra columns), [] without regressors; raises ValueError
    naming the key for a value that is not a list and for a name that is a column of the input or internal frames."""
    regs = (config.get("model", {}) or {}).get("regressors")
    if regs is None:
        return []
    if not isinstance(regs, (list, tuple)):
        raise ValueError(f"model.regressors must be a list of {{name, prior_scale?, standardize?, mode?}} (got {regs!r})")
    names = []
    for i, spec in enumerate(regs):
        name = spec.get("name") if isinstance(spec, dict) else None
        if isinstance(name, str) and name in INPUT_COLUMNS:
            raise ValueError(f"model.regressors[{i}].name: {name!r} is a column of the modeler's input; a regressor "
                             "column must have a name of its own")
        names.append(name)
    return names


def options_from_config(config) -> L.Options:
    """The job's fit options from ``model.*``.  Without ``model.seasonalities`` and without an int order for a built-in,
    batched.make_options as always; with either, batched.make_table_options (DESIGN §18), whose errors name the YAML key.
    A table that restates the default model gives the same pb200_options as the switches alone.  With
    ``model.regressors`` (DESIGN §20), batched.make_regressor_options with the same table keywords; an empty list (or
    ``model.holidays_prior_scale`` alone) is checked and then gives the options without it."""
    m = dict(config.get("model", {}) or {})
    kw = dict(growth=m.get("growth", "logistic"),
              seasonality_mode=m.get("seasonality_mode", "multiplicative"),
              n_changepoints=m.get("n_changepoints", 25),
              changepoint_range=m.get("changepoint_range", 0.8),
              changepoint_prior_scale=m.get("changepoint_prior_scale", 0.05),
              seasonality_prior_scale=m.get("seasonality_prior_scale", 10.0))
    keys = table_keys(config)
    rkeys = regressor_keys(config)
    if rkeys:
        names = regressor_names(config)
        seas = m.get("seasonalities")
        if seas is not None and not isinstance(seas, (list, tuple)):
            raise ValueError(f"model.seasonalities must be a list of {{name, period, fourier_order, prior_scale?, "
                             f"mode?}} (got {seas!r})")
        try:
            ropts = batched.make_regressor_options(regressors=m.get("regressors") or [],
                                                   holidays_prior_scale=m.get("holidays_prior_scale", 10.0),
                                                   seasonalities=seas or [],
                                                   **{k: m.get(k, "auto") for k in _BUILTIN_KEYS}, **kw)
        except ValueError as e:
            raise _model_key_error(e, keys + rkeys) from None
        if names:
            return ropts
    if not keys:
        return batched.make_options(yearly_seasonality=m.get("yearly_seasonality", "auto"),
                                    weekly_seasonality=m.get("weekly_seasonality", "auto"),
                                    daily_seasonality=m.get("daily_seasonality", "auto"), **kw)
    seas = m.get("seasonalities")
    if seas is None:
        seas = []
    if not isinstance(seas, (list, tuple)):
        raise ValueError(f"model.seasonalities must be a list of {{name, period, fourier_order, prior_scale?, mode?}} "
                         f"(got {seas!r})")
    for i, spec in enumerate(seas):
        name = spec.get("name") if isinstance(spec, dict) else None
        if isinstance(name, str) and (name in SCORER_COLUMNS or name.startswith("yhat_q")):
            raise ValueError(f"model.seasonalities[{i}].name: {name!r} is a column of the scorer's forecast frames; its "
                             "component column would shadow it")
    try:
        opts = batched.make_table_options(seasonalities=seas, **{k: m.get(k, "auto") for k in _BUILTIN_KEYS}, **kw)
    except ValueError as e:
        raise _model_key_error(e, keys) from None
    if batched.is_table(opts):
        return opts
    v1 = L.Options.from_buffer_copy(opts)
    v1.abi_version = L.ABI_VERSION
    return v1


def refuse_table_warm_start(config, opts) -> None:
    """Warm start needs the previous optimum in the options' layout, which the library takes for the default model only:
    a seasonality table with ``io.warm_start`` (also under ``insample.refit``) raises, naming both keys."""
    if batched.is_table(opts) and (config.get("io") or {}).get("warm_start"):
        raise ValueError(f"io.warm_start is not available for a model with a seasonality table "
                         f"({', '.join(table_keys(config))}): warm start serves the default seasonalities only"
                         + (" (insample.refit would start from it too)" if "insample" in config else ""))


def refuse_regressors(config) -> None:
    """Warm start and the in-sample predict have no regressor values: ``io.warm_start`` (and so ``insample.refit`` with
    it) and the ``insample`` section raise with ``model.regressors``, naming both keys, before any GPU work."""
    if not regressor_names(config):
        return
    if (config.get("io") or {}).get("warm_start"):
        raise ValueError("io.warm_start is not available with model.regressors: warm start serves models without extra "
                         "regressors only" + (" (insample.refit would start from it too)" if "insample" in config else ""))
    if "insample" in config:
        raise ValueError("insample is not available with model.regressors: the in-sample predict of a model with extra "
                         "regressors is not implemented")


def who(series_id, dim_id, mask) -> str:
    """The first offending group of a per-series bool mask, and how many there are, for an error message."""
    i = int(np.flatnonzero(mask)[0])
    return (f" (first offender: series_id {int(series_id[i])}, dim_id {int(dim_id[i])}; "
            f"{int(np.count_nonzero(mask))} group(s) in all)")


def _group_keys(series_id, dim_id) -> np.ndarray:
    """One int64 key per (series_id, dim_id) group."""
    return (np.asarray(series_id, dtype=np.int64) << 32) | (np.asarray(dim_id, dtype=np.int64) & 0xFFFFFFFF)


INSAMPLE_KEYS = ("interval_width", "uncertainty_samples", "seed", "refit")

# the io.fitted frame, but for y, which keeps the input column's type
FITTED_COLUMNS = [("series_id", pa.int32()), ("dim_id", pa.int32()), ("ds", pa.timestamp("ns")), ("y", None),
                  ("yhat", pa.float64()), ("yhat_lower", pa.float64()), ("yhat_upper", pa.float64()),
                  ("outlier", pa.bool_())]


def fitted_schema(y_type) -> pa.Schema:
    """The schema of the io.fitted frame for an input y column of type ``y_type``."""
    return pa.schema([pa.field(n, y_type if t is None else t, True) for n, t in FITTED_COLUMNS])


def insample_options(config):
    """The ``insample`` section as ``{interval_width, uncertainty_samples, seed, refit}`` with its defaults, or None when
    the config has no such section.  Raises ValueError naming the key for an unknown key, a missing or out-of-range
    ``interval_width``, ``uncertainty_samples`` outside [2, 1024], a bad ``seed`` or ``refit``, and for a section that
    would write nothing (neither ``io.fitted`` nor ``refit: true``)."""
    if "insample" not in config:
        return None
    sec = config["insample"]
    if not isinstance(sec, dict):
        raise ValueError(f"insample must be a mapping with at least insample.interval_width (got {sec!r})")
    unknown = sorted(set(sec) - set(INSAMPLE_KEYS))
    if unknown:
        raise ValueError(f"insample.{unknown[0]} is not a known key (known: {', '.join(INSAMPLE_KEYS)})")
    if "interval_width" not in sec:
        raise ValueError("insample.interval_width is required: it decides which history rows are outliers")
    w = sec["interval_width"]
    if isinstance(w, bool) or not isinstance(w, (int, float)) or not 0.0 <= float(w) <= 1.0:
        raise ValueError(f"insample.interval_width must be a number in [0, 1] (got {w!r})")
    n = sec.get("uncertainty_samples", 1000)
    if isinstance(n, bool) or not isinstance(n, int) or not 2 <= n <= 1024:
        raise ValueError(f"insample.uncertainty_samples must be an integer in [2, 1024] (got {n!r})")
    seed = sec.get("seed", 0)
    if isinstance(seed, bool) or not isinstance(seed, int) or not 0 <= seed < 2**64:
        raise ValueError(f"insample.seed must be an integer in [0, 2^64) (got {seed!r})")
    refit = sec.get("refit", False)
    if not isinstance(refit, bool):
        raise ValueError(f"insample.refit must be true or false (got {refit!r})")
    if not refit and not (config.get("io") or {}).get("fitted"):
        raise ValueError("insample needs io.fitted or insample.refit: true; as configured it would do nothing")
    return {"interval_width": float(w), "uncertainty_samples": int(n), "seed": int(seed), "refit": refit}


def insample_report(rows: int, flagged: int, series_flagged: int, refitted: int) -> str:
    """The job's one line about the in-sample predict."""
    return (f"In-sample: {rows} rows predicted, {flagged} flagged as outliers in {series_flagged} series; "
            f"{refitted} series refitted without them")


def null_rows_last_ds(table: pa.Table, series_id, dim_id) -> np.ndarray:
    """Per packed group ``(series_id, dim_id)``, the latest ds (ns) of its rows whose y is null or NaN, INT64_MIN for a
    group without one.  The pack drops those rows, but they count for the group's ``last_ds``, and a refit keeps them."""
    import pyarrow.compute as pc
    out = np.full(len(series_id), np.iinfo(np.int64).min, np.int64)
    null = pc.is_null(table["y"], nan_is_null=True)
    if not pc.any(null).as_py():
        return out
    sub = table.filter(null)
    ds = pc.cast(pc.cast(sub["ds"], pa.timestamp("ns")), pa.int64()).to_numpy()
    key = _group_keys(sub["series_id"].to_numpy(), sub["dim_id"].to_numpy())
    gkey = _group_keys(series_id, dim_id)
    order = np.argsort(gkey, kind="stable")
    pos = np.minimum(np.searchsorted(gkey[order], key), gkey.size - 1)
    hit = gkey[order][pos] == key
    np.maximum.at(out, order[pos[hit]], ds[hit])
    return out


def warm_start_init(table: pa.Table, opts: L.Options, series_id, dim_id, path: str = "io.warm_start"):
    """The previous models of the packed groups ``(series_id, dim_id)`` from a models table (MODEL_OUTPUT_SCHEMA), as
    the ``init`` of ``batched.fit_batch_device``: a host FittedBatch in the groups' order whose rows without a previous
    model have status -1.  Returns ``(init, unmatched)``, ``unmatched`` the number of table rows that match no group.
    Raises ValueError (naming ``path``) for a table fitted with other options or with a seasonality table, and for
    duplicate keys."""
    lay = L.get_layout(opts)
    n = len(series_id)
    gkey = _group_keys(series_id, dim_id)
    init = batched.FittedBatch(np.zeros((n, lay.pstride)), np.zeros((n, lay.smax)), np.zeros((n, 8), np.int32),
                               np.zeros((n, 2), np.int64), np.zeros((n, 4)), lay.smax, lay.kmax)
    init.meta_i32[:, 4] = -1
    if table.num_rows == 0:
        return init, 0
    tsid = table["series_id"].combine_chunks().to_numpy(zero_copy_only=False)
    tdid = table["dim_id"].combine_chunks().to_numpy(zero_copy_only=False)
    tkey = _group_keys(tsid, tdid)
    order = np.argsort(tkey, kind="stable")
    skey = tkey[order]
    dup = np.zeros(tkey.size, bool)
    dup[order[1:][skey[1:] == skey[:-1]]] = True
    if dup.any():
        raise ValueError(f"{path} holds more than one model for a (series_id, dim_id) group." + who(tsid, tdid, dup))
    prev, _, info = model_record.decode(table["model"])
    if "table" in info:
        # a seasonality table's records hold its mask and betas in the table's column order, not the default model's
        raise ValueError(f"{path} holds models fitted with a seasonality table (version-2 records); warm start serves "
                         "the default seasonalities only")
    want = {"logistic": opts.growth == L.GROWTH_LOGISTIC, "multiplicative": bool(opts.multiplicative),
            "yearly": int(opts.yearly), "weekly": int(opts.weekly), "daily": int(opts.daily),
            "n_changepoints": int(opts.n_changepoints)}
    diff = sorted(k for k in want if info[k] != want[k])
    if diff:
        raise ValueError(f"{path} was fitted with other options than this job's: " +
                         ", ".join(f"{k} {info[k]!r} (job: {want[k]!r})" for k in diff))
    pos = np.minimum(np.searchsorted(skey, gkey), skey.size - 1)
    hit = skey[pos] == gkey
    rows = order[pos[hit]]
    init.params[hit] = prev.params[rows]
    init.meta_i32[hit] = prev.meta_i32[rows]
    init.meta_i64[hit] = prev.meta_i64[rows]
    init.meta_f64[hit] = prev.meta_f64[rows]
    init.tchange[hit] = prev.tchange[rows]
    gsorted = np.sort(gkey)
    gp = np.minimum(np.searchsorted(gsorted, tkey), max(gsorted.size - 1, 0))
    unmatched = int(np.count_nonzero(gsorted[gp] != tkey)) if gsorted.size else int(tkey.size)
    return init, unmatched


def read_warm_start(path: str, series_id) -> pa.Table:
    """The rows of the models table at ``path`` whose series_id is one of ``series_id`` (under torchrun: this rank's)."""
    import pyarrow.compute as pc
    sids = pa.array(np.unique(np.asarray(series_id, dtype=np.int32)), pa.int32())
    return pads.dataset(path, format="parquet").to_table(filter=pc.field("series_id").isin(sids))


def warm_report(warm, unmatched: int) -> str:
    """The job's one line about where its fits started."""
    w = np.asarray(warm)
    return (f"Warm start: {int(np.count_nonzero(w == L.WARM_USED))} series warm; cold: "
            f"{int(np.count_nonzero(w == L.WARM_NONE))} without a previous model or not optimised, "
            f"{int(np.count_nonzero(w == L.WARM_SHAPE))} whose changepoints or seasonalities changed, "
            f"{int(np.count_nonzero(w == L.WARM_BAD))} with unusable previous values; "
            f"{unmatched} table row(s) matched no input group")


def models_table(fitted: batched.FittedBatch, series_id, dim_id, last_ds, opts: L.Options, floor) -> pa.Table:
    """The models table (MODEL_OUTPUT_SCHEMA) of a fitted batch (host arrays).  fbprophet's ValueErrors (cap <= floor,
    bad input) raise, naming the group; a failed fit (status < 0) -- the reference's RuntimeError -- prints a line and
    gets no row (prophet_modeler.py:81-85)."""
    n = fitted.n
    status = fitted.meta_i32[:, 4]
    if np.any(status == L.ST_CAP_LE_FLOOR):
        raise ValueError("cap must be greater than floor (which defaults to 0)." + who(series_id, dim_id, status == L.ST_CAP_LE_FLOOR))
    if np.any(status == L.ST_BAD_INPUT):
        raise ValueError("Found non-finite y or a zero time span in a series." + who(series_id, dim_id, status == L.ST_BAD_INPUT))
    bad = status == L.ST_BAD_REGRESSOR
    if np.any(bad):
        # fbprophet's setup_dataframe: "Found NaN in column <name>"; the regressor is the first one whose scale is NaN
        i = int(np.flatnonzero(bad)[0])
        r = int(np.flatnonzero(np.isnan(np.asarray(fitted.reg_scale)[i, :, 0]))[0])
        raise ValueError(f"Found NaN in column {opts.regressors[r].name.decode()}" + who(series_id, dim_id, bad))
    ok = status >= 0
    for i in np.flatnonzero(~ok):
        print(f"Runtime error (solver status {int(status[i])}) for series_id: {int(series_id[i])}, "
              f"dim_id: {int(dim_id[i])}")
    blobs = model_record.encode(fitted, last_ds, opts)
    cap64 = fitted.meta_f64[:, 2]
    out = pa.table({
        "series_id": pa.array(series_id, pa.int32()),
        "dim_id": pa.array(dim_id, pa.int32()),
        "floor": pa.array(np.full(n, floor, dtype=np.float32), pa.float32()),
        "cap": pa.array(cap64.astype(np.float32), pa.float32()),   # FloatType column, prophet_modeler.py:36
        "model": blobs,
    })
    if not ok.all():
        out = out.filter(pa.array(ok))
    return out


class _ModelTimeSeriesOp:
    """Batched GROUPED_MAP operator: all (series_id, dim_id) groups in one GPU launch."""

    def __init__(self, config):
        self.config = config

    def apply_batched(self, table: pa.Table, keys) -> pa.Table:
        execution_time = time.time()
        if list(keys) != ["series_id", "dim_id"]:
            raise ValueError("model_time_series groups by ('series_id', 'dim_id')")
        floor = self.config["model"]["floor"]
        cap_multiplier = self.config["model"]["cap_multiplier"]
        ins = insample_options(self.config)
        if table_keys(self.config):         # a table's refusals come before any GPU work
            refuse_table_warm_start(self.config, options_from_config(self.config))
        reg_names = regressor_names(self.config)
        if reg_names:                       # and so do the regressors'
            refuse_regressors(self.config)
            options_from_config(self.config)
        with_frame = ins is not None and bool((self.config.get("io") or {}).get("fitted"))
        # this rank's io.fitted frame (empty until a group is predicted)
        self.fitted_table = fitted_schema(table.schema.field("y").type).empty_table() if with_frame else None
        ctx = get_context()
        # group + sort on the GPU (two radix sorts), ds / y stay in HBM for the fit
        import torch
        torch.cuda.set_device(ctx.device)
        pk = pack_groups_cuda(table, device=f"cuda:{ctx.device}", reg_cols=reg_names)
        torch.cuda.synchronize()
        t_pack = time.time()
        rank, ws, _ = pdist.world()
        if ws > 1 and not getattr(self, "rank_local_input", False):
            # the table holds EVERY group (the caller did not read rank-locally): this rank fits its contiguous,
            # row-balanced shard of them
            lo, hi = pdist.shard_bounds(pk.offsets, ws)[rank]
            pk = pk.take(lo, hi)
        if pk.n == 0:
            return MODEL_OUTPUT_SCHEMA.empty_table()
        opts = options_from_config(self.config)
        print(f"Modeling {pk.n} series with {int(pk.offsets[-1])} modeling rows")
        # fbprophet raises ValueError (task failure, not RuntimeError) for < 2 rows:
        # keep that observable behaviour (prophet_modeler.py:81 only catches RuntimeError)
        short = np.diff(pk.offsets) < 2
        if np.any(short):
            raise ValueError("Dataframe has less than 2 non-NaN rows." + who(pk.series_id, pk.dim_id, short))
        warm_path = (self.config.get("io") or {}).get("warm_start")
        init = None
        if warm_path:
            init, unmatched = warm_start_init(read_warm_start(warm_path, pk.series_id), opts, pk.series_id, pk.dim_id)
        fitted_d = batched.fit_batch_device(ctx, opts, pk.ds.contiguous(), pk.y.contiguous(), pk.offsets,
                                            float(floor), float(cap_multiplier), init=init, regressors=pk.regressors)
        fitted = fitted_d.to_host()
        if warm_path:
            print(warm_report(fitted.warm, unmatched))
        t_fit = time.time()
        if ins is None:
            out = models_table(fitted, pk.series_id, pk.dim_id, pk.last_ds, opts, floor)
        else:
            out = self._insample(ctx, opts, ins, table, pk, fitted_d, fitted, floor, cap_multiplier, init,
                                 unmatched if warm_path else 0)
        # wall time per stage of the last call (tools/e2e_scaling.py reports them): upload + group + sort, GPU fit + D2H, encode
        self.last_timings = {"pack_s": t_pack - execution_time, "fit_s": t_fit - t_pack, "encode_s": time.time() - t_fit}
        print(f"Output df {out.num_rows} models trained in {time.time() - execution_time}")
        return out

    def _insample(self, ctx, opts, ins, table, pk, fitted_d, fitted, floor, cap_multiplier, init, unmatched):
        """The in-sample predict of the fitted batch, its outlier flags, the io.fitted frame and (insample.refit) the
        fit without the flagged rows; returns the models table the job writes."""
        import torch
        iopts = batched.copy_options(opts)
        iopts.interval_width = ins["interval_width"]
        iopts.uncertainty_samples = ins["uncertainty_samples"]
        # fbprophet predicts the history with the floor and cap it was fitted on: the fit's own (float64) values
        fl = fitted_d.meta_f64[:, 1].contiguous()
        cp = fitted_d.meta_f64[:, 2].contiguous()
        hf = batched.predict_history_device(ctx, iopts, fitted_d, pk.ds, pk.offsets, fl, cp, seed=ins["seed"])
        ol = batched.outliers_device(ctx, pk.ds, pk.y, pk.offsets, hf.yhat_lower, hf.yhat_upper)
        ok = fitted.meta_i32[:, 4] >= 0
        T = np.diff(pk.offsets)
        lost = T - ol.kept                                  # flagged rows per group (0 for a failed fit: NaN bounds)
        if self.fitted_table is not None:
            row_ok = np.repeat(ok, T)
            y_type = self.fitted_table.schema.field("y").type
            cols = {
                "series_id": np.repeat(pk.series_id, T), "dim_id": np.repeat(pk.dim_id, T),
                "ds": pk.ds.cpu().numpy().view("datetime64[ns]"), "y": pk.y.cpu().numpy(),
                "yhat": hf.yhat.cpu().numpy(), "yhat_lower": hf.yhat_lower.cpu().numpy(),
                "yhat_upper": hf.yhat_upper.cpu().numpy(), "outlier": ol.flag.cpu().numpy().astype(bool),
            }
            arrays = [pa.array(cols[n][row_ok], type=y_type if t is None else t) if n != "y"
                      else pa.array(cols[n][row_ok]).cast(y_type) for n, t in FITTED_COLUMNS]
            self.fitted_table = pa.Table.from_arrays(arrays, schema=self.fitted_table.schema)
        refitted = 0
        if not ins["refit"]:
            out = models_table(fitted, pk.series_id, pk.dim_id, pk.last_ds, opts, floor)
        else:
            short = np.diff(ol.offsets) < 2
            if np.any(short):
                raise ValueError("Dataframe has less than 2 non-NaN rows." + who(pk.series_id, pk.dim_id, short))
            refit = batched.fit_batch_device(ctx, opts, ol.ds, ol.y, ol.offsets, float(floor), float(cap_multiplier),
                                             init=init).to_host()
            if init is not None:
                print(warm_report(refit.warm, unmatched))
            kept_last = ol.ds[torch.from_numpy(ol.offsets[1:] - 1).to(ol.ds.device)].cpu().numpy()
            last_ds = np.maximum(kept_last, null_rows_last_ds(table, pk.series_id, pk.dim_id))
            out = models_table(refit, pk.series_id, pk.dim_id, last_ds, opts, floor)
            refitted = pk.n
        print(insample_report(int(T[ok].sum()), int(lost.sum()), int(np.count_nonzero(lost > 0)), refitted))
        return out

    def __call__(self, pdf):
        """Per-group form of the UDF (one pandas frame in, one-row frame out), for callers that
        still iterate groups themselves."""
        tbl = pa.Table.from_pandas(pdf[["series_id", "dim_id", "ds", "y"]], preserve_index=False)
        return self.apply_batched(tbl, ["series_id", "dim_id"]).to_pandas()


def rank_local_files(dset, rank: int, world_size: int):
    """Files of the hive-partitioned input this rank reads: the ``series_id=`` directories in ascending id order,
    cut into ``world_size`` contiguous ranges of (nearly) equal bytes.  Returns None when there are fewer
    directories than ranks (the caller then reads everything and shards the packed groups instead)."""
    by_sid = {}
    for f in dset.get_fragments():
        sid = pads.get_partition_keys(f.partition_expression).get("series_id")
        if sid is None:
            return None
        try:
            size = os.path.getsize(f.path)
        except OSError:
            size = 1
        ent = by_sid.setdefault(int(sid), [0, []])
        ent[0] += max(size, 1)
        ent[1].append(f.path)
    sids = sorted(by_sid)
    if len(sids) < world_size:
        return None
    sizes = np.array([by_sid[s][0] for s in sids], dtype=np.int64)
    offs = np.concatenate(([0], np.cumsum(sizes)))
    lo, hi = pdist.shard_bounds(offs, world_size)[rank]
    return [p for s in sids[lo:hi] for p in sorted(by_sid[s][1])]


def model_time_series(config):
    """Model time series per dimensions (series_id, dim_id)  -- reference prophet_modeler.py:22-87."""
    return _ModelTimeSeriesOp(config)


class ProphetModeler:
    """Create models to forecast quantities (reference prophet_modeler.py:90-143)."""

    def __init__(self, config, logger=None):
        self.logger = logger or logging.getLogger(self.__class__.__name__)
        self.config = config

    def read_input_dataframe(self, spark=None) -> Frame:
        """Header-less CSV ``dim_id,timestamp,quantity`` under hive dirs ``series_id=<int>/``
        (reference :102-116; fixture tests/fixtures/model-input).  Returns columns
        series_id, dim_id, ds, y -- and with ``model.regressors`` one float64 column per regressor, named as it is,
        read from the CSV columns after quantity (an empty field is null)."""
        pdist.size_host_pools()             # pyarrow threads = this rank's share of the lease, not os.cpu_count()
        path = self.config["io"]["input"]
        part = pads.partitioning(pa.schema([("series_id", pa.int32())]), flavor="hive")
        regs = regressor_names(self.config)
        names = [f.name for f in MODEL_INPUT_SCHEMA if f.name != "series_id"] + regs
        types = {f.name: f.type for f in MODEL_INPUT_SCHEMA if f.name != "series_id"}
        types.update({r: pa.float64() for r in regs})
        fmt = pads.CsvFileFormat(
            read_options=pacsv.ReadOptions(column_names=names),
            convert_options=pacsv.ConvertOptions(
                column_types=types, timestamp_parsers=["%Y-%m-%d %H:%M:%S", pacsv.ISO8601]))
        dset = pads.dataset(path, format=fmt, partitioning=part, exclude_invalid_files=False,
                            ignore_prefixes=[".", "_"])
        # Rank-local ingestion (SURVEY 8e): a group never spans two ``series_id=`` directories, so under torchrun each
        # rank parses, uploads and sorts only its own contiguous, byte-balanced range of directories -- the
        # counterpart of Spark tasks reading their own input splits.  With fewer directories than ranks every
        # rank reads everything and the groups are range-sharded after the pack instead.
        rank, ws, _ = pdist.world()
        self.rank_local_input = False
        if ws > 1:
            mine = rank_local_files(dset, rank, ws)
            if mine is not None:
                self.rank_local_input = True
                if not mine:
                    empty = pa.schema([("series_id", pa.int32()), ("dim_id", pa.int32()), ("ds", pa.timestamp("ns")),
                                       ("y", pa.int32())] + [(r, pa.float64()) for r in regs]).empty_table()
                    return Frame(empty)
                dset = pads.dataset(mine, format=fmt, partitioning=part, partition_base_dir=path,
                                    exclude_invalid_files=False)
        tbl = dset.to_table(columns=["series_id", "dim_id", "start_time", "quantity"] + regs)
        tbl = tbl.rename_columns(["series_id", "dim_id", "ds", "y"] + regs)
        return Frame(tbl)

    def persist_models(self, model_df: Frame):
        """Parquet, mode='overwrite' (reference :118-125); one part file per writer."""
        out = self.config["io"]["models"]
        rank = pdist.world()[0]
        if self.config["io"].get("warm_start"):
            pdist.barrier()                 # io.warm_start may be io.models: every rank has read it before rank 0 clears it
        pdist.prepare_output_dir(out)
        pq.write_table(model_df.table, os.path.join(out, f"part-{rank:05d}.parquet"))

    def persist_fitted(self, fitted: pa.Table):
        """The in-sample frame (insample with io.fitted): parquet, mode='overwrite', one part file per rank."""
        out = self.config["io"]["fitted"]
        pdist.prepare_output_dir(out)
        pq.write_table(fitted, os.path.join(out, f"part-{pdist.world()[0]:05d}.parquet"))

    @staticmethod
    def model(spark_session, config):
        """Create the trained time series models (reference :127-143)."""
        pdist.init_process_group()          # no-op unless launched by torchrun with WORLD_SIZE > 1
        scorer = ProphetModeler(config)
        input_df = scorer.read_input_dataframe(spark_session)
        op = model_time_series(scorer.config)
        op.rank_local_input = getattr(scorer, "rank_local_input", False)
        model_df = input_df.groupby("series_id", "dim_id").apply(op)
        scorer.persist_models(model_df)
        if getattr(op, "fitted_table", None) is not None:
            scorer.persist_fitted(op.fitted_table)
