"""Tuning job: fbprophet's documented hyperparameter search over the prior scales, for every (series_id, dim_id) group.

For each group and each point of the grid ``changepoint_prior_scale x seasonality_prior_scale`` (enumerated as
``itertools.product``), the job backtests the group (cross_validation with the ``backtest`` section's horizon, period and
initial) and scores it with performance_metrics(rolling_window=1) -- one number over all held-out rows.  The grid point
with the lowest score wins (the first in enumeration order on ties); the group is then fitted on its full history with
that pair.  A group with no eligible grid point (a failed cutoff fit, or a score that is not finite, e.g. mape on a group
with a zero) keeps the ``model.*`` prior scales.  All of it is one batched GPU job (batched.tune_device; DESIGN §10).

Keys: ``io.input``, ``model.*`` as the modeler, but for a seasonality table (``model.seasonalities`` or an int order
for a built-in, which raises: per-series prior scales are not available for tables; ``model.regressors`` raises too); ``backtest.horizon`` / ``period`` / ``initial`` as the backtest; and
``tune.*``:
  changepoint_prior_scale   list of values > 0, default [0.001, 0.01, 0.1, 0.5]
  seasonality_prior_scale   list of values > 0, default [0.01, 0.1, 1.0, 10.0]
  metric                    mse | rmse | mae | mape, default rmse
Outputs (parquet, one part file per rank):
  io.models   the modeler's table (series_id, dim_id, floor, cap, model): the scorer reads it unchanged
  io.tuning   series_id, dim_id, changepoint_prior_scale, seasonality_prior_scale, <metric> (NaN when not eligible),
              selected -- one row per (group, grid point), plus a row with the model.* pair for a group that fell back
"""
from __future__ import annotations

import itertools
import logging
import math
import os
import time

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from .. import _lib as L
from .. import batched
from .. import dist as pdist
from ..pack import pack_groups_cuda
from .prophet_backtest import backtest_spec_from_config
from .prophet_modeler import (MODEL_OUTPUT_SCHEMA, ProphetModeler, get_context, models_table, options_from_config,
                              regressor_names, table_keys, who)

# fbprophet's documentation: "Hyperparameter tuning"
DEFAULT_CHANGEPOINT_PRIOR_SCALES = (0.001, 0.01, 0.1, 0.5)
DEFAULT_SEASONALITY_PRIOR_SCALES = (0.01, 0.1, 1.0, 10.0)


def _scales(t: dict, key: str, default) -> list:
    v = t.get(key, default)
    if not isinstance(v, (list, tuple)) or len(v) == 0:
        raise ValueError(f"tune.{key} must be a non-empty list of numbers (got {v!r})")
    out = []
    for x in v:
        if isinstance(x, bool) or not isinstance(x, (int, float)):
            raise ValueError(f"tune.{key} must be a non-empty list of numbers (got {v!r})")
        if not (math.isfinite(float(x)) and float(x) > 0.0):
            raise ValueError(f"tune.{key} values must be finite and > 0 (got {x!r})")
        out.append(float(x))
    return out


def tune_spec_from_config(config) -> dict:
    """The ``tune`` section checked: the grid (list of (changepoint_prior_scale, seasonality_prior_scale) pairs in
    itertools.product order) and the metric."""
    t = dict(config.get("tune", {}) or {})
    cp = _scales(t, "changepoint_prior_scale", DEFAULT_CHANGEPOINT_PRIOR_SCALES)
    sp = _scales(t, "seasonality_prior_scale", DEFAULT_SEASONALITY_PRIOR_SCALES)
    metric = t.get("metric", "rmse")
    if metric == "coverage":
        raise ValueError("tune.metric 'coverage' needs prediction intervals, which tuning does not compute; "
                         f"use one of {', '.join(batched.TUNE_METRICS)}")
    if metric not in batched.TUNE_METRICS:
        raise ValueError(f"tune.metric must be one of {', '.join(batched.TUNE_METRICS)} (got {metric!r})")
    return {"grid": list(itertools.product(cp, sp)), "metric": metric}


def tuning_table(series_id, dim_id, res: batched.TuneResult, metric: str, default_pair) -> pa.Table:
    """One row per (group, grid point) -- the metric NaN where the point was not eligible -- and, for a group with no
    eligible point, one more row with ``default_pair`` (the model.* scales) selected."""
    n, g = res.scores.shape
    s = np.repeat(np.arange(n), g)
    gi = np.tile(np.arange(g), n)
    cp, sp = res.grid[gi, 0], res.grid[gi, 1]
    score = np.where(res.eligible, res.scores, np.nan).reshape(-1)
    sel = (res.chosen[s] == gi)
    fb = np.flatnonzero(res.chosen < 0)
    # fallback rows go right after their group's grid rows
    pos = np.concatenate((np.arange(n * g), (fb + 1) * g - 0.5))
    order = np.argsort(pos, kind="stable")
    s = np.concatenate((s, fb))[order]
    cols = {"series_id": pa.array(np.asarray(series_id)[s], pa.int32()),
            "dim_id": pa.array(np.asarray(dim_id)[s], pa.int32()),
            "changepoint_prior_scale": pa.array(np.concatenate((cp, np.full(fb.size, default_pair[0])))[order], pa.float64()),
            "seasonality_prior_scale": pa.array(np.concatenate((sp, np.full(fb.size, default_pair[1])))[order], pa.float64()),
            metric: pa.array(np.concatenate((score, np.full(fb.size, np.nan)))[order], pa.float64()),
            "selected": pa.array(np.concatenate((sel, np.ones(fb.size, bool)))[order], pa.bool_())}
    return pa.table(cols)


class ProphetTuner:
    """Tune every group's prior scales and fit its final model (one batched GPU job; see the module docstring)."""

    def __init__(self, config, logger=None):
        self.logger = logger or logging.getLogger(self.__class__.__name__)
        self.config = config
        self.rank_local_input = False

    def read_input_dataframe(self, spark=None):
        reader = ProphetModeler(self.config)
        frame = reader.read_input_dataframe(spark)
        self.rank_local_input = getattr(reader, "rank_local_input", False)
        return frame

    def tune(self, table: pa.Table):
        """(models table, tuning table) of the groups in ``table`` (columns series_id, dim_id, ds, y)."""
        t0 = time.time()
        spec = backtest_spec_from_config(self.config)
        ts = tune_spec_from_config(self.config)
        floor = self.config["model"]["floor"]
        cap_multiplier = float(self.config["model"]["cap_multiplier"])
        opts = options_from_config(self.config)
        if regressor_names(self.config):
            raise ValueError("model.regressors: the tuner fits every grid point with per-series prior scales, which a "
                             "model with extra regressors does not take; fit it with the modeler")
        if batched.is_table(opts):
            raise ValueError(f"{' / '.join(table_keys(self.config))}: the tuner fits every grid point with per-series "
                             "prior scales, which a model with a seasonality table does not take; tune the default "
                             "seasonalities, or fit the table with the modeler")
        default_pair = (opts.changepoint_prior_scale, opts.seasonality_prior_scale)
        metric = ts["metric"]
        ctx = get_context()
        import torch
        torch.cuda.set_device(ctx.device)
        pk = pack_groups_cuda(table, device=f"cuda:{ctx.device}")
        rank, ws, _ = pdist.world()
        if ws > 1 and not self.rank_local_input:
            lo, hi = pdist.shard_bounds(pk.offsets, ws)[rank]
            pk = pk.take(lo, hi)
        if pk.n == 0:
            empty = pa.schema([("series_id", pa.int32()), ("dim_id", pa.int32()), ("changepoint_prior_scale", pa.float64()),
                               ("seasonality_prior_scale", pa.float64()), (metric, pa.float64()), ("selected", pa.bool_())])
            return MODEL_OUTPUT_SCHEMA.empty_table(), empty.empty_table()
        ds, y = pk.ds.contiguous(), pk.y.contiguous()
        short = np.diff(pk.offsets) < 2
        if np.any(short):
            raise ValueError("Dataframe has less than 2 non-NaN rows." + who(pk.series_id, pk.dim_id, short))
        plan = batched.cv_plan_device(ctx, opts, ds, pk.offsets, spec["horizon"], spec["period"], spec["initial"])
        bad = batched.cv_plan_errors(plan)
        if bad is not None:
            raise ValueError(bad[0] + who(pk.series_id, pk.dim_id, bad[1]))
        n_grid = len(ts["grid"])
        print(f"Tuning {pk.n} series over {n_grid} grid points at {plan.n_pairs} cutoffs")
        res = batched.tune_device(ctx, opts, ds, y, pk.offsets, float(floor), cap_multiplier, spec["horizon"],
                                  spec["period"], spec["initial"], ts["grid"], metric=metric, plan=plan)
        for code, msg in ((L.ST_CAP_LE_FLOOR, "cap must be greater than floor (which defaults to 0)."),
                          (L.ST_BAD_INPUT, "Found non-finite y or a zero time span in a series.")):
            hit = np.zeros(pk.n, bool)
            hit[res.cv.pair_series[res.cv.pair_status == code] // n_grid] = True
            if hit.any():
                raise ValueError(msg + who(pk.series_id, pk.dim_id, hit))
        models = models_table(res.fitted.to_host(), pk.series_id, pk.dim_id, pk.last_ds, opts, floor)
        tuning = tuning_table(pk.series_id, pk.dim_id, res, metric, default_pair)
        print(f"Tuning: {int((res.chosen < 0).sum())} series kept the model.* prior scales; {models.num_rows} models in "
              f"{time.time() - t0:.1f} s")
        return models, tuning

    def persist(self, models: pa.Table, tuning: pa.Table) -> None:
        """Parquet part file per rank under io.models and io.tuning."""
        io = self.config["io"]
        rank = pdist.world()[0]
        for key, tbl in (("models", models), ("tuning", tuning)):
            if not io.get(key):
                continue
            pdist.prepare_output_dir(io[key])
            pq.write_table(tbl, os.path.join(io[key], f"part-{rank:05d}.parquet"))

    @staticmethod
    def run(spark_session, config):
        pdist.init_process_group()
        job = ProphetTuner(config)
        frame = job.read_input_dataframe(spark_session)
        models, tuning = job.tune(frame.table)
        job.persist(models, tuning)
        return models, tuning
