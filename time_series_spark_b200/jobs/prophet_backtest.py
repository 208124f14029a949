"""Backtest job: fbprophet.diagnostics.cross_validation + performance_metrics for every (series_id, dim_id) group.

Reads the modeler's input (``io.input``, same header-less hive-partitioned CSV) and fits each group at every cutoff of
its history with the modeler's options (``model.*``), then predicts the held-out rows after each cutoff and reduces
the errors to metrics by forecast horizon.  All of it on the GPU: the cutoff plan, the gathered truncated histories,
the fits, the prediction and the metrics (time_series_spark_b200/csrc/cv_kernel.cuh; semantics in DESIGN §9).
A seasonality table (``model.seasonalities`` or an int built-in order, DESIGN §18) is backtested as fbprophet's
prophet_copy does it: every cutoff fit takes the full history's active seasonalities and nothing else, with every
``backtest.*`` option below.  With ``model.regressors`` (DESIGN §20) the input's regressor columns are read as the
modeler reads them and every cutoff is fitted as fbprophet 0.5's cross_validation does it: on the full history's
standardised values, keeping the full model's (mu, std) where the cutoff's history is not standardised;
``backtest.aggregate`` (and so ``backtest.aggregate_quantiles``) and ``backtest.quantiles`` are refused with it.

Keys (``backtest.*``):
  horizon            pandas Timedelta string, required ("1 days")
  period             default horizon / 2
  initial            default 3 * horizon
  rolling_window     fraction of a series' held-out rows each metric averages over, in [0, 1]; default 0.1
  intervals          false (default): no yhat_lower / yhat_upper, no coverage column
  uncertainty_samples, interval_width, seed   1000, 0.8, 0 (used with intervals only)
  aggregate          a fixed-width duration W dividing the horizon ('1h', '8h', '1D'): also the held-out totals per
                     window (c + j W, c + (j + 1) W] after each cutoff c and their metrics by horizon (j + 1) W, with
                     intervals the coverage of the totals' joint-draw intervals (DESIGN §14); needs io.window_metrics
  quantiles          a list of 1 to 32 levels in [0, 1]: the held-out quantiles of each level from uncertainty_samples
                     draws (with or without intervals) and their pinball loss and share of y at or below them by
                     horizon (DESIGN §15); needs io.quantile_metrics, not with aggregate
  aggregate_quantiles  with aggregate and intervals, a list of 1 to 32 levels in [0, 1]: the quantiles of each
                     window's total from the draws behind its interval, and their pinball loss and share of the held-out
                     total at or below them by horizon (j + 1) W (DESIGN §21); needs io.window_quantile_metrics
Outputs (parquet, one part file per rank):
  io.metrics          series_id, dim_id, horizon duration[ns], mse, rmse, mae, mape[, coverage]
  io.cv_rows          (optional) series_id, dim_id, ds, cutoff, y, yhat[, yhat_lower, yhat_upper][, yhat_q<level>...]
  io.quantile_metrics (with quantiles) series_id, dim_id, horizon duration[ns], quantile, pinball_loss, share_below: one
                      row per (horizon, level)
  io.window_metrics   (with aggregate) series_id, dim_id, horizon duration[ns], mse, rmse, mae, mape[, coverage]
  io.window_rows      (optional, with aggregate) series_id, dim_id, cutoff, horizon, window_points, y, yhat[,
                      yhat_lower, yhat_upper][, yhat_q<level>... with aggregate_quantiles]
  io.window_quantile_metrics  (with aggregate_quantiles) io.quantile_metrics' columns over the window rows
"""
from __future__ import annotations

import logging
import os
import time

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from .. import _lib as L
from .. import batched
from .. import dist as pdist
from ..pack import pack_groups_cuda
from .prophet_modeler import ProphetModeler, get_context, options_from_config, regressor_names
from .prophet_scorer import quantile_column, quantile_levels


def _duration_ns(key: str, value) -> int:
    import pandas as pd
    try:
        ns = int(pd.Timedelta(value).value)
    except (ValueError, TypeError) as e:
        raise ValueError(f"backtest.{key} must be a duration such as '1 days' (got {value!r})") from e
    if ns <= 0:
        raise ValueError(f"backtest.{key} must be positive (got {value!r})")
    return ns


def backtest_spec_from_config(config) -> dict:
    """The ``backtest`` section checked and converted: durations in int64 ns, the metric window, interval options."""
    b = dict(config.get("backtest", {}) or {})
    if "horizon" not in b:
        raise ValueError("backtest.horizon is required")
    horizon = _duration_ns("horizon", b["horizon"])
    period = _duration_ns("period", b["period"]) if b.get("period") is not None else horizon // 2
    initial = _duration_ns("initial", b["initial"]) if b.get("initial") is not None else 3 * horizon
    if period <= 0:
        raise ValueError(f"backtest.period must be positive (horizon / 2 of {b['horizon']!r} is 0)")
    try:
        rw = float(b.get("rolling_window", 0.1))
    except (TypeError, ValueError):
        rw = float("nan")
    if not (0.0 <= rw <= 1.0):
        raise ValueError(f"backtest.rolling_window must be in [0, 1] (got {b.get('rolling_window')!r})")
    intervals = bool(b.get("intervals", False))
    spec = {"horizon": horizon, "period": period, "initial": initial, "rolling_window": rw, "intervals": intervals,
            "uncertainty_samples": 0, "interval_width": 0.8, "seed": int(b.get("seed", 0))}
    levels = quantile_levels(b, "backtest.quantiles")
    if intervals:
        width = float(b.get("interval_width", 0.8))
        if not (0.0 <= width <= 1.0):
            raise ValueError(f"backtest.interval_width must be in [0, 1] (got {b.get('interval_width')!r})")
        spec["interval_width"] = width
    if intervals or levels is not None:
        ns = int(b.get("uncertainty_samples", 1000))
        if not (2 <= ns <= 1024):
            raise ValueError(f"backtest.uncertainty_samples must be in [2, 1024] (got {b.get('uncertainty_samples')!r})")
        spec["uncertainty_samples"] = ns
    spec["aggregate"] = _aggregate_width(config, b, horizon)
    if levels is not None:
        if spec["aggregate"] is not None:
            raise ValueError("backtest.quantiles cannot be combined with backtest.aggregate")
        if not (config.get("io", {}) or {}).get("quantile_metrics"):
            raise ValueError("backtest.quantiles needs io.quantile_metrics, the directory the quantile metrics are written to")
    spec["quantiles"] = levels
    wlevels = quantile_levels({"quantiles": b.get("aggregate_quantiles")}, "backtest.aggregate_quantiles")
    if wlevels is not None:
        if spec["aggregate"] is None:
            raise ValueError("backtest.aggregate_quantiles needs backtest.aggregate: its levels are quantiles of the "
                             "window totals")
        if not intervals:
            raise ValueError("backtest.aggregate_quantiles needs backtest.intervals: the levels come from the draws "
                             "behind the window totals' intervals")
        if not (config.get("io", {}) or {}).get("window_quantile_metrics"):
            raise ValueError("backtest.aggregate_quantiles needs io.window_quantile_metrics, the directory the window "
                             "quantile metrics are written to")
        spec["aggregate_quantiles"] = wlevels
    return spec


def _aggregate_width(config, b: dict, horizon: int):
    """``backtest.aggregate`` in ns (None without the key): a fixed-width duration that divides the horizon, so that
    every window (c + j W, c + (j + 1) W] lies inside the held-out span (c, c + horizon]."""
    import pandas as pd
    from .prophet_scorer import _to_offset
    spec = b.get("aggregate")
    if spec is None:
        return None
    try:
        off = _to_offset(spec)
    except Exception:
        off = None                  # not a frequency alias: a Timedelta string such as '2 days', as backtest.horizon
    try:
        if off is None:
            width = int(pd.Timedelta(spec).value)
        else:
            width = int(7 * 86400 * 10**9 * off.n if isinstance(off, pd.offsets.Week) and off.weekday is None else off.nanos)
    except Exception:
        raise ValueError(f"backtest.aggregate must be a fixed-width duration such as '1h', '8h' or '1D' (got {spec!r}; "
                         "calendar offsets such as 'M' have no fixed width)") from None
    if width <= 0:
        raise ValueError(f"backtest.aggregate must be a positive duration (got {spec!r})")
    if horizon % width != 0:
        raise ValueError(f"backtest.aggregate ({spec!r}) must divide backtest.horizon ({b['horizon']!r}), so that every "
                         "window lies inside the held-out span")
    if not (config.get("io", {}) or {}).get("window_metrics"):
        raise ValueError("backtest.aggregate needs io.window_metrics, the directory the window metrics are written to")
    return width


def _who(series_id, dim_id, mask) -> str:
    i = int(np.flatnonzero(mask)[0])
    return (f" (first offender: series_id {int(series_id[i])}, dim_id {int(dim_id[i])}; "
            f"{int(np.count_nonzero(mask))} group(s) in all)")


def _failed_series(series_id, dim_id, res: batched.CvResult, announce: bool = True):
    """Per series: some cutoff fit failed (status < 0), where fbprophet's cross_validation would raise; a printed line
    names each such series and its first failed cutoff."""
    n = len(series_id)
    failed = np.zeros(n, bool)
    for p in np.flatnonzero(res.pair_status < 0):
        s = int(res.pair_series[p])
        if not failed[s] and announce:
            cut = np.datetime64(int(res.pair_cutoff[p]), "ns")
            print(f"Runtime error (solver status {int(res.pair_status[p])}) for series_id: {int(series_id[s])}, "
                  f"dim_id: {int(dim_id[s])}, cutoff: {cut}")
        failed[s] = True
    return failed


def _metrics_table(series_id, dim_id, m: dict, failed) -> pa.Table:
    keep = ~failed[m["series"]]
    ms = m["series"][keep]
    cols = {"series_id": pa.array(np.asarray(series_id)[ms], pa.int32()),
            "dim_id": pa.array(np.asarray(dim_id)[ms], pa.int32()),
            "horizon": pa.array(m["horizon"][keep], pa.duration("ns"))}
    for k in ("mse", "rmse", "mae", "mape"):
        cols[k] = pa.array(m[k][keep], pa.float64())
    if m["coverage"] is not None:
        cols["coverage"] = pa.array(m["coverage"][keep], pa.float64())
    return pa.table(cols)


def assemble_window_outputs(series_id, dim_id, res: batched.CvResult, with_rows: bool = True, levels=None):
    """Window metrics (and window row) tables of a CvResult made with aggregate_ns; the same failed-fit rule as
    assemble_outputs (which prints the lines).  ``levels`` (the CvResult made with them as window_quantiles): the rows
    get a yhat_q<level> column per level."""
    failed = _failed_series(series_id, dim_id, res, announce=False)
    w = res.windows
    metrics = _metrics_table(series_id, dim_id, w.metrics, failed)
    rows = None
    if with_rows:
        keep = ~failed[w.series]
        rs = w.series[keep]
        rc = {"series_id": pa.array(np.asarray(series_id)[rs], pa.int32()),
              "dim_id": pa.array(np.asarray(dim_id)[rs], pa.int32()),
              "cutoff": pa.array(w.cutoff[keep], pa.timestamp("ns")),
              "horizon": pa.array(w.horizon[keep], pa.duration("ns")),
              "window_points": pa.array(w.points[keep], pa.int32()),
              "y": pa.array(w.y[keep], pa.float64()),
              "yhat": pa.array(w.yhat[keep], pa.float64())}
        if w.yhat_lower is not None:
            rc["yhat_lower"] = pa.array(w.yhat_lower[keep], pa.float64())
            rc["yhat_upper"] = pa.array(w.yhat_upper[keep], pa.float64())
        for q, lv in enumerate(levels or ()):
            rc[quantile_column(lv)] = pa.array(w.yhat_q[q][keep], pa.float64())
        rows = pa.table(rc)
    return metrics, rows


QUANTILE_METRICS_SCHEMA = pa.schema([("series_id", pa.int32()), ("dim_id", pa.int32()), ("horizon", pa.duration("ns")),
                                     ("quantile", pa.float64()), ("pinball_loss", pa.float64()),
                                     ("share_below", pa.float64())])


def quantile_metrics_table(series_id, dim_id, res: batched.CvResult) -> pa.Table:
    """io.quantile_metrics of a CvResult made with quantiles: one row per (series, horizon, level); the same failed-fit
    rule as assemble_outputs (which prints the lines)."""
    return _quantile_metrics_table(series_id, dim_id, res.quantile_metrics,
                                   _failed_series(series_id, dim_id, res, announce=False))


def window_quantile_metrics_table(series_id, dim_id, res: batched.CvResult) -> pa.Table:
    """io.window_quantile_metrics of a CvResult made with window_quantiles: quantile_metrics_table's rows over the window
    rows, horizon (j + 1) W."""
    return _quantile_metrics_table(series_id, dim_id, res.windows.quantile_metrics,
                                   _failed_series(series_id, dim_id, res, announce=False))


def _quantile_metrics_table(series_id, dim_id, m: dict, failed) -> pa.Table:
    keep = ~failed[m["series"]]
    ms = m["series"][keep]
    return pa.table({"series_id": pa.array(np.asarray(series_id)[ms], pa.int32()),
                     "dim_id": pa.array(np.asarray(dim_id)[ms], pa.int32()),
                     "horizon": pa.array(m["horizon"][keep], pa.duration("ns")),
                     "quantile": pa.array(m["level"][keep], pa.float64()),
                     "pinball_loss": pa.array(m["pinball"][keep], pa.float64()),
                     "share_below": pa.array(m["share_below"][keep], pa.float64())}, schema=QUANTILE_METRICS_SCHEMA)


def assemble_outputs(series_id, dim_id, res: batched.CvResult, y_dtype, with_rows: bool = True, levels=None):
    """Metrics (and row) tables of a CvResult.  A series with a failed cutoff fit (status < 0) -- where fbprophet's
    cross_validation would raise -- gets no row in either table, and a printed line names it and the cutoff.  ``levels``
    (the CvResult made with them): the rows get a yhat_q<level> column per level."""
    failed = _failed_series(series_id, dim_id, res)
    metrics = _metrics_table(series_id, dim_id, res.metrics, failed)
    rows = None
    if with_rows:
        keep = ~failed[res.row_series]
        rs = res.row_series[keep]
        rc = {"series_id": pa.array(np.asarray(series_id)[rs], pa.int32()),
              "dim_id": pa.array(np.asarray(dim_id)[rs], pa.int32()),
              "ds": pa.array(res.ds[keep], pa.timestamp("ns")),
              "cutoff": pa.array(res.cutoff[keep], pa.timestamp("ns")),
              "y": pa.array(res.y[keep].astype(y_dtype)),
              "yhat": pa.array(res.yhat[keep], pa.float64())}
        if res.yhat_lower is not None:
            rc["yhat_lower"] = pa.array(res.yhat_lower[keep], pa.float64())
            rc["yhat_upper"] = pa.array(res.yhat_upper[keep], pa.float64())
        for q, lv in enumerate(levels or ()):
            rc[quantile_column(lv)] = pa.array(res.yhat_q[q][keep], pa.float64())
        rows = pa.table(rc)
    return metrics, rows


class ProphetBacktester:
    """Backtest every group of the modeler's input (one batched GPU job; see the module docstring)."""

    def __init__(self, config, logger=None):
        self.logger = logger or logging.getLogger(self.__class__.__name__)
        self.config = config
        self.rank_local_input = False
        self.window_outputs = None     # (window metrics, window rows or None) with backtest.aggregate
        self.quantile_metrics = None   # with backtest.quantiles
        self.window_quantile_metrics = None   # with backtest.aggregate_quantiles

    def read_input_dataframe(self, spark=None):
        reader = ProphetModeler(self.config)
        frame = reader.read_input_dataframe(spark)
        self.rank_local_input = getattr(reader, "rank_local_input", False)
        return frame

    def backtest(self, table: pa.Table):
        """(metrics table, row table or None) of the groups in ``table`` (columns series_id, dim_id, ds, y).  With
        backtest.aggregate, ``self.window_outputs`` gets the (window metrics, window rows or None) tables."""
        t0 = time.time()
        spec = backtest_spec_from_config(self.config)
        reg_names = regressor_names(self.config)
        if reg_names:
            for key in ("aggregate", "quantiles"):
                if spec[key] is not None:
                    raise ValueError(f"backtest.{key} is not available with model.regressors: the window totals and "
                                     "quantiles of a model with extra regressors are not implemented")
        floor = float(self.config["model"]["floor"])
        cap_multiplier = float(self.config["model"]["cap_multiplier"])
        opts = options_from_config(self.config)
        opts.uncertainty_samples = spec["uncertainty_samples"]
        opts.interval_width = spec["interval_width"]
        ctx = get_context()
        import torch
        torch.cuda.set_device(ctx.device)
        pk = pack_groups_cuda(table, device=f"cuda:{ctx.device}", reg_cols=reg_names)
        rank, ws, _ = pdist.world()
        if ws > 1 and not self.rank_local_input:
            lo, hi = pdist.shard_bounds(pk.offsets, ws)[rank]
            pk = pk.take(lo, hi)
        io = self.config.get("io", {}) or {}
        with_rows = bool(io.get("cv_rows"))
        W = spec["aggregate"]
        levels = spec["quantiles"]
        wlevels = spec.get("aggregate_quantiles")
        if pk.n == 0:
            empty_metrics = lambda: dict({k: np.zeros(0, np.int64 if k in ("series", "horizon") else np.float64)  # noqa: E731
                                          for k in ("series", "horizon", "mse", "rmse", "mae", "mape")},
                                         coverage=np.zeros(0) if spec["intervals"] else None)
            res = batched.CvResult(*(np.zeros(0, np.int64),) * 4, *(np.zeros(0, np.int64),) * 3, *(np.zeros(0),) * 2,
                                   None, None, metrics=empty_metrics())
            if spec["intervals"]:
                res.yhat_lower, res.yhat_upper = np.zeros(0), np.zeros(0)
            if W is not None:
                iv = np.zeros(0) if spec["intervals"] else None
                res.windows = batched.CvWindows(W, *(np.zeros(0, np.int64),) * 3, np.zeros(0, np.int32), np.zeros(0),
                                                np.zeros(0), iv, iv, empty_metrics())
                if wlevels is not None:
                    res.windows.yhat_q = np.zeros((len(wlevels), 0))
                    self.window_quantile_metrics = QUANTILE_METRICS_SCHEMA.empty_table()
                self.window_outputs = assemble_window_outputs(pk.series_id, pk.dim_id, res, bool(io.get("window_rows")),
                                                              wlevels)
            if levels is not None:
                res.yhat_q = np.zeros((len(levels), 0))
                self.quantile_metrics = QUANTILE_METRICS_SCHEMA.empty_table()
            return assemble_outputs(pk.series_id, pk.dim_id, res, np.dtype(str(pk.y.dtype).replace("torch.", "")), with_rows,
                                    levels)
        ds, y = pk.ds.contiguous(), pk.y.contiguous()
        short = np.diff(pk.offsets) < 2
        if np.any(short):
            raise ValueError("Dataframe has less than 2 non-NaN rows." + _who(pk.series_id, pk.dim_id, short))
        if reg_names:
            # fbprophet's setup_dataframe on the full history: "Found NaN in column <name>", as the modeler says it
            scale, nan = batched.regressor_scales_device(ctx, opts, pk.regressors, pk.offsets)
            nan = nan.cpu().numpy()
            if nan.any():
                r = int(np.flatnonzero(np.isnan(scale[int(np.flatnonzero(nan)[0]), :, 0].cpu().numpy()))[0])
                raise ValueError(f"Found NaN in column {reg_names[r]}" + _who(pk.series_id, pk.dim_id, nan))
        plan = batched.cv_plan_device(ctx, batched.plan_options(opts), ds, pk.offsets, spec["horizon"], spec["period"],
                                      spec["initial"])
        bad = batched.cv_plan_errors(plan)
        if bad is not None:
            raise ValueError(bad[0] + _who(pk.series_id, pk.dim_id, bad[1]))
        # the full history's float64 cap, as the modeler computes it: max(y) * cap_multiplier
        lens = torch.from_numpy(np.diff(pk.offsets)).to(ds.device)
        cap = torch.segment_reduce(y.to(torch.float64), "max", lengths=lens) * cap_multiplier
        print(f"Backtesting {pk.n} series at {plan.n_pairs} cutoffs")
        res = batched.cross_validation_device(ctx, opts, ds, y, pk.offsets, floor, cap, spec["horizon"], spec["period"],
                                              spec["initial"], intervals=spec["intervals"], seed=spec["seed"],
                                              rolling_window=spec["rolling_window"], plan=plan, aggregate_ns=W,
                                              quantiles=levels, regressors=pk.regressors, window_quantiles=wlevels)
        for code, msg in ((L.ST_CAP_LE_FLOOR, "cap must be greater than floor (which defaults to 0)."),
                          (L.ST_BAD_INPUT, "Found non-finite y or a zero time span in a series.")):
            hit = np.zeros(pk.n, bool)
            hit[res.pair_series[res.pair_status == code]] = True
            if hit.any():
                raise ValueError(msg + _who(pk.series_id, pk.dim_id, hit))
        out = assemble_outputs(pk.series_id, pk.dim_id, res, np.dtype(str(y.dtype).replace("torch.", "")), with_rows,
                               levels)
        if levels is not None:
            self.quantile_metrics = quantile_metrics_table(pk.series_id, pk.dim_id, res)
        if W is not None:
            self.window_outputs = assemble_window_outputs(pk.series_id, pk.dim_id, res, bool(io.get("window_rows")),
                                                          wlevels)
        if wlevels is not None:
            self.window_quantile_metrics = window_quantile_metrics_table(pk.series_id, pk.dim_id, res)
        print(f"Backtest: {out[0].num_rows} metrics rows in {time.time() - t0:.1f} s")
        return out

    def persist(self, metrics: pa.Table, rows) -> None:
        """Parquet part file per rank under io.metrics (and io.cv_rows, with backtest.aggregate io.window_metrics and
        io.window_rows, with backtest.quantiles io.quantile_metrics, with backtest.aggregate_quantiles
        io.window_quantile_metrics)."""
        io = self.config["io"]
        rank = pdist.world()[0]
        wm, wr = self.window_outputs or (None, None)
        for key, tbl in (("metrics", metrics), ("cv_rows", rows), ("window_metrics", wm), ("window_rows", wr),
                         ("quantile_metrics", self.quantile_metrics),
                         ("window_quantile_metrics", self.window_quantile_metrics)):
            if tbl is None or not io.get(key):
                continue
            pdist.prepare_output_dir(io[key])
            pq.write_table(tbl, os.path.join(io[key], f"part-{rank:05d}.parquet"))

    @staticmethod
    def run(spark_session, config):
        pdist.init_process_group()
        job = ProphetBacktester(config)
        frame = job.read_input_dataframe(spark_session)
        metrics, rows = job.backtest(frame.table)
        job.persist(metrics, rows)
        return metrics, rows
