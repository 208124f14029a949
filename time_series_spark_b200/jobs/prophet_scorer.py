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
``forecast.interval_width`` (0.8), ``forecast.seed``.
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


class _ForecastTimeSeriesOp:
    """Batched GROUPED_MAP operator over the models table."""

    def __init__(self, config):
        self.config = config

    def apply_batched(self, table: pa.Table, keys) -> pa.Table:
        if list(keys) != ["series_id", "dim_id"]:
            raise ValueError("forecast_time_series groups by ('series_id', 'dim_id')")
        fc = self.config["forecast"]
        want_intervals = bool(fc.get("intervals", False))
        rank, ws, _ = pdist.world()
        if ws > 1 and table.num_rows:      # shard the model rows across ranks (equal horizon => equal work)
            lo, hi = pdist.shard_bounds(np.arange(table.num_rows + 1, dtype=np.int64), ws)[rank]
            table = table.slice(lo, hi - lo)
        # every rank must hand back the same columns (an empty shard too): the optional gather issues one
        # collective per column
        empty_schema = FORECAST_SCHEMA
        if want_intervals:
            empty_schema = empty_schema.append(pa.field("yhat_lower", pa.float64())).append(pa.field("yhat_upper", pa.float64()))
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
        opts = batched.make_options(growth="logistic" if info["logistic"] else "linear",
                                    seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
                                    n_changepoints=info["n_changepoints"],
                                    interval_width=fc.get("interval_width", 0.8),
                                    uncertainty_samples=fc.get("uncertainty_samples", 1000) if want_intervals else 0)
        opts.yearly, opts.weekly, opts.daily = info["yearly"], info["weekly"], info["daily"]
        # reference :46-47: floor / cap are read back from the FLOAT32 columns of the models table
        floor = table["floor"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.float64)
        cap = table["cap"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.float64)
        periods = int(fc["periods"])
        future = frequency_to_future(last_ds, periods, fc["frequency"])
        ctx = get_context()
        res = batched.predict_batch_host(ctx, opts, fitted, future, floor, cap, seed=int(fc.get("seed", 0)),
                                         intervals=want_intervals)
        sid = table["series_id"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.int32)
        did = table["dim_id"].combine_chunks().to_numpy(zero_copy_only=False).astype(np.int32)
        ok = fitted.meta_i32[:, 4] >= 0
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
        out = pa.table(cols)
        if not ok.all():
            out = out.filter(pa.array(np.repeat(ok, periods)))
        return out

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
        for extra in ("yhat_lower", "yhat_upper"):
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

    @staticmethod
    def score(spark_session, config):
        pdist.init_process_group()          # no-op unless launched by torchrun with WORLD_SIZE > 1
        scorer = ProphetScorer(config)
        model_df = scorer.read_model_dataframe(spark_session)
        forecast_df = model_df.groupby("series_id", "dim_id").apply(forecast_time_series(scorer.config))
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
            arrays = [pa.array(a, pa.int64()).cast(pa.timestamp("ns")) if n == "ds" else pa.array(a)
                      for n, a in zip(t.column_names, got)]
            forecast_df = Frame(pa.table(dict(zip(t.column_names, arrays))).cast(t.schema))
        converted_df = scorer.convert_forecasts(forecast_df)
        scorer.write_forecasts(converted_df)
