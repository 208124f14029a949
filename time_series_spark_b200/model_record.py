"""Wire format of the ``model`` binary column of the models table.

The reference stores ``pickle.dumps(Prophet object)`` there (src/jobs/prophet_modeler.py:72-73,
read back by src/jobs/prophet_scorer.py:48): tens of KB per series carrying the whole
history frame.  The batched scorer needs only the fitted parameters and scaling metadata, so
the record is a fixed-layout little-endian struct (about 0.7 KB):

    magic 'PB2M' | u16 version | u16 flags (1 logistic, 2 multiplicative) | i32 smax | i32 kmax
    | i32[4] option switches (yearly, weekly, daily as PB200_SEAS_AUTO/0/1, n_changepoints)
    | i32[8] meta_i32 (T, S, n_changepoints_real, seasonality mask, status, iters, n_evals, i1)
    | i64[2] meta_i64 (start_ns, t_scale_ns) | i64 last_ds_ns (history_dates.max())
    | f64[4] meta_f64 (y_scale, floor, cap, neg_log_posterior)
    | f64[pstride] params (k, m, sigma_obs, delta[smax], beta[kmax]) | f64[smax] t_change

Version 2 is the record of a model with a seasonality table (DESIGN §18): the version-1 fields (meta_i32[3] then holds
the table mask, bit j = entry j of the normalised table active), followed by the table as it was given:

    | i32[3] built-in orders (yearly, weekly, daily; 0 = default) | i32 entry count
    | 8 x (name[16] NUL-padded | f64 period (days) | f64 prior_scale (0 = seasonality_prior_scale) | i32 fourier_order)

Options without a table, and a table that restates the default model, write version 1.  Every record of a table
has one version, and the version-2 records of a table one seasonality table.

Version 4 is the record of a model with extra regressors (DESIGN §20; version 3 was never written): the version-1
fields, each series' standardisation, then the bytes every record of the fit shares -- the table tail of version 2
(always present; it may restate the defaults) and the regressors as they were given:

    | f64[16][2] reg_scale (mu, std of regressor r; unused slots 0)
    | i32[3] built-in orders | i32 entry count | 8 x seasonality entry          (as version 2)
    | f64 holidays_prior_scale | i32 regressor count
    | 16 x (name[16] NUL-padded | f64 prior_scale (0 = holidays_prior_scale) | i32 standardize (-1 auto, 0, 1))

Encoding / decoding is vectorised over the whole batch (one numpy structured array),
never a per-row Python loop.
"""
from __future__ import annotations

import numpy as np
import pyarrow as pa

from . import _lib as L
from . import batched
from .batched import FittedBatch

MAGIC = b"PB2M"
VERSION = 1
VERSION_TABLE = 2
VERSION_REGRESSORS = 4
FLAG_LOGISTIC, FLAG_MULT = 1, 2
_BUILTIN_KEYS = ("yearly_seasonality", "weekly_seasonality", "daily_seasonality")
ENTRY_DTYPE = np.dtype([("name", "S16"), ("period", "<f8"), ("prior_scale", "<f8"), ("fourier_order", "<i4")])
REGRESSOR_DTYPE = np.dtype([("name", "S16"), ("prior_scale", "<f8"), ("standardize", "<i4")])


def record_dtype(smax: int, kmax: int, version: int = VERSION) -> np.dtype:
    pstride = 3 + smax + kmax
    fields = [("magic", "S4"), ("version", "<u2"), ("flags", "<u2"), ("smax", "<i4"), ("kmax", "<i4"),
              ("switches", "<i4", (4,)), ("meta_i32", "<i4", (8,)), ("meta_i64", "<i8", (2,)), ("last_ds", "<i8"),
              ("meta_f64", "<f8", (4,)), ("params", "<f8", (pstride,)), ("tchange", "<f8", (smax,))]
    table = [("orders", "<i4", (3,)), ("n_entries", "<i4"), ("entries", ENTRY_DTYPE, (L.MAX_SEASONALITIES,))]
    if version == VERSION_TABLE:
        fields += table
    elif version == VERSION_REGRESSORS:
        fields = fields + [("reg_scale", "<f8", (L.MAX_REGRESSORS, 2))] + table + [
            ("holidays_prior_scale", "<f8"), ("n_regressors", "<i4"), ("regressors", REGRESSOR_DTYPE, (L.MAX_REGRESSORS,))]
    elif version != VERSION:
        raise ValueError(f"unknown model record version {version}")
    return np.dtype(fields)


def _table_spec(opts) -> dict:
    """The seasonality table of pb200_options_v2 as make_table_options' keyword arguments."""
    spec = {}
    for key, sw, order in zip(_BUILTIN_KEYS, (opts.yearly, opts.weekly, opts.daily),
                              (opts.yearly_order, opts.weekly_order, opts.daily_order)):
        if sw == L.SEAS_AUTO:
            if order != 0:
                raise ValueError(f"{key}: an order ({order}) under an AUTO switch (make_table_options forces a "
                                 "built-in on when it is given an order)")
            spec[key] = "auto"
        else:
            spec[key] = (int(order) if order > 0 else True) if sw == 1 else False
    seas = []
    for i in range(opts.n_seasonalities):
        e = opts.seasonalities[i]
        d = {"name": e.name.decode(), "period": float(e.period), "fourier_order": int(e.fourier_order)}
        if e.prior_scale != 0.0:
            d["prior_scale"] = float(e.prior_scale)
        seas.append(d)
    spec["seasonalities"] = seas
    return spec


def _regressor_spec(opts) -> list:
    """The regressors of pb200_options_v3 as make_regressor_options' ``regressors``."""
    out = []
    for i in range(opts.n_regressors):
        e = opts.regressors[i]
        d = {"name": e.name.decode()}
        if e.prior_scale != 0.0:
            d["prior_scale"] = float(e.prior_scale)
        d["standardize"] = "auto" if e.standardize == L.STD_AUTO else bool(e.standardize)
        out.append(d)
    return out


def regressor_options(info: dict, **kw):
    """The options of a decoded version-4 record (``info["table"]``, ``info["regressors"]``,
    ``info["holidays_prior_scale"]``) for make_table_options' other keyword arguments ``kw``: the fit's options."""
    return batched.make_regressor_options(
        regressors=info["regressors"], holidays_prior_scale=info["holidays_prior_scale"],
        growth="logistic" if info["logistic"] else "linear",
        seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
        n_changepoints=info["n_changepoints"], **info["table"], **kw)


def table_options(info: dict, **kw):
    """The options of a decoded table (``info["table"]``) for make_table_options' other keyword arguments ``kw``
    (make_options'): the fit's seasonality table, layout and component names."""
    return batched.make_table_options(
        growth="logistic" if info["logistic"] else "linear",
        seasonality_mode="multiplicative" if info["multiplicative"] else "additive",
        n_changepoints=info["n_changepoints"], **info["table"], **kw)


def encode(fitted: FittedBatch, last_ds_ns: np.ndarray, opts) -> pa.Array:
    """FittedBatch (+ the pb200 Options it was fitted with) -> Arrow binary array, one record per model.  Options the
    record cannot represent -- a decoded record would rebuild another model from them -- raise ValueError."""
    logistic, multiplicative = opts.growth == 1, bool(opts.multiplicative)
    fitted = fitted.to_host()
    n = fitted.n
    table = batched.seasonality_table(opts)
    R = batched.n_regressors(opts)
    version = VERSION if table is None else VERSION_REGRESSORS if R else VERSION_TABLE
    if table is not None:
        try:
            spec = _table_spec(opts)
            kw = dict(growth="logistic" if logistic else "linear",
                      seasonality_mode="multiplicative" if multiplicative else "additive",
                      n_changepoints=opts.n_changepoints, seasonality_prior_scale=opts.seasonality_prior_scale, **spec)
            if R:
                rspec = _regressor_spec(opts)
                rebuilt = batched.make_regressor_options(regressors=rspec,
                                                         holidays_prior_scale=opts.holidays_prior_scale, **kw)
            else:
                rebuilt = batched.make_table_options(**kw)
        except ValueError as e:
            raise ValueError(f"these options have no model record: {e}") from None
        if batched.seasonality_table(rebuilt) != table:
            raise ValueError("these options have no model record: their seasonality table does not rebuild")
        if R:
            if fitted.reg_scale is None:
                raise ValueError("a fit with regressors needs its reg_scale (FittedBatch.reg_scale) in the model record")
            if np.shape(fitted.reg_scale) != (n, R, 2):
                raise ValueError(f"the fitted batch's reg_scale has shape {np.shape(fitted.reg_scale)}, not ({n}, {R}, 2)")
        lay = L.get_layout(opts)
        if (lay.smax, lay.kmax) != (fitted.smax, fitted.kmax):
            raise ValueError(f"the fitted batch's layout (smax {fitted.smax}, kmax {fitted.kmax}) is not the options' "
                             f"(smax {lay.smax}, kmax {lay.kmax})")
    dt = record_dtype(fitted.smax, fitted.kmax, version)
    rec = np.zeros(n, dtype=dt)
    rec["magic"] = MAGIC
    rec["version"] = version
    rec["flags"] = (FLAG_LOGISTIC if logistic else 0) | (FLAG_MULT if multiplicative else 0)
    rec["smax"], rec["kmax"] = fitted.smax, fitted.kmax
    rec["switches"] = np.array([opts.yearly, opts.weekly, opts.daily, opts.n_changepoints], dtype=np.int32)
    rec["meta_i32"], rec["meta_i64"], rec["meta_f64"] = fitted.meta_i32, fitted.meta_i64, fitted.meta_f64
    rec["last_ds"] = np.asarray(last_ds_ns, dtype=np.int64)
    rec["params"], rec["tchange"] = fitted.params, fitted.tchange
    if table is not None:
        rec["orders"] = np.array([opts.yearly_order, opts.weekly_order, opts.daily_order], dtype=np.int32)
        rec["n_entries"] = opts.n_seasonalities
        ent = np.zeros(L.MAX_SEASONALITIES, ENTRY_DTYPE)
        for i in range(opts.n_seasonalities):
            e = opts.seasonalities[i]
            ent[i] = (e.name, e.period, e.prior_scale, e.fourier_order)
        rec["entries"] = ent
    if version == VERSION_REGRESSORS:
        rec["reg_scale"][:, :R, :] = fitted.reg_scale
        rec["holidays_prior_scale"] = opts.holidays_prior_scale
        rec["n_regressors"] = R
        regs = np.zeros(L.MAX_REGRESSORS, REGRESSOR_DTYPE)
        for i in range(R):
            e = opts.regressors[i]
            regs[i] = (e.name, e.prior_scale, e.standardize)
        rec["regressors"] = regs
    size = dt.itemsize
    offsets = pa.py_buffer((np.arange(n + 1, dtype=np.int64) * size).astype(np.int32).tobytes()) \
        if n * size < 2**31 else None
    data = pa.py_buffer(rec.tobytes())
    if offsets is not None:
        return pa.Array.from_buffers(pa.binary(), n, [None, offsets, data])
    off64 = pa.py_buffer((np.arange(n + 1, dtype=np.int64) * size).tobytes())
    return pa.Array.from_buffers(pa.large_binary(), n, [None, off64, data])


_TABLE_TAIL = 16 + ENTRY_DTYPE.itemsize * L.MAX_SEASONALITIES     # orders, n_entries, entries: a v2 record's end
_REG_TAIL = 12 + REGRESSOR_DTYPE.itemsize * L.MAX_REGRESSORS      # holidays_prior_scale, n_regressors, regressors


def _column(col):
    """One Arrow array of the records, refused when empty or holding nulls."""
    if isinstance(col, pa.ChunkedArray):
        col = col.combine_chunks() if col.num_chunks != 1 else col.chunk(0)
    if len(col) == 0:
        raise ValueError("empty model column")
    if col.null_count:
        raise ValueError("model column holds nulls (the reference returns an empty frame for those rows)")
    return col


def _one_class(col):
    """(record offsets, data bytes, version) of a column whose records are one model class: a PB2M first record, every
    record's version known and the same, for version 2 one seasonality table, and for version 4 one seasonality table
    and one set of regressors.  Reads only the records' headers and shared tails, whatever their layouts."""
    n = len(col)
    if col[0].as_py()[:4] != MAGIC:
        raise ValueError("model blob is not a PB2M record (fbprophet pickles cannot be scored on this path)")
    bufs = col.buffers()
    off_dt = np.int64 if pa.types.is_large_binary(col.type) else np.int32
    offs = np.frombuffer(bufs[1], dtype=off_dt)[col.offset:col.offset + n + 1].astype(np.int64)
    if np.any(np.diff(offs) < 16):
        raise ValueError("bad model record header")
    # every record's version, read before the record layout it decides
    raw = np.frombuffer(bufs[2], dtype=np.uint8)
    ver = raw[offs[:-1] + 4].astype(np.int64) | (raw[offs[:-1] + 5].astype(np.int64) << 8)
    known = (ver == VERSION) | (ver == VERSION_TABLE) | (ver == VERSION_REGRESSORS)
    if not known.all():
        raise ValueError(f"model record version {int(ver[~known][0])} is unknown to this library (it reads versions "
                         f"{VERSION}, {VERSION_TABLE} and {VERSION_REGRESSORS})")
    version = int(ver[0])
    if not np.all(ver == version):
        if np.any(ver == VERSION_REGRESSORS):
            raise ValueError("version-4 model records with records of another version in one table: models with and "
                             "without extra regressors cannot be scored in one call")
        raise ValueError("version-1 and version-2 model records in one table: models without and with a seasonality "
                         "table cannot be scored in one call")
    if version != VERSION:
        reg = _REG_TAIL if version == VERSION_REGRESSORS else 0
        if np.any(np.diff(offs) < 16 + _TABLE_TAIL + reg):
            raise ValueError("bad model record header")
        tab = raw[(offs[1:] - reg - _TABLE_TAIL)[:, None] + np.arange(_TABLE_TAIL)[None, :]]
        if not np.all(tab == tab[0]):
            raise ValueError("model records with different seasonality tables in one table: each table's models are "
                             "scored with one set of options")
        if reg:
            regs = raw[(offs[1:] - reg)[:, None] + np.arange(reg)[None, :]]
            if not np.all(regs == regs[0]):
                raise ValueError("model records with different regressors in one table: each set of regressors' models "
                                 "is scored with one set of options and one io.future_regressors layout")
    return offs, bufs, version


def check_one_class(col) -> None:
    """Refuse, as decode does, a models column that mixes record versions or holds two seasonality tables or two sets
    of regressors, without decoding the records: for callers that decode the column in shards (one per rank) but must agree
    on the model class of the whole table."""
    _one_class(_column(col))


def decode(col) -> tuple:
    """Arrow binary column -> (FittedBatch, last_ds_ns, dict of the fit-time options).  Version-2 records add ``info["table"]``,
    the seasonality table as make_table_options' keyword arguments (``table_options`` rebuilds the fit's options from
    it); version-1 records have no such key.  Version-4 records add the table too, ``info["regressors"]`` (make_regressor_options'
    entries), ``info["holidays_prior_scale"]`` and the FittedBatch's ``reg_scale`` (``regressor_options`` rebuilds
    the fit's options)."""
    col = _column(col)
    n = len(col)
    offs, bufs, version = _one_class(col)
    first = col[0].as_py()
    smax, kmax = np.frombuffer(first[8:16], dtype="<i4")
    dt = record_dtype(int(smax), int(kmax), version)
    if not np.all(np.diff(offs) == dt.itemsize):
        raise ValueError("model records of differing layout in one table")
    rec = np.frombuffer(bufs[2], dtype=dt, count=n, offset=int(offs[0]))
    if not (np.all(rec["magic"] == MAGIC) and np.all(rec["version"] == version)):
        raise ValueError("bad model record header")
    flags = int(rec["flags"][0])
    fb = FittedBatch(np.ascontiguousarray(rec["params"]), np.ascontiguousarray(rec["tchange"]),
                     np.ascontiguousarray(rec["meta_i32"]), np.ascontiguousarray(rec["meta_i64"]),
                     np.ascontiguousarray(rec["meta_f64"]), int(smax), int(kmax))
    if not np.all(rec["switches"] == rec["switches"][0]) or not np.all(rec["flags"] == flags):
        raise ValueError("model records fitted with differing options in one table")
    sw = rec["switches"][0]
    info = {"logistic": bool(flags & FLAG_LOGISTIC), "multiplicative": bool(flags & FLAG_MULT),
            "yearly": int(sw[0]), "weekly": int(sw[1]), "daily": int(sw[2]), "n_changepoints": int(sw[3])}
    if version in (VERSION_TABLE, VERSION_REGRESSORS):
        ne = int(rec["n_entries"][0])
        if not 0 <= ne <= L.MAX_SEASONALITIES:
            raise ValueError(f"bad model record: {ne} seasonality entries")
        table = {}
        for key, s, order in zip(_BUILTIN_KEYS, sw[:3], rec["orders"][0]):
            table[key] = "auto" if s == L.SEAS_AUTO else ((int(order) if order > 0 else True) if s == 1 else False)
        table["seasonalities"] = [
            dict({"name": e["name"].decode(), "period": float(e["period"]), "fourier_order": int(e["fourier_order"])},
                 **({"prior_scale": float(e["prior_scale"])} if e["prior_scale"] != 0.0 else {}))
            for e in rec["entries"][0][:ne]]
        info["table"] = table
    if version == VERSION_REGRESSORS:
        R = int(rec["n_regressors"][0])
        if not 1 <= R <= L.MAX_REGRESSORS:
            raise ValueError(f"bad model record: {R} regressors")
        info["regressors"] = [
            dict({"name": e["name"].decode()}, **({"prior_scale": float(e["prior_scale"])} if e["prior_scale"] != 0.0
                                                  else {}),
                 standardize="auto" if e["standardize"] == L.STD_AUTO else bool(e["standardize"]))
            for e in rec["regressors"][0][:R]]
        info["holidays_prior_scale"] = float(rec["holidays_prior_scale"][0])
        fb.reg_scale = np.ascontiguousarray(rec["reg_scale"][:, :R, :])
    return fb, np.ascontiguousarray(rec["last_ds"]), info


def from_fbprophet_pickle(blobs, floor=None, cap=None):
    """Models written by the REFERENCE (``pickle.dumps(Prophet object)``, src/jobs/prophet_modeler.py:72-73) ->
    (FittedBatch, last_ds_ns, options dict), so that genuine fbprophet fits can be scored on the GPU path -- and
    compared with this repo's fits of the same input, the strongest parity check there is (SURVEY 8f-1, BASELINE.md
    section 2).

    Unpickling a Prophet object needs ``fbprophet`` (0.5, the reference's pin) or ``prophet`` importable; neither
    exists in this image (no network), so this function has NOT been exercised against a real pickle: it follows
    fbprophet 0.5's attribute names as recalled -- ``params`` {'k','m','delta','sigma_obs','beta'} (1 x n arrays),
    ``changepoints_t``, ``start``, ``t_scale``, ``y_scale``, ``seasonalities`` (OrderedDict name -> period /
    fourier_order / mode), ``growth``, ``seasonality_mode``, ``history_dates`` -- and raises ImportError with the
    reason when the class cannot be imported.  Only the default seasonalities (yearly 10, weekly 3, daily 4) map
    onto the compiled kernels; anything else is refused."""
    import pickle
    try:
        try:
            import fbprophet  # noqa: F401
        except ImportError:
            import prophet  # noqa: F401
    except ImportError as exc:
        raise ImportError("reading the reference's model pickles needs fbprophet (or prophet) importable: "
                          "pickle.loads re-creates a fbprophet.forecaster.Prophet object") from exc
    models = [pickle.loads(b) for b in blobs]
    n = len(models)
    if n == 0:
        raise ValueError("no models")
    m0 = models[0]
    logistic = m0.growth == "logistic"
    mult = getattr(m0, "seasonality_mode", "additive") == "multiplicative"
    orders = {"yearly": 10, "weekly": 3, "daily": 4}
    smax = max(1, max(len(np.atleast_1d(m.changepoints_t)) for m in models))
    sw = {k: 0 for k in orders}
    for m in models:
        for name, spec in m.seasonalities.items():
            if name not in orders or int(spec["fourier_order"]) != orders[name]:
                raise ValueError(f"seasonality {name!r} (order {spec.get('fourier_order')}) has no compiled kernel")
            sw[name] = 1
    kmax = sum(2 * orders[k] for k in orders if sw[k]) or 1
    pstride = 3 + smax + kmax
    params = np.zeros((n, pstride))
    tchange = np.zeros((n, smax))
    mi32 = np.zeros((n, 8), np.int32)
    mi64 = np.zeros((n, 2), np.int64)
    mf64 = np.zeros((n, 4))
    last = np.zeros(n, np.int64)
    for i, m in enumerate(models):
        p = {k: np.asarray(v, dtype=np.float64).reshape(-1) for k, v in m.params.items()}
        cps = np.atleast_1d(np.asarray(m.changepoints_t, dtype=np.float64))
        S = len(cps)
        mask, col = 0, 0
        beta = p["beta"]
        for bit, name in ((1, "yearly"), (2, "weekly"), (4, "daily")):
            if name in m.seasonalities:
                mask |= bit
        # fbprophet orders the seasonal columns as the seasonalities were added (yearly, weekly, daily for the defaults)
        k = 0
        for bit, name in ((1, "yearly"), (2, "weekly"), (4, "daily")):
            if sw[name]:
                if mask & bit:
                    params[i, 3 + smax + col:3 + smax + col + 2 * orders[name]] = beta[k:k + 2 * orders[name]]
                    k += 2 * orders[name]
                col += 2 * orders[name]
        params[i, 0], params[i, 1], params[i, 2] = p["k"][0], p["m"][0], p["sigma_obs"][0]
        params[i, 3:3 + S] = p["delta"][:S]
        tchange[i, :S] = cps
        start = np.datetime64(m.start, "ns").astype(np.int64)
        t_scale = np.timedelta64(m.t_scale, "ns").astype(np.int64)
        hist_max = np.datetime64(max(m.history_dates), "ns").astype(np.int64)
        mi32[i] = (len(m.history_dates), S, S, mask, 31, 0, 0, 0)
        mi64[i] = (start, t_scale)
        mf64[i] = (float(m.y_scale), 0.0 if floor is None else float(np.atleast_1d(floor)[min(i, np.size(floor) - 1)]),
                   np.nan if cap is None else float(np.atleast_1d(cap)[min(i, np.size(cap) - 1)]), np.nan)
        last[i] = hist_max
    fb = FittedBatch(params, tchange, mi32, mi64, mf64, smax, kmax)
    info = {"logistic": logistic, "multiplicative": mult, "yearly": sw["yearly"] or 0, "weekly": sw["weekly"] or 0,
            "daily": sw["daily"] or 0, "n_changepoints": smax}
    return fb, last, info
