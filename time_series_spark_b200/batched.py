"""Batched fit / predict: the host side of the GPU call that replaces the reference's
per-group pandas UDFs (model_time_series_udf, src/jobs/prophet_modeler.py:41-85;
forecast_time_series_udf, src/jobs/prophet_scorer.py:35-102).

All arithmetic happens in libprophet_b200.so; this module only moves buffers.
torch is used for device memory / streams when the caller wants inputs resident in HBM;
the *_host entry points take numpy arrays and stage through the library's own buffers.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, fields
from typing import Optional

import numpy as np

from . import _lib as L


def make_options(growth: str = "logistic", seasonality_mode: str = "multiplicative",
                 yearly_seasonality="auto", weekly_seasonality="auto", daily_seasonality="auto",
                 n_changepoints: int = 25, changepoint_range: float = 0.8,
                 changepoint_prior_scale: float = 0.05, seasonality_prior_scale: float = 10.0,
                 interval_width: float = 0.8, uncertainty_samples: int = 1000,
                 max_iter: int = 10000, algorithm: str = "LBFGS+Newton") -> L.Options:
    """Prophet.__init__ arguments -> pb200_options.  Defaults = the reference's hard-coded
    ``Prophet(growth='logistic', seasonality_mode='multiplicative')`` (prophet_modeler.py:65)."""
    o = L.default_options()
    if growth not in ("linear", "logistic"):
        raise ValueError('Parameter "growth" should be "linear" or "logistic".')
    if seasonality_mode not in ("additive", "multiplicative"):
        raise ValueError('seasonality_mode must be "additive" or "multiplicative"')
    o.growth = L.GROWTH_LOGISTIC if growth == "logistic" else L.GROWTH_LINEAR
    o.multiplicative = 1 if seasonality_mode == "multiplicative" else 0

    def sw(v, default_order):
        if isinstance(v, str) and v == "auto":
            return L.SEAS_AUTO
        if v is True:
            return 1
        if v is False:
            return 0
        if int(v) == 0:
            return 0
        if int(v) == default_order:
            return 1
        raise ValueError(f"only the default Fourier order {default_order} is compiled in (got {v})")

    o.yearly, o.weekly, o.daily = sw(yearly_seasonality, 10), sw(weekly_seasonality, 3), sw(daily_seasonality, 4)
    o.n_changepoints = int(n_changepoints)
    o.changepoint_range = float(changepoint_range)
    o.changepoint_prior_scale = float(changepoint_prior_scale)
    o.seasonality_prior_scale = float(seasonality_prior_scale)
    o.interval_width = float(interval_width)
    o.uncertainty_samples = int(uncertainty_samples)
    o.max_iter = int(max_iter)
    o.algorithm = {"LBFGS+Newton": L.ALG_LBFGS_NEWTON, "LBFGS": L.ALG_LBFGS, "Newton": L.ALG_NEWTON}[algorithm]
    return o


# fbprophet 0.5's validate_column_name: names a seasonality may not take (they are columns of its predict frame)
_RESERVED_NAMES = frozenset([
    "trend", "additive_terms", "multiplicative_terms", "holidays", "zeros", "extra_regressors_additive",
    "extra_regressors_multiplicative", "yhat", "ds", "y", "cap", "floor", "y_scaled", "cap_scaled"])


def _number(v, key: str) -> float:
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)):
        raise ValueError(f"{key} must be a number (got {v!r})")
    return float(v)


def make_table_options(seasonalities=(), yearly_seasonality="auto", weekly_seasonality="auto",
                       daily_seasonality="auto", seasonality_mode: str = "multiplicative",
                       seasonality_prior_scale: float = 10.0, **kw) -> L.OptionsV2:
    """make_options plus fbprophet's add_seasonality and any built-in Fourier order (DESIGN §18): a pb200_options_v2.

    ``yearly_seasonality`` / ``weekly_seasonality`` / ``daily_seasonality``: 'auto', True, False or an int order (> 0
    forces it on at that order, 0 is off).  ``seasonalities``: dicts ``{name, period, fourier_order, prior_scale?,
    mode?}`` in the order they were added; ``prior_scale`` defaults to ``seasonality_prior_scale`` and ``mode`` must be
    ``seasonality_mode``.  Other keyword arguments are make_options'.  A table that restates the defaults gives the
    default model; the limits (8 seasonalities, K <= 64, P <= 96) are checked here and by the library."""
    builtin = {}
    for key, v, dflt in (("yearly_seasonality", yearly_seasonality, 10), ("weekly_seasonality", weekly_seasonality, 3),
                         ("daily_seasonality", daily_seasonality, 4)):
        if isinstance(v, str):
            if v != "auto":
                raise ValueError(f"{key} must be 'auto', a bool or an int order (got {v!r})")
            builtin[key] = ("auto", 0)
        elif isinstance(v, (bool, np.bool_)):
            builtin[key] = (bool(v), 0)
        else:
            if not isinstance(v, (int, np.integer)):
                raise ValueError(f"{key} must be 'auto', a bool or an int order (got {v!r})")
            n = int(v)
            if n < 0:
                raise ValueError(f"{key} must be >= 0 (got {n})")
            builtin[key] = (n > 0, n if n > 0 else 0)
    o1 = make_options(yearly_seasonality=builtin["yearly_seasonality"][0],
                      weekly_seasonality=builtin["weekly_seasonality"][0],
                      daily_seasonality=builtin["daily_seasonality"][0], seasonality_mode=seasonality_mode,
                      seasonality_prior_scale=seasonality_prior_scale, **kw)
    o = L.OptionsV2()
    for name, _ in L.Options._fields_:
        setattr(o, name, getattr(o1, name))
    o.abi_version = L.ABI_VERSION_TABLE
    o.yearly_order = builtin["yearly_seasonality"][1]
    o.weekly_order = builtin["weekly_seasonality"][1]
    o.daily_order = builtin["daily_seasonality"][1]
    seasonalities = list(seasonalities or ())
    if len(seasonalities) > L.MAX_SEASONALITIES:
        raise ValueError(f"seasonalities: at most {L.MAX_SEASONALITIES} entries (got {len(seasonalities)})")
    arr = (L.Seasonality * max(1, len(seasonalities)))()
    names = set()
    for i, spec in enumerate(seasonalities):
        key = f"seasonalities[{i}]"
        if not isinstance(spec, dict):
            raise ValueError(f"{key} must be a mapping with name, period and fourier_order")
        unknown = set(spec) - {"name", "period", "fourier_order", "prior_scale", "mode"}
        if unknown:
            raise ValueError(f"{key}: unknown key(s) {sorted(unknown)}")
        for req in ("name", "period", "fourier_order"):
            if req not in spec:
                raise ValueError(f"{key}.{req} is required")
        name = spec["name"]
        if not isinstance(name, str) or not name or len(name.encode()) > 15:
            raise ValueError(f"{key}.name must be a non-empty string of at most 15 bytes (got {name!r})")
        if name in names:
            raise ValueError(f"{key}.name: seasonality {name!r} is added twice")
        if name in _RESERVED_NAMES or name.endswith(("_lower", "_upper")):
            raise ValueError(f"{key}.name: {name!r} is reserved (fbprophet's validate_column_name)")
        names.add(name)
        for b, bkey in (("yearly", "yearly_seasonality"), ("weekly", "weekly_seasonality"), ("daily", "daily_seasonality")):
            if name == b and builtin[bkey][0] != "auto":
                raise ValueError(f"{key}.name: {name!r} replaces the built-in only when {bkey} is 'auto'")
        period = _number(spec["period"], f"{key}.period")
        if not (np.isfinite(period) and period > 0):
            raise ValueError(f"{key}.period must be finite and > 0 (got {spec['period']!r})")
        order = spec["fourier_order"]
        if isinstance(order, (bool, np.bool_)) or not isinstance(order, (int, np.integer)) or int(order) <= 0:
            raise ValueError(f"{key}.fourier_order must be an int > 0 (got {order!r})")
        ps = spec.get("prior_scale")
        if ps is not None and not (np.isfinite(_number(ps, f"{key}.prior_scale")) and float(ps) > 0):
            raise ValueError(f"{key}.prior_scale must be > 0 (got {ps!r})")
        mode = spec.get("mode")
        if mode is not None and mode != seasonality_mode:
            raise ValueError(f"{key}.mode: every seasonality takes the model's seasonality_mode {seasonality_mode!r} "
                             f"(got {mode!r})")
        arr[i].name = name.encode()
        arr[i].period = period
        arr[i].fourier_order = int(order)
        arr[i].prior_scale = 0.0 if ps is None else float(ps)
    o.n_seasonalities = len(seasonalities)
    o.seasonalities = C.cast(arr, C.POINTER(L.Seasonality))
    o._table = arr      # keeps the entries alive as long as the options
    L.get_layout(o)     # the library's checks: the limits and the refusals, before any GPU call
    return o


def make_regressor_options(regressors=(), holidays_prior_scale: float = 10.0, **kw) -> L.OptionsV3:
    """make_table_options plus fbprophet's add_regressor (DESIGN §19): a pb200_options_v3.

    ``regressors``: dicts ``{name, prior_scale?, standardize?, mode?}`` in the order they were added.  ``prior_scale``
    defaults to ``holidays_prior_scale``; ``standardize`` is 'auto' (the default), True or False; ``mode`` must be the
    model's ``seasonality_mode``.  Other keyword arguments are make_table_options'.  With no regressor the options are
    exactly make_table_options'.  The limits (16 regressors, K + R <= 64, P <= 96) are checked here and by the library.
    The regressor values go to the ``regressors=`` argument of the fit and predict calls."""
    mode = kw.get("seasonality_mode", "multiplicative")
    o2 = make_table_options(**kw)
    o = L.OptionsV3()
    C.memmove(C.addressof(o), C.addressof(o2), C.sizeof(L.OptionsV2))
    o._table = o2._table
    o.abi_version = L.ABI_VERSION_REGRESSORS
    hps = _number(holidays_prior_scale, "holidays_prior_scale")
    if not (np.isfinite(hps) and hps > 0):
        raise ValueError(f"holidays_prior_scale must be finite and > 0 (got {holidays_prior_scale!r})")
    o.holidays_prior_scale = hps
    regressors = list(regressors or ())
    if len(regressors) > L.MAX_REGRESSORS:
        raise ValueError(f"regressors: at most {L.MAX_REGRESSORS} entries (got {len(regressors)})")
    seas_names = {o.seasonalities[i].name.decode() for i in range(o.n_seasonalities)} | {"yearly", "weekly", "daily"}
    arr = (L.Regressor * max(1, len(regressors)))()
    names = set()
    for i, spec in enumerate(regressors):
        key = f"regressors[{i}]"
        if not isinstance(spec, dict):
            raise ValueError(f"{key} must be a mapping with a name")
        unknown = set(spec) - {"name", "prior_scale", "standardize", "mode"}
        if unknown:
            raise ValueError(f"{key}: unknown key(s) {sorted(unknown)}")
        if "name" not in spec:
            raise ValueError(f"{key}.name is required")
        name = spec["name"]
        if not isinstance(name, str) or not name or len(name.encode()) > 15:
            raise ValueError(f"{key}.name must be a non-empty string of at most 15 bytes (got {name!r})")
        if name in _RESERVED_NAMES or name.endswith(("_lower", "_upper")):
            raise ValueError(f"{key}.name: {name!r} is reserved (fbprophet's validate_column_name)")
        if name in seas_names:
            raise ValueError(f"{key}.name: {name!r} is already used as a seasonality name")
        if name in names:
            raise ValueError(f"{key}.name: regressor {name!r} is added twice")
        names.add(name)
        ps = spec.get("prior_scale")
        if ps is not None and not (np.isfinite(_number(ps, f"{key}.prior_scale")) and float(ps) > 0):
            raise ValueError(f"{key}.prior_scale must be > 0 (got {ps!r})")
        st = spec.get("standardize", "auto")
        if not ((isinstance(st, str) and st == "auto") or isinstance(st, (bool, np.bool_))):
            raise ValueError(f"{key}.standardize must be 'auto', True or False (got {st!r})")
        rmode = spec.get("mode")
        if rmode is not None and rmode != mode:
            raise ValueError(f"{key}.mode: every regressor takes the model's seasonality_mode {mode!r} (got {rmode!r})")
        arr[i].name = name.encode()
        arr[i].prior_scale = 0.0 if ps is None else float(ps)
        arr[i].standardize = L.STD_AUTO if isinstance(st, str) else int(bool(st))
    o.n_regressors = len(regressors)
    o.regressors = C.cast(arr, C.POINTER(L.Regressor))
    o._regressors = arr     # keeps the entries alive as long as the options
    L.get_layout(o)         # the library's checks: the limits and the refusals, before any GPU call
    return o


def _has_table(opts) -> bool:
    """Whether ``opts`` carries a seasonality table: a pb200_options_v2, or a v3 (which embeds one)."""
    return getattr(opts, "abi_version", L.ABI_VERSION) in (L.ABI_VERSION_TABLE, L.ABI_VERSION_REGRESSORS)


def n_regressors(opts) -> int:
    """R of ``opts``: its regressor count at version 3, else 0."""
    return int(opts.n_regressors) if getattr(opts, "abi_version", L.ABI_VERSION) == L.ABI_VERSION_REGRESSORS else 0


def regressor_scales(reg, offsets, standardize, copy=None) -> np.ndarray:
    """fbprophet 0.5's initialize_scales for the regressors, restated on the host (the test reference of the library's
    standardisation): ``[n, R, 2]`` (mu, std) per series.  ``reg``: ``[R, n_rows]`` values aligned with the batch's rows;
    ``standardize``: per regressor 'auto', True or False.  Fewer than two distinct values, or 'auto' on values that are
    exactly {0, 1}: (0, 1), or with ``copy`` (``[n, R, 2]``, a prophet_copy's scales, DESIGN §20) the series' copy
    entry; else the mean and the sample standard deviation (ddof = 1).  A non-finite value: (NaN, NaN)."""
    reg = np.asarray(reg, np.float64)
    offsets = np.asarray(offsets, np.int64)
    n, R = offsets.size - 1, reg.shape[0]
    out = np.zeros((n, R, 2))
    out[:, :, 1] = 1.0
    if copy is not None:
        out[:] = np.asarray(copy, np.float64)
    for i in range(n):
        for r in range(R):
            x = reg[r, offsets[i]:offsets[i + 1]]
            if not np.all(np.isfinite(x)):
                out[i, r] = np.nan
                continue
            vals = np.unique(x)
            st = standardize[r]
            if vals.size < 2:
                continue
            if isinstance(st, str):
                st = set(vals.tolist()) != {0.0, 1.0}
            if st:
                mu = x.sum() / x.size
                out[i, r] = mu, np.sqrt(((x - mu) ** 2).sum() / (x.size - 1))
    return out


_BUILTINS = (("yearly", 1, 365.25, 10), ("weekly", 2, 7.0, 3), ("daily", 4, 1.0, 4))


def is_table(opts) -> bool:
    """Whether ``opts`` is a pb200_options_v2 whose table is not a restatement of the default model."""
    return seasonality_table(opts) is not None


def seasonality_table(opts):
    """The seasonality table of ``opts`` as the library normalises it (DESIGN §18): a list of entries
    ``(name, period, fourier_order, kind)`` in column order -- the custom entries as added, then the built-ins that are
    not off and not replaced by a custom entry of their name -- where ``kind`` is 0 for a custom entry and the built-in's
    mask bit (1 yearly, 2 weekly, 4 daily) otherwise.  None for v1 options and for a table that restates the defaults
    (the v1 model).  With regressors (version 3) it is never None: such a model is a table model even when its table
    restates the defaults."""
    if not _has_table(opts):
        return None
    custom = [opts.seasonalities[i] for i in range(opts.n_seasonalities)]
    orders = (opts.yearly_order, opts.weekly_order, opts.daily_order)
    switches = (opts.yearly, opts.weekly, opts.daily)
    if not custom and not n_regressors(opts) and all(o == 0 or o == d or s == 0 for o, s, (_, _, _, d) in zip(orders, switches, _BUILTINS)):
        return None
    names = [e.name.decode() for e in custom]
    out = [(e.name.decode(), float(e.period), int(e.fourier_order), 0) for e in custom]
    for (name, bit, period, dflt), order, sw in zip(_BUILTINS, orders, switches):
        if sw != 0 and name not in names:
            out.append((name, period, order or dflt, bit))
    return out


def table_mask(table, builtin_mask):
    """The table mask (bit j: entry j of ``seasonality_table`` active) of histories with built-in mask ``builtin_mask``
    (scalar or array): the library's tab_mask."""
    bm = np.asarray(builtin_mask)
    m = np.zeros(bm.shape, np.int32)
    for j, (_, _, _, kind) in enumerate(table):
        m |= np.where((kind == 0) | ((bm & kind) != 0), np.int32(1 << j), np.int32(0))
    return m


def copy_options(opts):
    """A copy of ``opts`` that shares nothing mutable with it: the whole pb200_options_v2 for a table (its entries kept
    alive by the copy), pb200_options otherwise."""
    version = getattr(opts, "abi_version", L.ABI_VERSION)
    if not _has_table(opts):
        return L.Options.from_buffer_copy(opts)
    o = (L.OptionsV2 if version == L.ABI_VERSION_TABLE else L.OptionsV3).from_buffer_copy(opts)
    n = opts.n_seasonalities
    arr = (L.Seasonality * max(1, n))()
    for i in range(n):
        arr[i] = L.Seasonality.from_buffer_copy(opts.seasonalities[i])
    o.seasonalities = C.cast(arr, C.POINTER(L.Seasonality))
    o._table = arr
    if version == L.ABI_VERSION_REGRESSORS:
        regs = (L.Regressor * max(1, opts.n_regressors))()
        for i in range(opts.n_regressors):
            regs[i] = L.Regressor.from_buffer_copy(opts.regressors[i])
        o.regressors = C.cast(regs, C.POINTER(L.Regressor))
        o._regressors = regs
    return o


@dataclass
class FittedBatch:
    """Fitted-model arrays of one shard (numpy on host, or torch tensors on device)."""
    params: object       # [N, pstride] f64: k, m, sigma_obs, delta[smax], beta[kmax]
    tchange: object      # [N, smax]    f64
    meta_i32: object     # [N, 8]  T, S, n_cp_real, seasonality mask, status, iters, n_evals, i1
    meta_i64: object     # [N, 2]  start_ns, t_scale_ns
    meta_f64: object     # [N, 4]  y_scale, floor, cap, neg_log_posterior
    smax: int
    kmax: int
    warm: object = None  # [N] int32 L.WARM_* of a warm-started fit (where each series started); None for a cold fit
    reg_scale: object = None  # [N, R, 2] f64 (mu, std) of each regressor (a fit with regressors), else None

    @property
    def n(self) -> int:
        return int(self.params.shape[0])

    @property
    def status(self):
        return self.meta_i32[:, 4]

    def to_host(self) -> "FittedBatch":
        if isinstance(self.params, np.ndarray):
            return self
        return FittedBatch(*(x.cpu().numpy() for x in (self.params, self.tchange, self.meta_i32,
                                                       self.meta_i64, self.meta_f64)),
                           smax=self.smax, kmax=self.kmax, warm=None if self.warm is None else self.warm.cpu().numpy(),
                           reg_scale=None if self.reg_scale is None else self.reg_scale.cpu().numpy())


def _seasonal_k(mask):
    """Fourier columns K of a seasonality mask (1 yearly 20 | 2 weekly 6 | 4 daily 8); fbprophet's single zero column
    when there is none."""
    mask = np.asarray(mask)
    k = 20 * (mask & 1 != 0) + 6 * (mask & 2 != 0) + 8 * (mask & 4 != 0)
    return np.where(k > 0, k, 1)


def warm_start(init: FittedBatch, S, mask, fitted) -> tuple:
    """Where each series of a warm-started fit starts (DESIGN §11, rules 1 and 2), restated on the host: the reference the
    device's choice (prep_kernel) is tested against.  ``init``: the previous models (host arrays, rows aligned with the
    batch); ``S`` / ``mask``: the new histories' changepoint count and seasonality mask; ``fitted``: whether a series is
    optimised at all (False after a prep error or for the constant-linear shortcut).  Returns ``(codes, x)``: int32
    ``L.WARM_*`` per series, and ``[n, pstride]`` start points in Stan's unconstrained order (k, m, delta[S],
    log sigma_obs, beta[K]) for the series whose code is ``L.WARM_USED`` (other rows NaN)."""
    init = init.to_host()
    S, mask, fitted = np.asarray(S), np.asarray(mask), np.asarray(fitted, dtype=bool)
    n, smax = init.n, init.smax
    p, mi = init.params, init.meta_i32
    K = _seasonal_k(mask)
    codes = np.full(n, L.WARM_NONE, np.int32)
    x = np.full(p.shape, np.nan)
    cand = fitted & (mi[:, 4] >= 0)
    shape_ok = (mi[:, 1] == S) & (mi[:, 3] == mask)
    codes[cand & ~shape_ok] = L.WARM_SHAPE
    col = np.arange(p.shape[1])[None, :]
    delta_in = (col >= 3) & (col < 3 + S[:, None])
    beta_in = (col >= 3 + smax) & (col < 3 + smax + K[:, None])
    used_cols = (col < 2) | delta_in | beta_in
    with np.errstate(invalid="ignore"):
        finite = np.all(np.isfinite(p) | ~used_cols, axis=1) & np.isfinite(p[:, 2]) & (p[:, 2] > 0)
    codes[cand & shape_ok & ~finite] = L.WARM_BAD
    use = cand & shape_ok & finite
    for i in np.flatnonzero(use):      # one row per used series: the test reference, not a hot path
        s_, k_ = int(S[i]), int(K[i])
        x[i, :3 + s_ + k_] = np.concatenate((p[i, :2], p[i, 3:3 + s_], [np.log(p[i, 2])], p[i, 3 + smax:3 + smax + k_]))
    codes[use] = L.WARM_USED
    return codes, x


def _check_init(init, n: int, lay) -> None:
    if not isinstance(init, FittedBatch):
        raise ValueError("init must be a FittedBatch of the previous models")
    if init.n != n or init.smax != lay.smax or init.kmax != lay.kmax:
        raise ValueError(f"init has {init.n} rows with smax {init.smax}, kmax {init.kmax}; the batch has {n} series and the "
                         f"options' layout smax {lay.smax}, kmax {lay.kmax}")


def _y_dtype(y) -> int:
    dt = str(y.dtype).replace("torch.", "")
    if dt == "int32":
        return L.Y_I32
    if dt == "float32":
        return L.Y_F32
    if dt == "float64":
        return L.Y_F64
    raise TypeError(f"y must be int32, float32 or float64 (got {y.dtype})")


def _np_ptr(a: np.ndarray) -> int:
    return a.ctypes.data


def _host_regressors(opts, regressors, rows: int) -> np.ndarray:
    """The ``regressors=`` values of a host call: float64 ``[R, rows]``."""
    R = n_regressors(opts)
    reg = np.ascontiguousarray(regressors, dtype=np.float64)
    if reg.size != R * rows:
        raise ValueError(f"regressors must hold [{R}, {rows}] values (got shape {reg.shape})")
    return reg.reshape(R, rows)


def _check_reg_scale(reg_scale, n: int, R: int, what: str, dev=None) -> None:
    """A (mu, std) array the library reads or writes as [n][R][2] doubles: float64, that shape, contiguous (and on ``dev``
    for a device call)."""
    if reg_scale is None:
        raise ValueError(f"{what} is missing (a fit with regressors)")
    dt = str(reg_scale.dtype).replace("torch.", "")
    contiguous = reg_scale.is_contiguous() if dev is not None else True
    if (dt != "float64" or tuple(reg_scale.shape) != (n, R, 2) or not contiguous
            or (dev is not None and getattr(reg_scale, "device", None) != dev)):
        raise ValueError(f"{what} must be a contiguous float64 array of shape ({n}, {R}, 2)"
                         + (f" on {dev}" if dev is not None else "") + f" (got {dt} {tuple(reg_scale.shape)})")


class _Space:
    """Where a call's arrays live: numpy on the host (``dev`` None), or torch tensors on the device ``dev``.  The
    entry points of a call family differ only in this, and in their suffix."""

    def __init__(self, dev=None):
        self.dev = dev
        self.suffix = "_host" if dev is None else "_device"

    def empty(self, shape, dtype: str):
        if self.dev is None:
            return np.empty(shape, dtype)
        import torch
        return torch.empty(shape, dtype=getattr(torch, dtype), device=self.dev)

    def zeros(self, shape, dtype: str):
        if self.dev is None:
            return np.zeros(shape, dtype)
        import torch
        return torch.zeros(shape, dtype=getattr(torch, dtype), device=self.dev)

    def asarray(self, a, dtype: str):
        """``a`` (numpy, or a torch tensor for a device call) as a contiguous ``dtype`` array here; a copy only where
        needed."""
        if self.dev is None:
            return np.ascontiguousarray(a, dtype=dtype)
        import torch
        return torch.as_tensor(a, dtype=getattr(torch, dtype), device=self.dev).contiguous()

    def ptr(self, a):
        if a is None:
            return None
        return a.ctypes.data if self.dev is None else a.data_ptr()

    def sync_torch(self) -> None:
        """Before a device call: its inputs were produced on torch's current stream; the library has its own stream."""
        if self.dev is not None:
            import torch
            torch.cuda.current_stream(self.dev).synchronize()


_HOST = _Space()


def _call(entry: str, *args) -> None:
    L.check(getattr(L.load(), entry)(*args), entry)


_FIT_FIELDS = ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")


def _fitted_outputs(space: _Space, n: int, lay, R: int = 0, zeros: bool = False) -> FittedBatch:
    """A FittedBatch for ``n`` series of layout ``lay`` for a fit to write, with ``reg_scale`` when R > 0.  ``zeros``:
    params and tchange start zero-filled (a fit narrower than ``lay`` leaves their pad columns at 0)."""
    pad = space.zeros if zeros else space.empty
    return FittedBatch(pad((n, lay.pstride), "float64"), pad((n, lay.smax), "float64"), space.empty((n, 8), "int32"),
                       space.empty((n, 2), "int64"), space.empty((n, 4), "float64"), lay.smax, lay.kmax,
                       reg_scale=space.empty((n, R, 2), "float64") if R else None)


def _fit(space: _Space, ctx, opts, ds_ns, y, offsets, floor, cap_multiplier, kind: str, cap=None, prior=None,
         init=None, regressors=None, reg_scale_copy=None, trace_cap: int = 0, out=None, sync: bool = False):
    """The body of the fit wrappers: pb200_fit[_<kind>][_copy]_host / _device, ``kind`` "fit", "trace" or "warm", or
    "regressors" whenever ``regressors`` is given.  A host call converts its inputs and returns a trace array for the
    trace, and for the warm and regressor fits with ``trace_cap`` > 0; a device call checks its inputs and synchronises
    the context after the call with ``sync`` or ``init``.  Returns (FittedBatch, trace or None)."""
    host = space.dev is None
    if host:
        ds_ns, y = np.ascontiguousarray(ds_ns, dtype=np.int64), np.ascontiguousarray(y)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    n = offsets.size - 1
    lay = L.get_layout(opts)
    R = 0
    if reg_scale_copy is not None and regressors is None:
        raise ValueError("reg_scale_copy goes with regressors")
    if regressors is not None:
        if prior is not None or init is not None:
            raise ValueError("regressors are not supported with prior or init")
        kind, R = "regressors", n_regressors(opts)
        if host:
            regressors = _host_regressors(opts, regressors, ds_ns.size)
        else:
            import torch
            rows = int(offsets[-1])
            if (regressors.dtype != torch.float64 or tuple(regressors.shape) != (R, rows)
                    or not regressors.is_contiguous() or regressors.device != space.dev):
                raise ValueError(f"regressors must be a contiguous float64 tensor of shape ({R}, {rows}) on {space.dev}")
    if init is not None:
        _check_init(init, n, lay)
    if out is None:
        out = _fitted_outputs(space, n, lay, R)
    if R:
        if out.reg_scale is None:
            out.reg_scale = space.empty((n, R, 2), "float64")
        if not host:
            _check_reg_scale(out.reg_scale, n, R, "out.reg_scale", space.dev)
            if reg_scale_copy is not None:
                _check_reg_scale(reg_scale_copy, n, R, "reg_scale_copy", space.dev)
    ip = im = None
    if init is not None:
        src = init.to_host() if host else init
        ip, im = space.asarray(src.params, "float64"), space.asarray(src.meta_i32, "int32")
        if out.warm is None:
            out.warm = space.empty(n, "int32")
    if host:
        if cap is not None:
            cap = np.ascontiguousarray(cap, dtype=np.float64)
        if prior is not None:
            prior = np.ascontiguousarray(prior, dtype=np.float64).reshape(n, 2)
    trace = space.zeros((n, trace_cap, 4), "float64") if kind == "trace" or trace_cap > 0 else None
    if n > 0:
        if not host:
            import torch
            if prior is not None and (prior.dtype != torch.float64 or tuple(prior.shape) != (n, 2)
                                      or not prior.is_contiguous() or prior.device != space.dev):
                raise ValueError(f"prior must be a contiguous float64 tensor of shape ({n}, 2) on {space.dev}")
            space.sync_torch()
        p = space.ptr
        args = [ctx.handle, C.byref(opts), p(ds_ns), p(y), _y_dtype(y), _np_ptr(offsets), n, float(floor),
                float(cap_multiplier)]
        if kind != "trace":
            args.append(p(cap))
        if kind == "warm":
            args += [p(prior), p(ip), p(im)]
        if kind == "regressors":
            args += [p(regressors)] + ([p(reg_scale_copy)] if reg_scale_copy is not None else []) + [p(out.reg_scale)]
        args += [p(getattr(out, f)) for f in _FIT_FIELDS]
        if kind == "warm":
            args.append(p(out.warm) if init is not None else None)
        if host and kind != "fit":
            args += [p(trace), int(trace_cap)]
        entry = "pb200_fit" + ("" if kind == "fit" else "_" + kind) + ("_copy" if reg_scale_copy is not None else "")
        _call(entry + space.suffix, *args)
        if not host and (sync or init is not None):       # (the uploaded copies of init must outlive the call)
            ctx.synchronize()
    return out, trace


def fit_batch_host(ctx: L.Context, opts: L.Options, ds_ns: np.ndarray, y: np.ndarray, offsets: np.ndarray,
                   floor: float, cap_multiplier: float, cap: Optional[np.ndarray] = None, regressors=None) -> FittedBatch:
    """pb200_fit_host: numpy (ideally pinned) buffers in, numpy out; copies inside the call.  ``regressors``: None, or
    for options with regressors (make_regressor_options) their values ``[R, n_rows]`` aligned with ``ds_ns``
    (pb200_fit_regressors_host); ``FittedBatch.reg_scale`` then holds each series' standardisation."""
    return _fit(_HOST, ctx, opts, ds_ns, y, offsets, floor, cap_multiplier, "fit", cap=cap, regressors=regressors)[0]


def fit_batch_trace_host(ctx: L.Context, opts: L.Options, ds_ns: np.ndarray, y: np.ndarray, offsets: np.ndarray,
                         floor: float, cap_multiplier: float, trace_cap: int = 256, regressors=None):
    """pb200_fit_trace_host (parity-test hook): the fit plus, per series, one row
    ``(iteration, f_k, alpha_k, n_evals)`` per accepted L-BFGS iteration (``[n, trace_cap, 4]``).  ``regressors``: as
    fit_batch_host's (pb200_fit_regressors_host with the trajectory)."""
    return _fit(_HOST, ctx, opts, ds_ns, y, offsets, floor, cap_multiplier, "trace", regressors=regressors,
                trace_cap=int(trace_cap))


def fit_batch_warm_host(ctx: L.Context, opts: L.Options, ds_ns: np.ndarray, y: np.ndarray, offsets: np.ndarray,
                        floor: float, cap_multiplier: float, init: Optional[FittedBatch], cap: Optional[np.ndarray] = None,
                        prior: Optional[np.ndarray] = None, trace_cap: int = 0):
    """pb200_fit_warm_host: ``fit_batch_device(init=...)`` on numpy buffers, plus (``trace_cap`` > 0) the trajectory rows
    of ``fit_batch_trace_host``.  Returns ``(FittedBatch, trace or None)``; ``FittedBatch.warm`` holds the
    ``L.WARM_*`` codes when ``init`` is given."""
    return _fit(_HOST, ctx, opts, ds_ns, y, offsets, floor, cap_multiplier, "warm", cap=cap, prior=prior, init=init,
                trace_cap=trace_cap)


def regressor_scales_device(ctx: L.Context, opts, regressors, offsets_host: np.ndarray):
    """pb200_regressor_scales_device: the standardisation a fit with ``regressors`` (a contiguous float64 CUDA tensor
    ``[R, n_rows]``) gives each series, without the fit: ``(reg_scale [n, R, 2] float64, bad [n] bool)`` CUDA tensors,
    ``bad`` where a value of the series is not finite."""
    import torch
    offsets_host = np.ascontiguousarray(offsets_host, dtype=np.int64)
    n = offsets_host.size - 1
    R = n_regressors(opts)
    dev = regressors.device
    rows = int(offsets_host[-1])
    if (regressors.dtype != torch.float64 or tuple(regressors.shape) != (R, rows) or not regressors.is_contiguous()):
        raise ValueError(f"regressors must be a contiguous float64 tensor of shape ({R}, {rows})")
    scale = torch.empty((n, R, 2), dtype=torch.float64, device=dev)
    bad = torch.zeros(n, dtype=torch.uint8, device=dev)
    if n:
        torch.cuda.current_stream(dev).synchronize()
        L.check(L.load().pb200_regressor_scales_device(ctx.handle, C.byref(opts), regressors.data_ptr(),
                                                       _np_ptr(offsets_host), n, scale.data_ptr(), bad.data_ptr()),
                "pb200_regressor_scales_device")
    return scale, bad.bool()


def fit_batch_device(ctx: L.Context, opts: L.Options, ds_ns, y, offsets_host: np.ndarray,
                     floor: float, cap_multiplier: float, cap=None, out: Optional[FittedBatch] = None,
                     sync: bool = True, prior=None, init: Optional[FittedBatch] = None, regressors=None,
                     reg_scale_copy=None) -> FittedBatch:
    """pb200_fit_warm_device: ``ds_ns`` / ``y`` / ``cap`` are torch CUDA tensors already in HBM.  ``prior``: None (the
    options' prior scales) or a float64 CUDA tensor ``[n, 2]`` of (changepoint_prior_scale, seasonality_prior_scale)
    per series; a series whose pair is not finite and > 0 gets status ``L.ST_BAD_PRIOR``.  ``init``: None (every
    series starts from fbprophet's stan_init) or the previous models, a FittedBatch (host or device) whose rows are
    aligned with the batch and whose layout is the options'; each series then starts from its previous optimum when
    DESIGN §11's rule allows, and ``out.warm`` receives the ``L.WARM_*`` code of every series.  ``regressors``: None, or
    for options with regressors (make_regressor_options) a contiguous float64 CUDA tensor ``[R, n_rows]`` of their
    values aligned with ``ds_ns`` (pb200_fit_regressors_device; not with ``prior`` or ``init``); ``out.reg_scale``
    then receives each series' standardisation ``[n, R, 2]``.  ``reg_scale_copy`` (with ``regressors``): a float64 CUDA
    tensor ``[n, R, 2]``, the (mu, std) each regressor keeps where it is not standardised instead of (0, 1)
    (pb200_fit_regressors_copy_device; the backtest's prophet_copy, DESIGN §20)."""
    return _fit(_Space(ds_ns.device), ctx, opts, ds_ns, y, offsets_host, floor, cap_multiplier, "warm", cap=cap,
                prior=prior, init=init, regressors=regressors, reg_scale_copy=reg_scale_copy, out=out, sync=sync)[0]


@dataclass
class ForecastBatch:
    future_ds: object    # [N, H] int64 ns
    yhat: object         # [N, H] f64
    yhat_lower: object   # [N, H] f64 or None
    yhat_upper: object
    yhat_int: object     # [N, H] int32 (truncated, floor-clamped)
    components: object = None   # [C, N, H] f64, planes in component_names(opts) order (components=True), else None
    trend_lower: object = None  # [N, H] f64 (components=True with intervals), else None
    trend_upper: object = None
    quantiles: object = None    # [Q, N, H] f64 (predict_quantiles_*), else None
    names: tuple = L.COMPONENTS  # the component planes' names

    def component(self, name: str):
        """One component plane by its fbprophet column name (trend, multiplicative_terms, additive_terms, yearly, weekly,
        daily, and a seasonality table's custom entries)."""
        return self.components[self.names.index(name)]


def component_names(opts: L.Options) -> tuple:
    """The planes of pb200_predict_components_* for these options: L.COMPONENTS, then each custom seasonality of a
    seasonality table not named like a built-in, in table order."""
    n = L.load().pb200_component_count(C.byref(opts))
    L.check(min(n, 0), "pb200_component_count")
    extra = []
    if _has_table(opts):
        extra = [opts.seasonalities[i].name.decode() for i in range(opts.n_seasonalities)]
        extra = [x for x in extra if x not in ("yearly", "weekly", "daily")]
    names = L.COMPONENTS + tuple(extra)
    assert len(names) == n
    return names


def make_future(last_ds_ns: np.ndarray, periods: int, freq_ns: int) -> np.ndarray:
    """Prophet.make_future_dataframe(include_history=False) for a fixed-width frequency
    (prophet_scorer.py:64-66): last + (1..periods) * freq."""
    last = np.asarray(last_ds_ns, dtype=np.int64)
    return last[:, None] + np.int64(freq_ns) * np.arange(1, periods + 1, dtype=np.int64)[None, :]


def make_future_device(ctx: L.Context, last_ds_ns, periods: int, freq_ns: int):
    """pb200_make_future_device: the same grid built on the GPU from a CUDA int64 tensor of last history timestamps
    (for callers that keep the scorer's inputs resident)."""
    import torch
    n = int(last_ds_ns.shape[0])
    out = torch.empty((n, periods), dtype=torch.int64, device=last_ds_ns.device)
    if n and periods:
        torch.cuda.current_stream(last_ds_ns.device).synchronize()
        rc = L.load().pb200_make_future_device(ctx.handle, last_ds_ns.data_ptr(), n, int(periods), int(freq_ns), out.data_ptr())
        L.check(rc, "pb200_make_future_device")
        ctx.synchronize()
    return out


def join_future_regressors_device(ctx: L.Context, tab_ds, tab_offsets_host: np.ndarray, tab_reg, model_group,
                                  future_ds):
    """pb200_join_future_regressors_device (DESIGN §20): the regressors' values of every model's forecast grid from a
    packed table.  ``tab_ds`` int64 ``[rows]`` and ``tab_reg`` float64 ``[R, rows]`` CUDA tensors packed by group
    (``tab_offsets_host`` ``[n_groups + 1]``, timestamps ascending and distinct within a group); ``model_group`` int64
    ``[n]`` each model's group (-1: none); ``future_ds`` int64 ``[n, H]``.  Returns ``(future_reg [R, n, H] float64,
    missing [n] int32, first_missing [n] int64)`` CUDA tensors: NaN where a grid point has no row, the count of such
    points per model and the first one's timestamp (INT64_MIN where there is none); rows off the grid are ignored.
    ``future_reg`` is what predict_batch_device's ``regressors=`` takes."""
    import torch
    dev = future_ds.device
    n, h = int(future_ds.shape[0]), int(future_ds.shape[1])
    R = int(tab_reg.shape[0])
    rows = int(tab_ds.shape[0])
    for t, dt, shape in ((tab_ds, torch.int64, (rows,)), (tab_reg, torch.float64, (R, rows)),
                         (model_group, torch.int64, (n,)), (future_ds, torch.int64, (n, h))):
        if t.dtype != dt or tuple(t.shape) != shape or not t.is_contiguous() or t.device != dev:
            raise ValueError(f"join_future_regressors_device wants contiguous {dt} tensors of shape {shape} on {dev}")
    offs = torch.from_numpy(np.ascontiguousarray(tab_offsets_host, dtype=np.int64)).to(dev)
    out = torch.empty((R, n, h), dtype=torch.float64, device=dev)
    missing = torch.empty(n, dtype=torch.int32, device=dev)
    first = torch.empty(n, dtype=torch.int64, device=dev)
    if n:
        torch.cuda.current_stream(dev).synchronize()
        rc = L.load().pb200_join_future_regressors_device(ctx.handle, tab_ds.data_ptr() if rows else None,
                                                          offs.data_ptr(), tab_reg.data_ptr() if rows else None, rows, R,
                                                          model_group.data_ptr(), future_ds.data_ptr(), n, h,
                                                          out.data_ptr(), missing.data_ptr(), first.data_ptr())
        L.check(rc, "pb200_join_future_regressors_device")
        ctx.synchronize()
    return out, missing, first


def forecast_csv_device(ctx: L.Context, series_id, dim_id, ds_ns, quantity, created: bytes):
    """The CSV text of forecast rows, formatted on the GPU (pb200_forecast_csv_{lengths,rows}_device): int32 / int32 /
    int64 ns / int32 CUDA tensors of equal length in, one uint8 CUDA tensor out (no header line).  Row format and the
    supported timestamp range: include/prophet_b200.h."""
    import torch
    n = int(series_id.shape[0])
    dev = series_id.device
    if n == 0:
        return torch.empty(0, dtype=torch.uint8, device=dev)
    for t, dt in ((series_id, torch.int32), (dim_id, torch.int32), (ds_ns, torch.int64), (quantity, torch.int32)):
        if t.dtype != dt or not t.is_contiguous() or int(t.shape[0]) != n or t.device != dev:
            raise ValueError("forecast_csv_device wants contiguous int32 / int32 / int64 / int32 tensors of one length on one device")
    lib = L.load()
    lens = torch.empty(n, dtype=torch.int64, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    L.check(lib.pb200_forecast_csv_lengths_device(ctx.handle, series_id.data_ptr(), dim_id.data_ptr(), quantity.data_ptr(), n,
                                                  len(created), lens.data_ptr()), "pb200_forecast_csv_lengths_device")
    ctx.synchronize()
    ends = torch.cumsum(lens, 0)                      # the scan is plumbing (torch); the two passes over the rows are the kernels
    total = int(ends[-1].item())
    offs = ends - lens
    out = torch.empty(total, dtype=torch.uint8, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    L.check(lib.pb200_forecast_csv_rows_device(ctx.handle, series_id.data_ptr(), dim_id.data_ptr(), ds_ns.data_ptr(),
                                               quantity.data_ptr(), n, created, len(created), offs.data_ptr(), out.data_ptr()),
            "pb200_forecast_csv_rows_device")
    ctx.synchronize()
    return out


def forecast_csv_row_host(series_id: int, dim_id: int, ds_ns: int, quantity: int, created: bytes) -> bytes:
    """One row through the same formatter on the host (pb200_forecast_csv_row_host; tests)."""
    import ctypes
    buf = ctypes.create_string_buffer(160)
    n = L.load().pb200_forecast_csv_row_host(int(series_id), int(dim_id), int(ds_ns), int(quantity), created, len(created), buf)
    if n < 0:
        raise ValueError("pb200_forecast_csv_row_host refused the row")
    return buf.raw[:n]


class _Args(tuple):
    """A library call's arguments.  ``keep`` holds the arrays made for the call, which its pointers point into: they
    must live until the call is made."""
    keep = ()


def _predict_head(space: _Space, ctx, opts, fitted: FittedBatch, grid, floor, cap, seed, shape, bounds: bool,
                  yint: bool = True, out: Optional["ForecastBatch"] = None):
    """What every predict entry point starts with: the arguments (handle, options, fitted's five arrays, n, the two
    ``grid`` arguments, floor, cap, seed) and the outputs it writes first, yhat, the bounds (with ``bounds``, else None)
    and (with ``yint``) yhat_int, each of ``shape``, or ``out``'s.  A host call takes ``fitted`` as contiguous numpy and
    floor / cap broadcast to one float64 per model; the arguments (an _Args) keep those arrays alive.  Returns (args,
    (yhat, lower, upper, yhat_int))."""
    n = fitted.n
    if space.dev is None:
        fitted = fitted.to_host()
        floor, cap = (np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (n,))) for v in (floor, cap))
        models = [np.ascontiguousarray(getattr(fitted, f)) for f in _FIT_FIELDS]
    else:
        models = (fitted.params, fitted.tchange, fitted.meta_i32, fitted.meta_i64, fitted.meta_f64)
    if out is not None:
        outputs = (out.yhat, out.yhat_lower, out.yhat_upper, out.yhat_int)
    else:
        outputs = (space.empty(shape, "float64"), space.empty(shape, "float64") if bounds else None,
                   space.empty(shape, "float64") if bounds else None, space.empty(shape, "int32") if yint else None)
    p = space.ptr
    args = _Args((ctx.handle, C.byref(opts), *map(p, models), n, *grid, p(floor), p(cap), int(seed) & (2**64 - 1)))
    args.keep = (models, floor, cap)
    return args, outputs


def _future_host(future_ds, n: int) -> np.ndarray:
    return np.ascontiguousarray(future_ds, dtype=np.int64).reshape(n, -1)


def _predict_regressors(space: _Space, opts, fitted: FittedBatch, regressors, components: bool, n: int, h: int):
    """The future regressor values and the fit's reg_scale a regressor predict reads: a host call's converted, a device
    call's checked."""
    if components:
        raise ValueError("components are not supported with regressors")
    R = n_regressors(opts)
    _check_reg_scale(fitted.reg_scale, n, R, "fitted.reg_scale", space.dev)
    if space.dev is None:
        return _host_regressors(opts, regressors, n * h), np.ascontiguousarray(fitted.reg_scale)
    import torch
    if (regressors.dtype != torch.float64 or regressors.numel() != R * n * h or not regressors.is_contiguous()
            or regressors.device != space.dev):
        raise ValueError(f"regressors must be a contiguous float64 tensor of shape ({R}, {n}, {h}) on {space.dev}")
    return regressors, fitted.reg_scale


def _predict(space: _Space, ctx, opts, fitted, future_ds, floor, cap, seed, intervals, components, regressors,
             out=None, sync=False) -> "ForecastBatch":
    """The body of predict_batch_host / predict_batch_device: pb200_predict[_components|_regressors]_host / _device.
    A device call synchronises torch's stream first unless it reuses ``out``, and the context after with ``sync``."""
    host = space.dev is None
    n = fitted.n
    if host:
        fitted = fitted.to_host()
        future_ds = _future_host(future_ds, n)
    h = int(future_ds.shape[1])
    do_mc = intervals and opts.uncertainty_samples > 0
    if out is not None:
        comp, tlo, thi = out.components, out.trend_lower, out.trend_upper
    else:
        comp = space.empty((len(component_names(opts)), n, h), "float64") if components else None
        tlo = space.empty((n, h), "float64") if components and do_mc else None
        thi = space.empty((n, h), "float64") if components and do_mc else None
    if host and regressors is not None:
        regressors, reg_scale = _predict_regressors(space, opts, fitted, regressors, components, n, h)
    args, (yhat, lo, hi, yint) = _predict_head(space, ctx, opts, fitted, (space.ptr(future_ds), h), floor, cap, seed,
                                               (n, h), do_mc, out=out)
    if n > 0 and h > 0:
        if out is None:
            space.sync_torch()
        p = space.ptr
        mc = p if do_mc else lambda a: None         # (``out`` may hold bounds this call does not write)
        outputs = (p(yhat), mc(lo), mc(hi), p(yint))
        if regressors is not None:
            if not host:
                regressors, reg_scale = _predict_regressors(space, opts, fitted, regressors, components, n, h)
            _call("pb200_predict_regressors" + space.suffix, *args, p(regressors), p(reg_scale), *outputs)
        elif components:
            _call("pb200_predict_components" + space.suffix, *args, *outputs, p(comp), mc(tlo), mc(thi))
        else:
            _call("pb200_predict" + space.suffix, *args, *outputs)
        if sync:
            ctx.synchronize()
    return ForecastBatch(future_ds, yhat, lo, hi, yint, comp, tlo, thi,
                         names=component_names(opts) if components else L.COMPONENTS)


def predict_batch_host(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds: np.ndarray,
                       floor: np.ndarray, cap: np.ndarray, seed: int = 0, intervals: bool = True,
                       components: bool = False, regressors=None) -> ForecastBatch:
    """pb200_predict_host.  ``floor`` / ``cap`` per model as the scorer reads them back from
    the float32 model-table columns (prophet_scorer.py:46-47,67-68).  ``components``: pb200_predict_components_host,
    which also fills ``components`` and, with intervals, ``trend_lower`` / ``trend_upper``.  ``regressors``: None, or
    for a fit with regressors their future values ``[R, N, H]`` (pb200_predict_regressors_host, with the fit's
    ``reg_scale``; not with ``components``)."""
    return _predict(_HOST, ctx, opts, fitted, future_ds, floor, cap, seed, intervals, components, regressors)


def predict_batch_device(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds, floor, cap,
                         seed: int = 0, intervals: bool = True, sync: bool = True,
                         out: Optional["ForecastBatch"] = None, components: bool = False,
                         regressors=None) -> ForecastBatch:
    """pb200_predict_device with torch CUDA tensors (``out`` reuses a previous result's buffers, which must have been
    made with the same ``components``).  ``components``: pb200_predict_components_device, as in predict_batch_host.
    ``regressors``: None, or for a fit with regressors a contiguous float64 CUDA tensor ``[R, N, H]`` of their future
    values (pb200_predict_regressors_device, with ``fitted.reg_scale``; not with ``components``)."""
    return _predict(_Space(future_ds.device), ctx, opts, fitted, future_ds, floor, cap, seed, intervals, components,
                    regressors, out=out, sync=sync)


QUANTILES_MAX = 32


def quantile_percentiles(levels) -> np.ndarray:
    """Levels (fractions in [0, 1], 1 to 32 of them, any order, repeats allowed) as the kernel's percentiles 100 q."""
    lv = np.asarray(levels, dtype=np.float64)
    if lv.ndim != 1 or not 1 <= lv.size <= QUANTILES_MAX or not np.all((lv >= 0.0) & (lv <= 1.0)):
        raise ValueError(f"levels must be 1 to {QUANTILES_MAX} fractions in [0, 1] (got {levels!r})")
    return np.ascontiguousarray(100.0 * lv)


def _quantiles(space: _Space, ctx, opts, fitted, future_ds, floor, cap, levels, seed, intervals, sync=False):
    """The body of predict_quantiles_host / predict_quantiles_device."""
    pct = quantile_percentiles(levels)
    n = fitted.n
    if space.dev is None:
        future_ds = _future_host(future_ds, n)
    h = int(future_ds.shape[1])
    p = space.ptr
    args, (yhat, lo, hi, yint) = _predict_head(space, ctx, opts, fitted, (p(future_ds), h), floor, cap, seed, (n, h),
                                               intervals)
    qs = space.empty((pct.size, n, h), "float64")
    space.sync_torch()
    _call("pb200_predict_quantiles" + space.suffix, *args, p(yhat), p(lo), p(hi), p(yint), int(pct.size), _np_ptr(pct),
          p(qs))
    if sync:
        ctx.synchronize()
    return ForecastBatch(future_ds, yhat, lo, hi, yint, quantiles=qs)


def predict_quantiles_host(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds: np.ndarray, floor, cap,
                           levels, seed: int = 0, intervals: bool = False) -> ForecastBatch:
    """pb200_predict_quantiles_host: predict_batch_host's ForecastBatch (the bounds with ``intervals``) and
    ``quantiles`` [Q, N, H], the percentile 100 q of each point's uncertainty_samples draws for each level q of
    ``levels`` (DESIGN §15).  The draws are those behind yhat_lower / yhat_upper."""
    return _quantiles(_HOST, ctx, opts, fitted, future_ds, floor, cap, levels, seed, intervals)


def predict_quantiles_device(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds, floor, cap, levels,
                             seed: int = 0, intervals: bool = False, sync: bool = True) -> ForecastBatch:
    """pb200_predict_quantiles_device with torch CUDA tensors; as predict_quantiles_host."""
    return _quantiles(_Space(future_ds.device), ctx, opts, fitted, future_ds, floor, cap, levels, seed, intervals, sync)


@dataclass
class HistoryForecast:
    """The in-sample predict of pb200_predict_history_* (DESIGN §16): one value per history row, model i's rows at
    [offsets[i], offsets[i + 1]) as in the batch that was fitted."""
    offsets: np.ndarray      # [N + 1] int64 (host)
    yhat: object             # [rows] f64
    yhat_lower: object       # [rows] f64, or None without intervals
    yhat_upper: object


def _history_offsets(offsets, n: int) -> np.ndarray:
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    if offsets.shape != (n + 1,):
        raise ValueError(f"offsets must have n_models + 1 = {n + 1} entries (got shape {offsets.shape})")
    return offsets


def _history(space: _Space, ctx, opts, fitted, ds_ns, offsets, floor, cap, seed, intervals, sync=False):
    """The body of predict_history_host / predict_history_device."""
    n = fitted.n
    offsets = _history_offsets(offsets, n)
    if space.dev is None:
        ds_ns = np.ascontiguousarray(ds_ns, dtype=np.int64)
    rows = int(offsets[-1])
    p = space.ptr
    args, (yhat, lo, hi, _) = _predict_head(space, ctx, opts, fitted, (p(ds_ns), _np_ptr(offsets)), floor, cap, seed,
                                            rows, intervals and opts.uncertainty_samples > 0, yint=False)
    if n > 0 and rows > 0:
        space.sync_torch()
        _call("pb200_predict_history" + space.suffix, *args, p(yhat), p(lo), p(hi))
        if sync:
            ctx.synchronize()
    return HistoryForecast(offsets, yhat, lo, hi)


def predict_history_host(ctx: L.Context, opts: L.Options, fitted: FittedBatch, ds_ns: np.ndarray, offsets: np.ndarray,
                         floor, cap, seed: int = 0, intervals: bool = True) -> HistoryForecast:
    """pb200_predict_history_host: fbprophet's ``m.predict()`` (no frame: the history itself) for every model of
    ``fitted`` over its rows ``[offsets[i], offsets[i + 1])`` of ``ds_ns``; ``floor`` / ``cap`` per model (the fit's:
    ``fitted.meta_f64[:, 1]`` / ``[:, 2]``).  With ``intervals`` the bounds of ``opts.interval_width`` from
    ``opts.uncertainty_samples`` draws, bit-identical to predict_batch_host on the history padded by its last timestamp."""
    return _history(_HOST, ctx, opts, fitted, ds_ns, offsets, floor, cap, seed, intervals)


def predict_history_device(ctx: L.Context, opts: L.Options, fitted: FittedBatch, ds_ns, offsets_host: np.ndarray, floor,
                           cap, seed: int = 0, intervals: bool = True, sync: bool = True) -> HistoryForecast:
    """pb200_predict_history_device: predict_history_host with torch CUDA tensors (``fitted`` on the device, ``ds_ns``
    the packed history, ``floor`` / ``cap`` float64 [N]); the offsets stay on the host."""
    return _history(_Space(ds_ns.device), ctx, opts, fitted, ds_ns, offsets_host, floor, cap, seed, intervals, sync)


@dataclass
class Outliers:
    """The rows outside their in-sample interval and the batch without them (pb200_outlier_*_device, DESIGN §16)."""
    flag: object             # [rows] uint8 CUDA: 1 where y < lower or y > upper
    kept: np.ndarray         # [N] int64 (host): rows kept per series
    offsets: np.ndarray      # [N + 1] int64 (host): the kept batch's offsets, for fit_batch_device
    ds: object               # [offsets[-1]] int64 CUDA: the kept rows in their order
    y: object                # [offsets[-1]] CUDA, y's dtype


def outliers_device(ctx: L.Context, ds_ns, y, offsets_host: np.ndarray, lower, upper) -> Outliers:
    """Flags each row whose y lies outside ``[lower, upper]`` (a NaN bound never flags) and packs the other rows into a
    batch that ``fit_batch_device`` takes as it is.  Counts, scan, rows: the kept counts are the only device-to-host
    copy, for the host offsets of the new batch; ds / y never leave the device."""
    import torch
    offsets_host = np.ascontiguousarray(offsets_host, dtype=np.int64)
    n = offsets_host.size - 1
    rows = int(offsets_host[-1])
    dev = ds_ns.device
    for t, what in ((lower, "lower"), (upper, "upper")):
        if t.dtype != torch.float64 or not t.is_contiguous() or t.device != dev or int(t.numel()) < rows:
            raise ValueError(f"{what} must be a contiguous float64 tensor of at least {rows} rows on {dev}")
    lib = L.load()
    ydt = _y_dtype(y)
    flag = torch.empty(rows, dtype=torch.uint8, device=dev)
    kept = torch.empty(n, dtype=torch.int32, device=dev)
    d_off = torch.from_numpy(offsets_host).to(dev)
    if n > 0:
        torch.cuda.current_stream(dev).synchronize()
        L.check(lib.pb200_outlier_counts_device(ctx.handle, y.data_ptr(), ydt, d_off.data_ptr(), n, lower.data_ptr(),
                                                upper.data_ptr(), flag.data_ptr(), kept.data_ptr()),
                "pb200_outlier_counts_device")
        ctx.synchronize()
    kept_h = kept.cpu().numpy().astype(np.int64)
    new_off = np.zeros(n + 1, np.int64)
    np.cumsum(kept_h, out=new_off[1:])
    total = int(new_off[-1])
    ds_out = torch.empty(total, dtype=torch.int64, device=dev)
    y_out = torch.empty(total, dtype=y.dtype, device=dev)
    if total > 0:
        d_kept_off = torch.from_numpy(new_off).to(dev)
        torch.cuda.current_stream(dev).synchronize()
        L.check(lib.pb200_outlier_compact_device(ctx.handle, ds_ns.data_ptr(), y.data_ptr(), ydt, d_off.data_ptr(), n,
                                                 flag.data_ptr(), d_kept_off.data_ptr(), ds_out.data_ptr(),
                                                 y_out.data_ptr()),
                "pb200_outlier_compact_device")
        ctx.synchronize()
    return Outliers(flag, kept_h, new_off, ds_out, y_out)


@dataclass
class WindowSums:
    """Forecast totals over fixed-width time windows (pb200_predict_sums_*) or calendar periods
    (pb200_predict_period_sums_*), each [N, wmax]; slots at or past a model's ``n_windows`` hold INT64_MIN / 0 / NaN."""
    n_windows: object     # [N] int32
    start: object         # int64 ns: origin + window index * width, or the period's start
    points: object        # int32: frame points in the window
    yhat_sum: object      # f64: yhat summed in frame order
    quantity_sum: object  # int64: yhat_int summed
    lower: object         # f64: percentiles over the draws' window sums
    upper: object


@dataclass
class WindowQuantiles(WindowSums):
    """WindowSums plus the quantiles of each window's total at ``levels`` (DESIGN §21): the predict_*sums_* wrappers'
    second result when called with ``levels``."""
    levels: np.ndarray    # [Q] f64 fractions, as given
    quantiles: object     # [Q, N, wmax] f64: percentile 100 q over the draws' window sums; NaN past n_windows


def window_slots(first_ds, last_ds, width_ns: int, origin_ns: int) -> int:
    """An upper bound on a model's windows from the first and last column of an ascending frame:
    max_i (w(last_i) - w(first_i) + 1), w = floor((ds - origin) / width).  Exact when the grid is no coarser than the
    width; windows that hold no point take no slot."""
    if len(first_ds) == 0:
        return 1
    return int(((last_ds - origin_ns) // width_ns - (first_ds - origin_ns) // width_ns).max()) + 1


def _check_window_slots(wmax: int, n_windows_max: int) -> None:
    if n_windows_max > wmax:
        raise ValueError(f"a model has {n_windows_max} windows, more than the {wmax} slots sized from the frame's first and "
                         "last columns: is every model's future frame ascending?")


def _period_rule_checked(months: int, month_shift: int):
    months, month_shift = int(months), int(month_shift)
    if months not in (1, 3, 12) or not 0 <= month_shift < months:
        raise ValueError(f"months must be 1, 3 or 12 and month_shift in [0, months) (got {months}, {month_shift})")
    return months, month_shift


def periods_host(ds, months: int, month_shift: int):
    """pb200_period_host: the calendar period of each timestamp (int64 ns) under (months, month_shift) and the period's
    start, computed by the functions the calendar kernel runs.  Returns (period, start), int64 arrays of ds's shape."""
    months, month_shift = _period_rule_checked(months, month_shift)
    ds = np.ascontiguousarray(ds, dtype=np.int64)
    period = np.empty(ds.shape, np.int64)
    start = np.empty(ds.shape, np.int64)
    L.check(L.load().pb200_period_host(_np_ptr(ds), ds.size, months, month_shift, _np_ptr(period), _np_ptr(start)),
            "pb200_period_host")
    return period, start


def period_slots(first_ds, last_ds, months: int, month_shift: int) -> int:
    """window_slots for calendar periods: max_i (p(last_i) - p(first_i) + 1).  Refuses, with a ValueError, a frame whose
    first point's period starts before the int64-ns minimum (1677-09-21), where its start is not representable."""
    first_ds = np.asarray(first_ds, np.int64)
    if first_ds.size == 0:
        return 1
    p0, s0 = periods_host(first_ds, months, month_shift)
    bad = np.flatnonzero(s0 > first_ds)         # the start wrapped: it lies before the int64-ns minimum
    if bad.size:
        raise ValueError(f"the period of {int(first_ds[bad[0]])} ns starts before the earliest representable timestamp "
                         "(1677-09-21): no window_start can be written for it")
    p1, _ = periods_host(last_ds, months, month_shift)
    return int((p1 - p0).max()) + 1


def _window_sums(space: _Space, ctx, opts, fitted, future_ds, floor, cap, seed, intervals, entry: str, rule, wmax,
                 levels=None):
    """The body of the predict_*sums_* wrappers: ``entry`` the C function without its suffix, ``rule`` its arguments
    between yhat_int and wmax, ``wmax`` the slots per model or a function ``slots(first_ds, last_ds)`` of the frame's
    first and last columns (numpy) that gives them.  ``levels``: the ``entry``_quantiles twin, whose planes make the
    result a WindowQuantiles.  A device call always synchronises the context."""
    pct = quantile_percentiles(levels) if levels is not None else None
    n = fitted.n
    if space.dev is None:
        future_ds = np.ascontiguousarray(future_ds, dtype=np.int64)
        future_ds = future_ds.reshape(n, -1) if n else future_ds.reshape(0, future_ds.shape[-1] if future_ds.ndim == 2 else 0)
    h = int(future_ds.shape[1])
    if callable(wmax):
        slots, wmax = wmax, 1
        if n and h:
            ends = future_ds[:, [0, -1]]
            ends = ends if space.dev is None else ends.cpu().numpy()
            wmax = slots(ends[:, 0], ends[:, 1])
    p = space.ptr
    args, (yhat, lo, hi, yint) = _predict_head(space, ctx, opts, fitted, (p(future_ds), h), floor, cap, seed, (n, h),
                                               intervals)
    ws = WindowSums(space.zeros(n, "int32"), *(space.empty((n, wmax), dt) for dt in
                                              ("int64", "int32", "float64", "int64", "float64", "float64")))
    quant = ()
    if pct is not None:
        ws = WindowQuantiles(*(getattr(ws, f.name) for f in fields(WindowSums)),
                             np.asarray(levels, dtype=np.float64), space.empty((pct.size, n, wmax), "float64"))
        entry += "_quantiles"
        quant = (int(pct.size), _np_ptr(pct), p(ws.quantiles))
    space.sync_torch()
    _call(entry + space.suffix, *args, p(yhat), p(lo), p(hi), p(yint), *rule, wmax,
          *(p(a) for a in (ws.n_windows, ws.start, ws.points, ws.yhat_sum, ws.quantity_sum, ws.lower, ws.upper)), *quant)
    if space.dev is not None:
        ctx.synchronize()
    _check_window_slots(wmax, int(ws.n_windows.max()) if n else 0)
    return ForecastBatch(future_ds, yhat, lo, hi, yint), ws


def predict_sums_host(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds: np.ndarray, floor: np.ndarray,
                      cap: np.ndarray, width_ns: int, origin_ns: int = 0, seed: int = 0, intervals: bool = False,
                      levels=None):
    """pb200_predict_sums_host: predict_batch_host's ForecastBatch and the WindowSums of the windows
    floor((ds - origin_ns) / width_ns) of each model's ascending frame -- totals of yhat / yhat_int per window and the
    interval of each total from the joint draws (fbprophet's predictive_samples summed per window).  Needs
    ``opts.uncertainty_samples`` in [2, 1024]; ``intervals`` asks for the pointwise yhat_lower / yhat_upper as well.
    ``levels`` (1 to 32 fractions in [0, 1], any order): pb200_predict_sums_quantiles_host, which returns a
    WindowQuantiles with each window total's quantiles at those levels from the same draws (DESIGN §21); every other
    output is the same."""
    return _fixed_sums(_HOST, ctx, opts, fitted, future_ds, floor, cap, width_ns, origin_ns, seed, intervals, levels)


def predict_period_sums_host(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds: np.ndarray, floor, cap,
                             months: int, month_shift: int, seed: int = 0, intervals: bool = False, levels=None):
    """pb200_predict_period_sums_host: predict_sums_host over calendar periods (DESIGN §17) -- the windows are the
    periods floor((mi + month_shift) / months) of each model's ascending frame, mi the months of ds's civil date since
    1970-01, and ``WindowSums.start`` holds each period's start.  ``period_rule`` turns a pandas alias into the rule.
    ``levels``: pb200_predict_period_sums_quantiles_host, as in predict_sums_host."""
    return _period_sums(_HOST, ctx, opts, fitted, future_ds, floor, cap, months, month_shift, seed, intervals, levels)


def _fixed_sums(space, ctx, opts, fitted, future_ds, floor, cap, width_ns, origin_ns, seed, intervals, levels=None):
    width_ns, origin_ns = int(width_ns), int(origin_ns)
    if width_ns <= 0:
        raise ValueError(f"width_ns must be > 0 (got {width_ns})")
    return _window_sums(space, ctx, opts, fitted, future_ds, floor, cap, seed, intervals, "pb200_predict_sums",
                        (width_ns, origin_ns), lambda a, b: window_slots(a, b, width_ns, origin_ns), levels)


def _period_sums(space, ctx, opts, fitted, future_ds, floor, cap, months, month_shift, seed, intervals, levels=None):
    months, month_shift = _period_rule_checked(months, month_shift)
    return _window_sums(space, ctx, opts, fitted, future_ds, floor, cap, seed, intervals, "pb200_predict_period_sums",
                        (months, month_shift), lambda a, b: period_slots(a, b, months, month_shift), levels)


def predict_sums_device(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds, floor, cap, width_ns: int,
                        origin_ns: int = 0, seed: int = 0, intervals: bool = False, levels=None):
    """pb200_predict_sums_device with torch CUDA tensors; as predict_sums_host (``levels``:
    pb200_predict_sums_quantiles_device)."""
    return _fixed_sums(_Space(future_ds.device), ctx, opts, fitted, future_ds, floor, cap, width_ns, origin_ns, seed,
                       intervals, levels)


def predict_period_sums_device(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds, floor, cap, months: int,
                               month_shift: int, seed: int = 0, intervals: bool = False, levels=None):
    """pb200_predict_period_sums_device with torch CUDA tensors; as predict_period_sums_host (``levels``:
    pb200_predict_period_sums_quantiles_device)."""
    return _period_sums(_Space(future_ds.device), ctx, opts, fitted, future_ds, floor, cap, months, month_shift, seed,
                        intervals, levels)


_MONTHS = ("JAN", "FEB", "MAR", "APR", "MAY", "JUN", "JUL", "AUG", "SEP", "OCT", "NOV", "DEC")
_WEEKDAYS = ("MON", "TUE", "WED", "THU", "FRI", "SAT", "SUN")


def period_rule(alias: str):
    """A pandas period alias as a window rule (DESIGN §17): ``("months", months, shift)`` for 'M', 'Q', 'Q-<MON>', 'Y'
    and 'Y-<MON>' (the periods of predict_period_sums_*), ``("fixed", width_ns, origin_ns)`` for 'W' and 'W-<DAY>' (a
    week is the fixed rule 7D whose origin is the day after <DAY>: W-SUN weeks start on Monday, origin 1970-01-05).
    Anything else -- 'D', 'h', '7D', 'MS', 'QS', 'A', 'B', multiples such as '2M' -- is refused with a ValueError."""
    import re
    m = re.fullmatch(r"([A-Z])(?:-([A-Z]{3}))?", alias) if isinstance(alias, str) else None
    kind, anchor = (m.group(1), m.group(2)) if m else (None, None)
    if kind == "W" and (anchor is None or anchor in _WEEKDAYS):
        d = _WEEKDAYS.index(anchor or "SUN")
        return "fixed", 7 * 86400 * 10**9, ((d + 1 - 3) % 7) * 86400 * 10**9     # 1970-01-01 was a Thursday (3)
    if kind == "M" and anchor is None:
        return "months", 1, 0
    if kind in ("Q", "Y") and (anchor is None or anchor in _MONTHS):
        months = 3 if kind == "Q" else 12
        end = _MONTHS.index(anchor or "DEC") + 1
        return "months", months, (12 - end) % months
    raise ValueError(f"{alias!r} is not a period alias: use 'W', 'W-<DAY>', 'M', 'Q', 'Q-<MON>', 'Y' or 'Y-<MON>'")


def predict_sums_anchored_device(ctx: L.Context, opts: L.Options, fitted: FittedBatch, future_ds, floor, cap,
                                 width_ns: int, origins, frame_len, seed: int = 0, intervals: bool = False,
                                 wmax: Optional[int] = None, levels=None):
    """pb200_predict_sums_anchored_device with torch CUDA tensors: predict_sums_device with a window origin per model
    (``origins`` int64 [N]) whose windows cover only the first ``frame_len[i]`` points of row i (int32 [N]; the rest
    of the row is padding that is predicted but summed into no window).  ``wmax`` defaults to the bound
    ``window_slots`` gives over each model's first and last walked point.  ``levels``:
    pb200_predict_sums_anchored_quantiles_device, as in predict_sums_host."""
    import torch
    n = fitted.n
    h = int(future_ds.shape[1])
    dev = future_ds.device
    width_ns = int(width_ns)
    if width_ns <= 0:
        raise ValueError(f"width_ns must be > 0 (got {width_ns})")
    origins = origins.to(device=dev, dtype=torch.int64).contiguous()
    frame_len = frame_len.to(device=dev, dtype=torch.int32).contiguous()
    if wmax is None:
        wmax = 1
        if n and h:
            last = future_ds.gather(1, (frame_len.long().clamp(1, h) - 1)[:, None])[:, 0]
            w = (last - origins).div(width_ns, rounding_mode="floor") - (future_ds[:, 0] - origins).div(width_ns, rounding_mode="floor")
            wmax = max(1, int(w.max().item()) + 1)
    return _window_sums(_Space(dev), ctx, opts, fitted, future_ds, floor, cap, seed, intervals,
                        "pb200_predict_sums_anchored", (width_ns, origins.data_ptr(), frame_len.data_ptr()), int(wmax),
                        levels)


def objective_host(ctx: L.Context, opts: L.Options, ds_ns: np.ndarray, y: np.ndarray, offsets: np.ndarray,
                   floor: float, cap_multiplier: float, theta: np.ndarray, regressors=None):
    """pb200_objective_host (parity-test hook): objective and gradient at ``theta`` rows
    (Stan unconstrained order k, m, delta[S], log sigma, beta[K], zero-padded to pstride).  ``regressors``: None, or
    their values ``[R, n_rows]`` (pb200_objective_regressors_host: beta[K] is then the seasonal columns followed by the
    R regressors); the standardisation used, ``[n, R, 2]``, is returned as a fourth value."""
    ds_ns = np.ascontiguousarray(ds_ns, dtype=np.int64)
    y = np.ascontiguousarray(y)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    n = offsets.size - 1
    lay = L.get_layout(opts)
    th = np.zeros((n, lay.pstride), np.float64)
    th[:, :theta.shape[1]] = theta
    f = np.empty(n, np.float64)
    g = np.empty((n, lay.pstride), np.float64)
    mi32 = np.empty((n, 8), np.int32)
    reg = rsc = None
    if regressors is not None:
        reg = _host_regressors(opts, regressors, ds_ns.size)
        rsc = np.empty((n, reg.shape[0], 2), np.float64)
    args = (ctx.handle, C.byref(opts), _np_ptr(ds_ns), _np_ptr(y), _y_dtype(y), _np_ptr(offsets), n, float(floor),
            float(cap_multiplier))
    outputs = (_np_ptr(th), _np_ptr(f), _np_ptr(g), _np_ptr(mi32))
    if reg is None:
        _call("pb200_objective_host", *args, *outputs)
        return f, g, mi32
    _call("pb200_objective_regressors_host", *args, _np_ptr(reg), _np_ptr(rsc), *outputs)
    return f, g, mi32, rsc


# ---------------------------------------------------------------------------------------------------------------------
# Backtest: fbprophet.diagnostics.cross_validation / performance_metrics for every series of a batch (DESIGN §9)
# ---------------------------------------------------------------------------------------------------------------------
# Rows (history prefixes plus held-out windows) gathered per chunk.  50k series x 22 cutoffs of ~840 history rows are
# ~1e9 rows (~11 GB with int32 y); chunks of whole series keep the gathered batch and the fit outputs bounded.
CV_ROW_BUDGET = 1 << 27


@dataclass
class CvPlan:
    """Per series (host numpy): cutoff count, full-history seasonality mask, error bits (L.CV_ERR_*), and the
    exclusive scan of the counts; per (series, cutoff) pair (CUDA tensors, cutoffs ascending within a series): series
    index, cutoff ns, first row > cutoff (``hist_end``) and first row > cutoff + horizon (``win_end``), absolute rows."""
    n_cutoffs: np.ndarray
    mask: np.ndarray
    err: np.ndarray
    pair_off: np.ndarray
    pair_series: object
    cutoff: object
    hist_end: object
    win_end: object

    @property
    def n_pairs(self) -> int:
        return int(self.pair_off[-1])


def cv_plan_device(ctx: L.Context, opts: L.Options, ds_ns, offsets_host: np.ndarray, horizon_ns: int, period_ns: int,
                   initial_ns: int) -> CvPlan:
    """pb200_cv_plan_counts_device, the scan, pb200_cv_plan_device: generate_cutoffs for every series of a packed batch
    (``ds_ns`` a CUDA int64 tensor sorted within each series)."""
    import torch
    offsets_host = np.ascontiguousarray(offsets_host, dtype=np.int64)
    n = offsets_host.size - 1
    dev = ds_ns.device
    lib = L.load()
    d_off = torch.from_numpy(offsets_host).to(dev)
    n_cut = torch.zeros(n, dtype=torch.int32, device=dev)
    mask = torch.zeros(n, dtype=torch.int32, device=dev)
    err = torch.zeros(n, dtype=torch.int32, device=dev)
    torch.cuda.current_stream(dev).synchronize()
    L.check(lib.pb200_cv_plan_counts_device(ctx.handle, C.byref(opts), ds_ns.data_ptr(), d_off.data_ptr(), n, int(horizon_ns),
                                            int(period_ns), int(initial_ns), n_cut.data_ptr(), mask.data_ptr(), err.data_ptr()),
            "pb200_cv_plan_counts_device")
    ctx.synchronize()
    counts = n_cut.cpu().numpy()
    pair_off = np.zeros(n + 1, np.int64)
    np.cumsum(counts, out=pair_off[1:])
    p = int(pair_off[-1])
    ps = torch.empty(p, dtype=torch.int32, device=dev)
    cut, he, we = (torch.empty(p, dtype=torch.int64, device=dev) for _ in range(3))
    if p:                  # with no cutoff anywhere there is nothing to write (and the error bits are complete)
        d_poff = torch.from_numpy(pair_off).to(dev)
        torch.cuda.current_stream(dev).synchronize()
        L.check(lib.pb200_cv_plan_device(ctx.handle, C.byref(opts), ds_ns.data_ptr(), d_off.data_ptr(), n, int(horizon_ns),
                                         int(period_ns), int(initial_ns), d_poff.data_ptr(), err.data_ptr(), ps.data_ptr(),
                                         cut.data_ptr(), he.data_ptr(), we.data_ptr()), "pb200_cv_plan_device")
        ctx.synchronize()
    return CvPlan(counts, mask.cpu().numpy(), err.cpu().numpy(), pair_off, ps, cut, he, we)


def plan_options(opts):
    """The options cv_plan_device takes for ``opts``: the plan reads the seasonalities only, so options with regressors
    give their pb200_options_v2 part (version 2, the same table); any other options are returned as they are."""
    if not n_regressors(opts):
        return opts
    o = L.OptionsV2.from_buffer_copy(opts)
    o.abi_version = L.ABI_VERSION_TABLE
    o._source = opts        # keeps the table entries alive as long as the copy
    return o


def cv_plan_errors(plan: CvPlan):
    """(message, per-series bool mask) of the first kind of plan error present, or None: fbprophet's exceptions."""
    for bit, msg in ((L.CV_ERR_HORIZON, "Less data than horizon."),
                     (L.CV_ERR_INITIAL, "Less data than horizon after initial window. Make horizon or initial shorter."),
                     (L.CV_ERR_FEW, "Less than two datapoints before cutoff. Increase initial window.")):
        bad = (plan.err & bit) != 0
        if bad.any():
            return msg, bad
    return None


def _with_mask(opts: L.Options, mask: int) -> L.Options:
    """The options of a cutoff fit: the full model's, seasonalities forced to the full history's auto mask (fbprophet
    0.5's prophet_copy, which gives the copy the fitted model's seasonalities and turns the built-in switches off).  For
    a seasonality table the cutoff fit keeps every custom entry and the orders; a built-in is forced on or off by the
    mask only where no custom entry carries its name -- such an entry replaces the built-in, whose switch must stay
    AUTO."""
    o = copy_options(opts)
    custom = set()
    if _has_table(opts):
        custom = {opts.seasonalities[i].name.decode() for i in range(opts.n_seasonalities)}
    for name, bit, _, _ in _BUILTINS:
        if name not in custom:
            setattr(o, name, int(mask & bit != 0))
    return o


@dataclass
class CvResult:
    """Output of cross_validation_device (host numpy).

    Pairs, in plan order (series ascending, cutoffs ascending): ``pair_series``, ``pair_cutoff``, ``pair_status`` (the
    cutoff fit's solver status; < 0: failed), ``pair_mask`` (the built-in seasonality mask it was fitted with; with a
    seasonality table the kept fits' meta_i32[:, 3] holds the table mask of ``opts``).
    Held-out rows, ordered by (series, cutoff, ds): ``row_series``, ``ds``, ``cutoff``, ``y`` (float64 of the input
    value), ``yhat`` and, with intervals, ``yhat_lower`` / ``yhat_upper``.
    Metrics rows (when requested), ordered by (series, horizon): ``m_series``, ``horizon`` (ns), ``mse``, ``rmse``,
    ``mae``, ``mape``, ``coverage`` (None without intervals).
    ``fitted``: with ``keep_fits``, the cutoff fits in plan order, each record in the layout of ``opts`` (beta packed
    by its mask, zero beyond); with regressors its ``reg_scale`` is each cutoff fit's (mu, std).
    With a ``grid`` of n_grid prior-scale pairs every series index above is a virtual one, ``s * n_grid + g`` for series
    ``s`` fitted with grid point ``g``, and "plan order" is (series, grid point, cutoff)."""
    pair_series: np.ndarray
    pair_cutoff: np.ndarray
    pair_status: np.ndarray
    pair_mask: np.ndarray
    row_series: np.ndarray
    ds: np.ndarray
    cutoff: np.ndarray
    y: np.ndarray
    yhat: np.ndarray
    yhat_lower: Optional[np.ndarray]
    yhat_upper: Optional[np.ndarray]
    metrics: Optional[dict] = None
    fitted: Optional[FittedBatch] = None
    windows: Optional["CvWindows"] = None
    yhat_q: Optional[np.ndarray] = None           # [Q, rows] held-out quantiles (quantiles=levels)
    quantile_metrics: Optional[dict] = None       # quantile_metrics_device's columns (quantiles with rolling_window)


@dataclass
class CvWindows:
    """Window rows of cross_validation_device(aggregate_ns=W) (DESIGN §14), host numpy, ordered by (series, cutoff,
    window).  Window j of cutoff c is (c + j W, c + (j + 1) W]; only windows holding a held-out row have a row.
    ``series`` (as CvResult.row_series), ``cutoff``, ``horizon`` ((j + 1) W, ns), ``points`` (held-out rows in the
    window), ``y`` / ``yhat`` (their float64 y / yhat summed in row order) and, with intervals, ``yhat_lower`` /
    ``yhat_upper`` (percentiles over the joint draws' window sums).  ``metrics`` (with ``rolling_window``):
    performance_metrics over the window rows with ``horizon`` as the horizon, keyed as CvResult.metrics.
    With ``window_quantiles`` (DESIGN §21): ``yhat_q`` [Q, rows], the quantiles of each window's total at those levels
    from the same draws, and (with ``rolling_window``) ``quantile_metrics``, quantile_metrics_device over the window
    rows with ``horizon`` as the horizon."""
    width_ns: int
    series: np.ndarray
    cutoff: np.ndarray
    horizon: np.ndarray
    points: np.ndarray
    y: np.ndarray
    yhat: np.ndarray
    yhat_lower: Optional[np.ndarray]
    yhat_upper: Optional[np.ndarray]
    metrics: Optional[dict] = None
    yhat_q: Optional[np.ndarray] = None
    quantile_metrics: Optional[dict] = None


def cv_windows_device(ctx: L.Context, ds_ns, y, plan: CvPlan, pairs, yhat, width_ns: int, wmax: Optional[int] = None):
    """pb200_cv_windows_device: the window totals (DESIGN §14) of the gathered entries ``pairs`` (int64 CUDA tensor of
    plan pairs) over the original ``ds_ns`` / ``y`` and the predict frame ``yhat`` [len(pairs), hmax] of those entries.
    Returns CUDA tensors n_windows [n] and, [n, wmax], start (cutoff + j W), points, y_sum, yhat_sum.  ``wmax``
    defaults to the entries' largest held-out row count (a pair has no more windows than held-out rows)."""
    import torch
    dev = yhat.device
    n, hmax = int(yhat.shape[0]), int(yhat.shape[1])
    width_ns = int(width_ns)
    if width_ns <= 0:
        raise ValueError(f"width_ns must be > 0 (got {width_ns})")
    pairs = pairs.to(device=dev, dtype=torch.int64).contiguous()
    if wmax is None:
        wmax = max(1, int((plan.win_end[pairs] - plan.hist_end[pairs]).max().item())) if n else 1
    wmax = int(wmax)
    out = {"n_windows": torch.zeros(n, dtype=torch.int32, device=dev),
           "start": torch.empty((n, wmax), dtype=torch.int64, device=dev),
           "points": torch.empty((n, wmax), dtype=torch.int32, device=dev),
           "y_sum": torch.empty((n, wmax), dtype=torch.float64, device=dev),
           "yhat_sum": torch.empty((n, wmax), dtype=torch.float64, device=dev)}
    if n:
        yh = yhat.contiguous()
        torch.cuda.current_stream(dev).synchronize()
        L.check(L.load().pb200_cv_windows_device(
            ctx.handle, ds_ns.data_ptr(), y.data_ptr(), _y_dtype(y), plan.cutoff.data_ptr(), plan.hist_end.data_ptr(),
            plan.win_end.data_ptr(), pairs.data_ptr(), n, yh.data_ptr(), hmax, width_ns, wmax,
            out["n_windows"].data_ptr(), out["start"].data_ptr(), out["points"].data_ptr(), out["y_sum"].data_ptr(),
            out["yhat_sum"].data_ptr()), "pb200_cv_windows_device")
        ctx.synchronize()
        _check_window_slots(wmax, int(out["n_windows"].max().item()))
    return out


def _cv_chunks(plan: CvPlan, offsets_host: np.ndarray, budget: int, n_grid: int = 1):
    """Series ranges [s0, s1) whose gathered rows (history prefixes + held-out windows, once per grid point) stay within
    ``budget``; a series is never split (its metrics need all of its rows)."""
    he = plan.hist_end.cpu().numpy()
    we = plan.win_end.cpu().numpy()
    ps = np.repeat(np.arange(plan.n_cutoffs.size), plan.n_cutoffs)
    per_pair = (he - offsets_host[:-1][ps]) + (we - he)
    per_series = np.zeros(plan.n_cutoffs.size, np.int64)
    np.add.at(per_series, ps, per_pair)
    per_series *= n_grid
    out, s0, acc = [], 0, 0
    for s in range(per_series.size):
        if acc and acc + per_series[s] > budget:
            out.append((s0, s))
            s0, acc = s, 0
        acc += int(per_series[s])
    if s0 < per_series.size:
        out.append((s0, per_series.size))
    return out, he, we


def _cv_entries(plan: CvPlan, s0: int, s1: int, n_grid: int):
    """The cutoff fits of series [s0, s1) under ``n_grid`` grid points, in plan order (series, grid point, cutoff): the
    plan pair, the series and the grid point of each."""
    vs = np.repeat(np.arange(s0, s1), n_grid)                 # (series, grid point) -> series
    vg = np.tile(np.arange(n_grid), s1 - s0)
    vn = np.repeat(plan.n_cutoffs[s0:s1].astype(np.int64), n_grid)
    e = np.repeat(np.arange(vs.size), vn)
    voff = np.zeros(vs.size + 1, np.int64)
    np.cumsum(vn, out=voff[1:])
    series = vs[e]
    return plan.pair_off[series] + (np.arange(int(voff[-1])) - voff[:-1][e]), series, vg[e]


def cross_validation_device(ctx: L.Context, opts: L.Options, ds_ns, y, offsets_host: np.ndarray, floor: float, cap,
                            horizon_ns: int, period_ns: int, initial_ns: int, intervals: bool = False, seed: int = 0,
                            rolling_window: Optional[float] = None, plan: Optional[CvPlan] = None,
                            keep_fits: bool = False, timings: Optional[dict] = None,
                            _row_budget: Optional[int] = None, grid=None,
                            aggregate_ns: Optional[int] = None, quantiles=None, regressors=None,
                            window_quantiles=None) -> CvResult:
    """fbprophet.diagnostics.cross_validation (and, with ``rolling_window``, performance_metrics) for every series of a
    packed batch: ``ds_ns`` / ``y`` CUDA tensors sorted within each series, ``cap`` the float64 CUDA tensor of each
    series' full-history cap.  Per chunk of series: one gather, one pb200_fit_device per full-history seasonality mask
    class, one predict, and the metrics kernel.  Plan errors raise ValueError (see ``cv_plan_errors``).  ``timings``
    (a dict) accumulates seconds per stage -- plan, gather, fit, predict, metrics, each ending in a synchronisation.
    ``grid``: a list of (changepoint_prior_scale, seasonality_prior_scale) pairs.  Every cutoff fit is then made once per
    pair, in the same fit calls (each entry with its own prior scales), and the result's series are the virtual
    ``s * n_grid + g`` (see CvResult): one backtest per grid point for the price of one batch.
    ``quantiles`` (levels, fractions in [0, 1]): the chunk's predict is pb200_predict_quantiles_device, whose pointwise
    outputs are pb200_predict_device's; ``CvResult.yhat_q`` holds each held-out row's quantiles and, with
    ``rolling_window``, ``CvResult.quantile_metrics`` their calibration by horizon (stage ``quantile_metrics``, DESIGN
    §15).  It does not combine with ``aggregate_ns`` or ``grid``.
    ``aggregate_ns`` (a width W dividing ``horizon_ns``): also the held-out totals per window (c + j W, c + (j + 1) W]
    after each cutoff c, with their metrics, as ``CvResult.windows`` (DESIGN §14).  Every other output is unchanged.
    With intervals the chunk's predict is pb200_predict_sums_anchored_device, whose pointwise outputs are
    pb200_predict_device's; the window totals are pb200_cv_windows_device's (stages ``windows`` and
    ``window_metrics``).
    ``window_quantiles`` (levels, fractions in [0, 1]; needs ``aggregate_ns``, ``intervals`` and uncertainty_samples
    > 0): that anchored call is pb200_predict_sums_anchored_quantiles_device, whose other outputs are the same, and
    ``CvWindows.yhat_q`` / ``CvWindows.quantile_metrics`` hold the totals' quantiles and, with ``rolling_window``,
    their calibration by horizon (stage ``window_quantile_metrics``, DESIGN §21).
    ``regressors`` (for options with regressors, required with them): a contiguous float64 CUDA tensor ``[R, rows]``
    aligned with ``ds_ns``.  fbprophet 0.5's cross_validation with prophet_copy (DESIGN §20): the full histories' (mu,
    std) by pb200_regressor_scales_device (a non-finite value raises ValueError), the cutoff fits on z = (x - mu_full) /
    std_full gathered by pb200_cv_gather_regressors_device and fitted with those scales as their copy
    (pb200_fit_regressors_copy_device), the held-out rows' z predicted with each cutoff fit's own (mu, std).  The plan
    is made with ``plan_options(opts)``; ``CvResult.fitted`` carries ``reg_scale``.  Not with ``grid``,
    ``aggregate_ns`` or ``quantiles``."""
    import time
    import torch
    tm = timings if timings is not None else {}
    clock = [time.perf_counter()]

    def lap(stage):
        t = time.perf_counter()
        tm[stage] = tm.get(stage, 0.0) + t - clock[0]
        clock[0] = t
    offsets_host = np.ascontiguousarray(offsets_host, dtype=np.int64)
    dev = ds_ns.device
    R = n_regressors(opts)
    if (regressors is None) != (R == 0):
        raise ValueError("regressors= is required with options that have regressors, and taken only with them")
    if R and (grid is not None or aggregate_ns is not None or quantiles is not None):
        raise ValueError("grid, aggregate_ns and quantiles are not supported with regressors")
    wlevels = None
    if window_quantiles is not None:
        if aggregate_ns is None or not intervals or opts.uncertainty_samples <= 0:
            raise ValueError("window_quantiles need aggregate_ns, intervals and uncertainty_samples > 0")
        wlevels = np.asarray(window_quantiles, dtype=np.float64)
        quantile_percentiles(wlevels)
    if plan is None:
        plan = cv_plan_device(ctx, plan_options(opts), ds_ns, offsets_host, horizon_ns, period_ns, initial_ns)
        lap("plan")
    bad = cv_plan_errors(plan)
    if bad is not None:
        raise ValueError(f"{bad[0]} (first offender: series {int(np.flatnonzero(bad[1])[0])}; "
                         f"{int(bad[1].sum())} series in all)")
    lib = L.load()
    lay = L.get_layout(opts)
    table = seasonality_table(opts)
    ydt = _y_dtype(y)
    d_off = torch.from_numpy(offsets_host).to(dev)
    n_grid, grid_h = 1, None
    if grid is not None:
        grid_h = np.ascontiguousarray(np.asarray(grid, dtype=np.float64))
        if grid_h.ndim != 2 or grid_h.shape[1] != 2 or grid_h.shape[0] == 0:
            raise ValueError("grid must be a non-empty list of (changepoint_prior_scale, seasonality_prior_scale) pairs")
        n_grid = grid_h.shape[0]
    W = None
    if aggregate_ns is not None:
        W = int(aggregate_ns)
        if W <= 0 or int(horizon_ns) % W != 0:
            raise ValueError(f"aggregate_ns must be a positive width that divides the horizon (got {aggregate_ns!r} for "
                             f"a horizon of {int(horizon_ns)} ns)")
    sums = W is not None and intervals and opts.uncertainty_samples > 0
    levels = None
    if quantiles is not None:
        if W is not None or grid is not None:
            raise ValueError("quantiles do not combine with aggregate_ns or grid")
        levels = np.asarray(quantiles, dtype=np.float64)
        quantile_percentiles(levels)
    if R:
        rows_all = int(offsets_host[-1])
        if (regressors.dtype != torch.float64 or tuple(regressors.shape) != (R, rows_all)
                or not regressors.is_contiguous() or regressors.device != dev):
            raise ValueError(f"regressors must be a contiguous float64 tensor of shape ({R}, {rows_all}) on {dev}")
        scale_full, bad_reg = regressor_scales_device(ctx, opts, regressors, offsets_host)
        bad_h = bad_reg.cpu().numpy()
        if bad_h.any():
            i = int(np.flatnonzero(bad_h)[0])
            r = int(torch.nonzero(torch.isnan(scale_full[i, :, 0]))[0, 0])
            raise ValueError(f"Found NaN in column {opts.regressors[r].name.decode()} (first offender: series {i}; "
                             f"{int(bad_h.sum())} series in all)")
        lap("scales")
    chunks, he_h, we_h = _cv_chunks(plan, offsets_host, int(_row_budget or CV_ROW_BUDGET), n_grid)
    cap = cap.to(device=dev, dtype=torch.float64)
    pieces = []
    clock[0] = time.perf_counter()
    for s0, s1 in chunks:
        p0, p1 = int(plan.pair_off[s0]), int(plan.pair_off[s1])
        if p1 == p0:
            continue
        ent_h, ps_h, g_h = _cv_entries(plan, s0, s1, n_grid)
        pmask = plan.mask[ps_h]
        # gathered order: fits grouped by mask class (stable), so that every class is one contiguous fit batch
        perm = np.argsort(pmask, kind="stable")
        pairs_h = ent_h[perm].astype(np.int64)
        hist_len = he_h[pairs_h] - offsets_host[ps_h[perm]]
        win_len = we_h[pairs_h] - he_h[pairs_h]
        fit_off = np.zeros(pairs_h.size + 1, np.int64)
        np.cumsum(hist_len, out=fit_off[1:])
        hmax = int(win_len.max())
        n = pairs_h.size
        d_pairs = torch.from_numpy(pairs_h).to(dev)
        d_fit_off = torch.from_numpy(fit_off).to(dev)
        ds_g = torch.empty(int(fit_off[-1]), dtype=torch.int64, device=dev)
        y_g = torch.empty(int(fit_off[-1]), dtype=y.dtype, device=dev)
        fut = torch.empty((n, hmax), dtype=torch.int64, device=dev)
        torch.cuda.current_stream(dev).synchronize()
        L.check(lib.pb200_cv_gather_device(ctx.handle, ds_ns.data_ptr(), y.data_ptr(), ydt, d_off.data_ptr(),
                                           plan.pair_series.data_ptr(), plan.hist_end.data_ptr(), plan.win_end.data_ptr(),
                                           d_pairs.data_ptr(), n, d_fit_off.data_ptr(), hmax, ds_g.data_ptr(),
                                           y_g.data_ptr(), fut.data_ptr()), "pb200_cv_gather_device")
        if R:
            reg_g = torch.empty((R, int(fit_off[-1])), dtype=torch.float64, device=dev)
            reg_f = torch.empty((R, n, hmax), dtype=torch.float64, device=dev)
            L.check(lib.pb200_cv_gather_regressors_device(
                ctx.handle, regressors.data_ptr(), int(offsets_host[-1]), R, scale_full.data_ptr(), d_off.data_ptr(),
                plan.pair_series.data_ptr(), plan.hist_end.data_ptr(), plan.win_end.data_ptr(), d_pairs.data_ptr(), n,
                d_fit_off.data_ptr(), hmax, reg_g.data_ptr(), reg_f.data_ptr()), "pb200_cv_gather_regressors_device")
            copy_p = scale_full[torch.from_numpy(ps_h[perm]).to(dev)].contiguous()
        ctx.synchronize()
        lap("gather")
        # fits, one call per mask class; records re-laid into the layout of ``opts`` for the one predict call
        sp = pmask[perm]
        fitted = _fitted_outputs(_Space(dev), n, lay, R, zeros=True)
        cap_p = cap[torch.from_numpy(ps_h[perm]).to(dev)].contiguous()
        prior_p = torch.from_numpy(grid_h[g_h[perm]]).to(dev) if grid_h is not None else None
        bounds = np.flatnonzero(np.diff(np.concatenate(([-1], sp, [-1])))).tolist()
        for a, b in zip(bounds[:-1], bounds[1:]):
            oc = _with_mask(opts, int(sp[a]))
            r0, r1 = int(fit_off[a]), int(fit_off[b])
            fc = fit_batch_device(ctx, oc, ds_g[r0:r1], y_g[r0:r1], fit_off[a:b + 1] - r0, float(floor), 1.0,
                                  cap=cap_p[a:b], prior=prior_p[a:b] if prior_p is not None else None,
                                  regressors=reg_g[:, r0:r1].contiguous() if R else None,
                                  reg_scale_copy=copy_p[a:b] if R else None)
            if R:
                fitted.reg_scale[a:b] = fc.reg_scale
            # a table's cutoff fit packs the same active columns as the full model (never more: every entry of its
            # table is an active entry of the full one); its table drops the built-ins forced off and so numbers the
            # entries differently, and the mask is restated in the full table's entries
            w = fc.params.shape[1]
            assert w <= lay.pstride, (w, lay.pstride)
            fitted.params[a:b, :w] = fc.params
            fitted.tchange[a:b] = fc.tchange
            fitted.meta_i32[a:b] = fc.meta_i32
            if table is not None:
                fitted.meta_i32[a:b, 3] = int(table_mask(table, int(sp[a])))
            fitted.meta_i64[a:b] = fc.meta_i64
            fitted.meta_f64[a:b] = fc.meta_f64
        torch.cuda.current_stream(dev).synchronize()
        lap("fit")
        floor_p = torch.full((n,), float(floor), dtype=torch.float64, device=dev)
        if W is not None:
            wmax = max(1, min(hmax, int(horizon_ns) // W))      # a pair has no more windows than held-out rows
        if sums:
            origins = plan.cutoff[d_pairs] + 1
            flen = torch.from_numpy(win_len.astype(np.int32)).to(dev)
            fcst, ws = predict_sums_anchored_device(ctx, opts, fitted, fut, floor_p, cap_p, W, origins, flen, seed=seed,
                                                    intervals=True, wmax=wmax, levels=wlevels)
        elif levels is not None:
            fcst = predict_quantiles_device(ctx, opts, fitted, fut, floor_p, cap_p, levels, seed=seed,
                                            intervals=intervals and opts.uncertainty_samples > 0)
        else:
            fcst = predict_batch_device(ctx, opts, fitted, fut, floor_p, cap_p, seed=seed, intervals=intervals,
                                        regressors=reg_f if R else None)
        lap("predict")
        # back to plan order, then the held-out rows
        inv = torch.from_numpy(np.argsort(perm, kind="stable")).to(dev)
        yhat = fcst.yhat[inv]
        lo = fcst.yhat_lower[inv] if fcst.yhat_lower is not None else None
        hi = fcst.yhat_upper[inv] if fcst.yhat_upper is not None else None
        futp = fut[inv]
        d_ent = torch.from_numpy(ent_h).to(dev)
        wl = torch.from_numpy(we_h[ent_h] - he_h[ent_h]).to(dev)
        valid = torch.arange(hmax, device=dev)[None, :] < wl[:, None]
        kk, jj = torch.nonzero(valid, as_tuple=True)
        src_row = plan.hist_end[d_ent][kk] + jj
        rows = {"series": torch.from_numpy(ps_h * n_grid + g_h).to(dev)[kk], "ds": futp[kk, jj],
                "cutoff": plan.cutoff[d_ent][kk], "y": y[src_row].to(torch.float64), "yhat": yhat[kk, jj],
                "yhat_lower": lo[kk, jj] if lo is not None else None, "yhat_upper": hi[kk, jj] if hi is not None else None}
        met = None
        if rolling_window is not None:
            v0 = s0 * n_grid
            met = performance_metrics_device(ctx, rows["series"] - v0, rows["ds"] - rows["cutoff"], rows["y"], rows["yhat"],
                                             rows["yhat_lower"], rows["yhat_upper"], (s1 - s0) * n_grid, rolling_window)
            met["series"] = met["series"] + v0
            lap("metrics")
        qpiece = None
        if levels is not None:
            yq = fcst.quantiles[:, inv][:, kk, jj]
            qmet = None
            if rolling_window is not None:
                qmet = quantile_metrics_device(ctx, rows["series"] - s0, rows["ds"] - rows["cutoff"], rows["y"], yq, levels,
                                               s1 - s0, rolling_window)
                qmet["series"] = qmet["series"] + s0
                lap("quantile_metrics")
            qpiece = (yq.cpu().numpy(), qmet)
        wpiece = None
        if W is not None:
            cw = cv_windows_device(ctx, ds_ns, y, plan, d_pairs, fcst.yhat, W, wmax)
            nwin = cw["n_windows"][inv].long()
            wk, wj = torch.nonzero(torch.arange(wmax, device=dev)[None, :] < nwin[:, None], as_tuple=True)
            wcut = plan.cutoff[d_ent][wk]
            wrows = {"series": torch.from_numpy(ps_h * n_grid + g_h).to(dev)[wk], "cutoff": wcut,
                     "horizon": cw["start"][inv][wk, wj] - wcut + W, "points": cw["points"][inv][wk, wj],
                     "y": cw["y_sum"][inv][wk, wj], "yhat": cw["yhat_sum"][inv][wk, wj],
                     "yhat_lower": ws.lower[inv][wk, wj] if sums else None,
                     "yhat_upper": ws.upper[inv][wk, wj] if sums else None}
            lap("windows")
            wmet = None
            if rolling_window is not None:
                v0 = s0 * n_grid
                wmet = performance_metrics_device(ctx, wrows["series"] - v0, wrows["horizon"], wrows["y"], wrows["yhat"],
                                                  wrows["yhat_lower"], wrows["yhat_upper"], (s1 - s0) * n_grid,
                                                  rolling_window)
                wmet["series"] = wmet["series"] + v0
                lap("window_metrics")
            wq = None
            if wlevels is not None:
                wyq = ws.quantiles[:, inv][:, wk, wj]
                wqmet = None
                if rolling_window is not None:
                    v0 = s0 * n_grid
                    wqmet = quantile_metrics_device(ctx, wrows["series"] - v0, wrows["horizon"], wrows["y"], wyq, wlevels,
                                                    (s1 - s0) * n_grid, rolling_window)
                    wqmet["series"] = wqmet["series"] + v0
                    lap("window_quantile_metrics")
                wq = (wyq.cpu().numpy(), wqmet)
            wpiece = ({k: (v.cpu().numpy() if v is not None else None) for k, v in wrows.items()}, wmet, wq)
        fh = None
        if keep_fits:
            fh = FittedBatch(*(x[inv].cpu().numpy() for x in (fitted.params, fitted.tchange, fitted.meta_i32,
                                                               fitted.meta_i64, fitted.meta_f64)), lay.smax, lay.kmax,
                             reg_scale=fitted.reg_scale[inv].cpu().numpy() if R else None)
        pieces.append(({k: (v.cpu().numpy() if v is not None else None) for k, v in rows.items()}, met,
                       fitted.meta_i32[inv, 4].cpu().numpy(), fh, wpiece, qpiece))
        lap("rows")
    cat = lambda xs: np.concatenate(xs) if xs else None                       # noqa: E731
    rows = {k: cat([p[0][k] for p in pieces]) if (pieces and pieces[0][0][k] is not None) else None
            for k in ("series", "ds", "cutoff", "y", "yhat", "yhat_lower", "yhat_upper")}
    if not pieces:
        rows.update({k: np.zeros(0, np.int64) for k in ("series", "ds", "cutoff")})
        rows.update({k: np.zeros(0) for k in ("y", "yhat")})
    metrics = None
    if rolling_window is not None:
        keys = ("series", "horizon", "mse", "rmse", "mae", "mape", "coverage")
        metrics = {k: (cat([p[1][k] for p in pieces]) if pieces and pieces[0][1][k] is not None else None) for k in keys}
        if not pieces:
            metrics = performance_metrics_device(ctx, *(torch.zeros(0, dtype=t, device=dev) for t in
                                                        (torch.int64, torch.int64, torch.float64, torch.float64)),
                                                 None, None, 0, rolling_window)
    fitted_all = None
    if keep_fits and pieces:
        fitted_all = FittedBatch(*(np.concatenate([getattr(p[3], f) for p in pieces])
                                   for f in ("params", "tchange", "meta_i32", "meta_i64", "meta_f64")), lay.smax, lay.kmax,
                                 reg_scale=np.concatenate([p[3].reg_scale for p in pieces]) if R else None)
    ent_all, ps_all, g_all = _cv_entries(plan, 0, plan.n_cutoffs.size, n_grid)
    status = cat([p[2] for p in pieces]) if pieces else np.zeros(0, np.int32)
    windows = None
    if W is not None:
        i64, f64 = np.zeros(0, np.int64), np.zeros(0)
        empty = {"series": i64, "cutoff": i64, "horizon": i64, "points": np.zeros(0, np.int32), "y": f64, "yhat": f64,
                 "yhat_lower": f64 if sums else None, "yhat_upper": f64 if sums else None}
        wr = {k: (cat([p[4][0][k] for p in pieces]) if pieces else v) if v is not None else None for k, v in empty.items()}
        wm = None
        if rolling_window is not None:
            keys = ("series", "horizon", "mse", "rmse", "mae", "mape", "coverage")
            if pieces:
                wm = {k: (cat([p[4][1][k] for p in pieces]) if pieces[0][4][1][k] is not None else None) for k in keys}
            else:
                wm = performance_metrics_device(ctx, *(torch.zeros(0, dtype=t, device=dev) for t in
                                                       (torch.int64, torch.int64, torch.float64, torch.float64)),
                                                *((torch.zeros(0, dtype=torch.float64, device=dev),) * 2 if sums else
                                                  (None, None)), 0, rolling_window)
        windows = CvWindows(W, wr["series"], wr["cutoff"], wr["horizon"], wr["points"], wr["y"], wr["yhat"],
                            wr["yhat_lower"], wr["yhat_upper"], wm)
        if wlevels is not None:
            windows.yhat_q = (np.concatenate([p[4][2][0] for p in pieces], axis=1) if pieces
                              else np.zeros((wlevels.size, 0)))
            if rolling_window is not None:
                keys = ("series", "horizon", "level", "pinball", "share_below")
                windows.quantile_metrics = (
                    {k: cat([p[4][2][1][k] for p in pieces]) for k in keys} if pieces else
                    {k: np.zeros(0, np.int64 if k in ("series", "horizon") else np.float64) for k in keys})
    yhat_q = qmetrics = None
    if levels is not None:
        yhat_q = np.concatenate([p[5][0] for p in pieces], axis=1) if pieces else np.zeros((levels.size, 0))
        if rolling_window is not None:
            keys = ("series", "horizon", "level", "pinball", "share_below")
            qmetrics = ({k: cat([p[5][1][k] for p in pieces]) for k in keys} if pieces else
                        {k: np.zeros(0, np.int64 if k in ("series", "horizon") else np.float64) for k in keys})
    return CvResult(ps_all * n_grid + g_all, plan.cutoff.cpu().numpy()[ent_all], status, plan.mask[ps_all], rows["series"],
                    rows["ds"], rows["cutoff"], rows["y"], rows["yhat"], rows["yhat_lower"], rows["yhat_upper"], metrics,
                    fitted_all, windows, yhat_q, qmetrics)


def _metric_slots(series, horizon_ns, n_series: int):
    """The rows sorted by (series, horizon), stable (two stable sorts: plumbing), the rows per series and their
    exclusive scan: the row order and slots of the metrics kernels."""
    import torch
    dev = series.device
    o1 = torch.sort(horizon_ns, stable=True).indices
    o2 = torch.sort(series[o1], stable=True).indices
    order = o1[o2].contiguous()
    R = int(series.shape[0])
    counts = torch.bincount(series, minlength=n_series) if R else torch.zeros(n_series, dtype=torch.int64, device=dev)
    srow_off = torch.zeros(n_series + 1, dtype=torch.int64, device=dev)
    srow_off[1:] = torch.cumsum(counts, 0)
    return order, counts, srow_off


def quantile_metrics_device(ctx: L.Context, series, horizon_ns, y, yq, levels, n_series: int,
                            rolling_window: float = 0.1) -> dict:
    """Calibration of held-out quantiles per series and horizon (pb200_cv_quantile_metrics_device, DESIGN §15): rows as
    performance_metrics_device's, ``yq`` [Q, rows] float64 the quantile of each level of ``levels`` (fractions).  Per
    (series, horizon, level), the rolling-window means of the pinball loss max(q e, (q - 1) e), e = y - yq, and of
    [y <= yq].  Returns host numpy columns series, horizon, level, pinball, share_below, ordered by (series, horizon,
    level as given)."""
    import torch
    lv = np.ascontiguousarray(np.asarray(levels, dtype=np.float64))
    quantile_percentiles(lv)
    if not (0.0 <= float(rolling_window) <= 1.0):
        raise ValueError(f"rolling_window must be in [0, 1] (got {rolling_window!r})")
    dev = y.device
    R, Q = int(y.shape[0]), lv.size
    order, counts, srow_off = _metric_slots(series, horizon_ns, n_series)
    out_h, scratch = (torch.empty(R, dtype=torch.int64, device=dev) for _ in range(2))
    pin, below = (torch.empty((Q, R), dtype=torch.float64, device=dev) for _ in range(2))
    valid = torch.zeros(R, dtype=torch.int32, device=dev)
    if R and n_series:
        h, yy, q = horizon_ns.contiguous(), y.contiguous(), yq.contiguous()
        torch.cuda.current_stream(dev).synchronize()
        L.check(L.load().pb200_cv_quantile_metrics_device(
            ctx.handle, h.data_ptr(), yy.data_ptr(), q.data_ptr(), R, Q, _np_ptr(lv), order.data_ptr(), srow_off.data_ptr(),
            int(n_series), float(rolling_window), out_h.data_ptr(), scratch.data_ptr(), pin.data_ptr(), below.data_ptr(),
            valid.data_ptr()), "pb200_cv_quantile_metrics_device")
        ctx.synchronize()
    keep = valid.bool()
    slot_series = torch.repeat_interleave(torch.arange(n_series, device=dev), counts) if R else torch.zeros(0, dtype=torch.int64, device=dev)
    m = int(keep.sum().item())
    out = {"series": slot_series[keep].repeat_interleave(Q), "horizon": out_h[keep].repeat_interleave(Q),
           "level": torch.from_numpy(lv).to(dev).repeat(m), "pinball": pin[:, keep].T.reshape(-1),
           "share_below": below[:, keep].T.reshape(-1)}
    return {k: v.cpu().numpy() for k, v in out.items()}


def performance_metrics_device(ctx: L.Context, series, horizon_ns, y, yhat, yhat_lower, yhat_upper, n_series: int,
                               rolling_window: float = 0.1) -> dict:
    """fbprophet.diagnostics.performance_metrics per series (pb200_cv_metrics_device) over held-out rows given as CUDA
    tensors: ``series`` int64 in [0, n_series), ``horizon_ns`` int64 (ds - cutoff), ``y`` / ``yhat`` (and optionally
    ``yhat_lower`` / ``yhat_upper``) float64.  Rows of one series are summed in their given order within a horizon.
    Returns host numpy columns series, horizon, mse, rmse, mae, mape, coverage (None without intervals), ordered by
    (series, horizon)."""
    import torch
    if not (0.0 <= float(rolling_window) <= 1.0):
        raise ValueError(f"rolling_window must be in [0, 1] (got {rolling_window!r})")
    dev = y.device
    R = int(y.shape[0])
    order, counts, srow_off = _metric_slots(series, horizon_ns, n_series)
    out_h, scratch = (torch.empty(R, dtype=torch.int64, device=dev) for _ in range(2))
    mse, rmse, mae, mape, cov = (torch.empty(R, dtype=torch.float64, device=dev) for _ in range(5))
    valid = torch.zeros(R, dtype=torch.int32, device=dev)
    has_iv = yhat_lower is not None
    if R and n_series:
        h, yy, yh = horizon_ns.contiguous(), y.contiguous(), yhat.contiguous()
        lo = yhat_lower.contiguous() if has_iv else None
        hi = yhat_upper.contiguous() if has_iv else None
        torch.cuda.current_stream(dev).synchronize()
        L.check(L.load().pb200_cv_metrics_device(
            ctx.handle, h.data_ptr(), yy.data_ptr(), yh.data_ptr(), lo.data_ptr() if has_iv else None,
            hi.data_ptr() if has_iv else None, order.data_ptr(), srow_off.data_ptr(), int(n_series), float(rolling_window),
            out_h.data_ptr(), scratch.data_ptr(), mse.data_ptr(), rmse.data_ptr(), mae.data_ptr(), mape.data_ptr(),
            cov.data_ptr(), valid.data_ptr()), "pb200_cv_metrics_device")
        ctx.synchronize()
    keep = valid.bool()
    slot_series = torch.repeat_interleave(torch.arange(n_series, device=dev), counts) if R else torch.zeros(0, dtype=torch.int64, device=dev)
    out = {"series": slot_series[keep], "horizon": out_h[keep], "mse": mse[keep], "rmse": rmse[keep], "mae": mae[keep],
           "mape": mape[keep], "coverage": cov[keep] if has_iv else None}
    return {k: (v.cpu().numpy() if v is not None else None) for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------------------------
# Hyperparameter tuning: fbprophet's documented grid search over the prior scales, every series in one job (DESIGN §10)
# ---------------------------------------------------------------------------------------------------------------------
TUNE_METRICS = ("mse", "rmse", "mae", "mape")


@dataclass
class TuneResult:
    """Output of tune_device.  ``grid`` [n_grid, 2]: the (changepoint_prior_scale, seasonality_prior_scale) pairs in
    enumeration order.  Per (series, grid point), host numpy [n, n_grid]: ``scores`` (the metric over all of the series'
    held-out rows: performance_metrics with rolling_window = 1) and ``eligible`` (every cutoff fit succeeded and the
    score is finite).  Per series: ``chosen`` (grid index of the lowest eligible score, the first on ties; -1: none
    eligible, the options' scales were used), ``prior`` [n, 2] (the pair of the final fit) and ``fitted``, the
    full-history fits with those pairs (CUDA tensors).  ``cv``: the grid backtest itself (virtual series)."""
    grid: np.ndarray
    scores: np.ndarray
    eligible: np.ndarray
    chosen: np.ndarray
    prior: np.ndarray
    fitted: FittedBatch
    cv: CvResult


def tune_device(ctx: L.Context, opts: L.Options, ds_ns, y, offsets_host: np.ndarray, floor: float, cap_multiplier: float,
                horizon_ns: int, period_ns: int, initial_ns: int, grid, metric: str = "rmse",
                plan: Optional[CvPlan] = None, timings: Optional[dict] = None,
                _row_budget: Optional[int] = None) -> TuneResult:
    """For every series of a packed batch: cross_validation + performance_metrics(rolling_window=1) at every grid point
    (one cross_validation_device call with ``grid``), the grid point with the lowest ``metric``, then one
    pb200_fit_warm_device (fit_batch_device with ``prior``) over the full histories, each series with its chosen pair (the options' for a series with no
    eligible point).  ``cap_multiplier`` gives every fit the full history's cap, max(y) * cap_multiplier, as the modeler
    does.  ``timings`` as in cross_validation_device, plus ``final_fit``."""
    import time
    import torch
    if metric not in TUNE_METRICS:
        raise ValueError(f"metric must be one of {', '.join(TUNE_METRICS)} (got {metric!r})")
    offsets_host = np.ascontiguousarray(offsets_host, dtype=np.int64)
    n = offsets_host.size - 1
    grid_h = np.ascontiguousarray(np.asarray(grid, dtype=np.float64).reshape(-1, 2))
    g = grid_h.shape[0]
    dev = ds_ns.device
    lens = torch.from_numpy(np.diff(offsets_host)).to(dev)
    cap = torch.segment_reduce(y.to(torch.float64), "max", lengths=lens) * float(cap_multiplier)
    cv = cross_validation_device(ctx, opts, ds_ns, y, offsets_host, floor, cap, horizon_ns, period_ns, initial_ns,
                                 rolling_window=1.0, plan=plan, timings=timings, _row_budget=_row_budget, grid=grid_h)
    scores = np.full(n * g, np.nan)
    scores[cv.metrics["series"]] = cv.metrics[metric]
    fit_ok = np.ones(n * g, bool)
    fit_ok[cv.pair_series[cv.pair_status < 0]] = False
    scores = scores.reshape(n, g)
    eligible = fit_ok.reshape(n, g) & np.isfinite(scores)
    chosen = np.argmin(np.where(eligible, scores, np.inf), axis=1)        # the first of equal minima
    chosen[~eligible.any(axis=1)] = -1
    prior = np.where((chosen >= 0)[:, None], grid_h[np.maximum(chosen, 0)],
                     np.array([[opts.changepoint_prior_scale, opts.seasonality_prior_scale]]))
    t0 = time.perf_counter()
    fitted = fit_batch_device(ctx, opts, ds_ns, y, offsets_host, float(floor), float(cap_multiplier),
                              prior=torch.from_numpy(np.ascontiguousarray(prior)).to(dev))
    if timings is not None:
        timings["final_fit"] = timings.get("final_fit", 0.0) + time.perf_counter() - t0
    return TuneResult(grid_h, scores, eligible, chosen, prior, fitted, cv)
