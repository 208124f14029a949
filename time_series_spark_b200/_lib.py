"""ctypes binding of libprophet_b200.so (C ABI in include/prophet_b200.h and include/prophet_b200_window_quantiles.h).

There is no CPU fallback: importing this module never builds or emulates anything, and
``load()`` raises if the CUDA library is missing; ``Context()`` raises if no H100 is visible.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_VARIANT = os.environ.get("PB200_VARIANT", "")          # dev only: load an A/B build (see build.py)
LIB_PATH = os.path.join(_HERE, f"libprophet_b200{'_' + _VARIANT if _VARIANT else ''}.so")

ABI_VERSION = 1
Y_I32, Y_F32, Y_F64 = 0, 1, 2
GROWTH_LINEAR, GROWTH_LOGISTIC = 0, 1
SEAS_AUTO = -1

# per-series status codes (include/prophet_b200.h)
ST_ABSX, ST_ABSF, ST_RELF, ST_ABSGRAD, ST_RELGRAD, ST_MAXIT, ST_CONST_LINEAR = 10, 20, 21, 30, 31, 40, 50
ST_NEWTON = 60
ALG_LBFGS_NEWTON, ALG_LBFGS, ALG_NEWTON = 0, 1, 2
ST_LSFAIL, ST_INIT_ERROR, ST_TOO_FEW, ST_CAP_LE_FLOOR, ST_BAD_INPUT, ST_BAD_PRIOR = -1, -2, -3, -4, -5, -6
# where a series of a warm-started fit started (PB200_WARM_*)
WARM_USED, WARM_NONE, WARM_SHAPE, WARM_BAD = 1, 0, -1, -2
# planes of pb200_predict_components_* (PB200_COMP_*), in order
COMPONENTS = ("trend", "multiplicative_terms", "additive_terms", "yearly", "weekly", "daily")
N_COMPONENTS = len(COMPONENTS)


class Options(C.Structure):
    """struct pb200_options."""
    _fields_ = [
        ("abi_version", C.c_int32), ("growth", C.c_int32), ("multiplicative", C.c_int32),
        ("n_changepoints", C.c_int32), ("changepoint_range", C.c_double),
        ("changepoint_prior_scale", C.c_double), ("seasonality_prior_scale", C.c_double),
        ("yearly", C.c_int32), ("weekly", C.c_int32), ("daily", C.c_int32),
        ("max_iter", C.c_int32), ("history_size", C.c_int32),
        ("init_alpha", C.c_double), ("tol_obj", C.c_double), ("tol_rel_obj", C.c_double),
        ("tol_grad", C.c_double), ("tol_rel_grad", C.c_double), ("tol_param", C.c_double),
        ("interval_width", C.c_double), ("uncertainty_samples", C.c_int32), ("algorithm", C.c_int32),
    ]


ABI_VERSION_TABLE = 2
MAX_SEASONALITIES = 8


class Seasonality(C.Structure):
    """struct pb200_seasonality."""
    _fields_ = [("name", C.c_char * 16), ("period", C.c_double), ("prior_scale", C.c_double),
                ("fourier_order", C.c_int32), ("reserved", C.c_int32)]


class OptionsV2(Options):
    """struct pb200_options_v2: pb200_options followed by the seasonality table (passed where an Options is taken)."""
    _fields_ = [("yearly_order", C.c_int32), ("weekly_order", C.c_int32), ("daily_order", C.c_int32),
                ("n_seasonalities", C.c_int32), ("seasonalities", C.POINTER(Seasonality))]


ABI_VERSION_REGRESSORS = 3
MAX_REGRESSORS = 16
STD_AUTO = -1
ST_BAD_REGRESSOR = -7


class Regressor(C.Structure):
    """struct pb200_regressor."""
    _fields_ = [("name", C.c_char * 16), ("prior_scale", C.c_double), ("standardize", C.c_int32),
                ("reserved", C.c_int32)]


class OptionsV3(OptionsV2):
    """struct pb200_options_v3: pb200_options_v2 followed by the extra regressors (DESIGN §19)."""
    _fields_ = [("holidays_prior_scale", C.c_double), ("n_regressors", C.c_int32), ("reserved", C.c_int32),
                ("regressors", C.POINTER(Regressor))]


class Layout(C.Structure):
    """struct pb200_layout."""
    _fields_ = [("smax", C.c_int32), ("kmax", C.c_int32), ("pstride", C.c_int32),
                ("meta_i32_stride", C.c_int32), ("meta_i64_stride", C.c_int32), ("meta_f64_stride", C.c_int32)]


EXPORTS = [
    "pb200_default_options", "pb200_get_layout", "pb200_create", "pb200_destroy", "pb200_last_error",
    "pb200_stream", "pb200_launch_count", "pb200_last_fit_variant_counts", "pb200_tab_chunk", "pb200_fit_device", "pb200_fit_prior_device", "pb200_fit_warm_device", "pb200_fit_host", "pb200_fit_warm_host", "pb200_predict_device",
    "pb200_predict_host", "pb200_predict_components_device", "pb200_predict_components_host",
    "pb200_predict_sums_device", "pb200_predict_sums_host", "pb200_make_future_device", "pb200_synchronize", "pb200_objective_host",
    "pb200_fit_trace_host", "pb200_forecast_csv_lengths_device", "pb200_forecast_csv_rows_device", "pb200_forecast_csv_row_host",
    "pb200_cv_plan_counts_device", "pb200_cv_plan_device", "pb200_cv_gather_device", "pb200_cv_metrics_device",
    "pb200_predict_sums_anchored_device", "pb200_cv_windows_device", "pb200_predict_quantiles_device",
    "pb200_predict_quantiles_host", "pb200_cv_quantile_metrics_device", "pb200_predict_history_device",
    "pb200_predict_history_host", "pb200_outlier_counts_device", "pb200_outlier_compact_device",
    "pb200_predict_period_sums_device", "pb200_predict_period_sums_host", "pb200_period_host",
    "pb200_last_fit_table_count", "pb200_component_count", "pb200_fit_regressors_device", "pb200_fit_regressors_host",
    "pb200_objective_regressors_host", "pb200_predict_regressors_device", "pb200_predict_regressors_host",
    "pb200_join_future_regressors_device", "pb200_regressor_scales_device", "pb200_cv_gather_regressors_device",
    "pb200_fit_regressors_copy_device",
]
# declared in include/prophet_b200_window_quantiles.h (DESIGN §21)
WINDOW_QUANTILE_EXPORTS = [
    "pb200_predict_sums_quantiles_device", "pb200_predict_sums_quantiles_host",
    "pb200_predict_period_sums_quantiles_device", "pb200_predict_period_sums_quantiles_host",
    "pb200_predict_sums_anchored_quantiles_device",
]
CV_ERR_HORIZON, CV_ERR_INITIAL, CV_ERR_FEW = 1, 2, 4

_lib = None


def load() -> C.CDLL:
    """dlopen the in-tree library and declare prototypes.  Raises if it was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m time_series_spark_b200.build` "
            "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    vp, i64, i32, dbl, u64 = C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_uint64
    OP = C.POINTER(Options)
    fit_args = [vp, OP, vp, vp, i32, vp, i64, dbl, dbl, vp, vp, vp, vp, vp, vp]
    pred_args = [vp, OP, vp, vp, vp, vp, vp, i64, vp, i32, vp, vp, u64, vp, vp, vp, vp]
    hist_args = [vp, OP, vp, vp, vp, vp, vp, i64, vp, vp, vp, vp, u64, vp, vp, vp]
    twins = {      # the same arguments at both suffixes, _host and _device
        "pb200_predict": pred_args,
        "pb200_predict_components": pred_args + [vp, vp, vp],
        "pb200_predict_sums": pred_args + [i64, i64, i32] + [vp] * 7,
        "pb200_predict_period_sums": pred_args + [i32, i32, i32] + [vp] * 7,
        "pb200_predict_quantiles": pred_args + [i32, vp, vp],
        "pb200_predict_sums_quantiles": pred_args + [i64, i64, i32] + [vp] * 7 + [i32, vp, vp],
        "pb200_predict_period_sums_quantiles": pred_args + [i32, i32, i32] + [vp] * 7 + [i32, vp, vp],
        "pb200_predict_history": hist_args,
        "pb200_predict_regressors": pred_args[:13] + [vp, vp] + pred_args[13:],
    }
    prototypes = {name + s: args for name, args in twins.items() for s in ("_host", "_device")}
    prototypes.update({
        "pb200_default_options": [OP],
        "pb200_get_layout": [OP, C.POINTER(Layout)],
        "pb200_create": [C.c_int],
        "pb200_destroy": [vp],
        "pb200_last_error": [],
        "pb200_stream": [vp],
        "pb200_launch_count": [vp],
        "pb200_tab_chunk": [i32, i32],
        "pb200_last_fit_variant_counts": [vp, vp],
        "pb200_last_fit_table_count": [vp, vp],
        "pb200_component_count": [OP],
        "pb200_synchronize": [vp],
        "pb200_fit_device": fit_args,
        "pb200_fit_host": fit_args,
        "pb200_fit_prior_device": fit_args[:10] + [vp] + fit_args[10:],
        "pb200_fit_warm_device": fit_args[:10] + [vp, vp, vp] + fit_args[10:] + [vp],
        "pb200_fit_warm_host": fit_args[:10] + [vp, vp, vp] + fit_args[10:] + [vp, vp, i32],
        "pb200_fit_trace_host": fit_args[:9] + fit_args[10:] + [vp, i32],
        "pb200_fit_regressors_device": fit_args[:10] + [vp, vp] + fit_args[10:],
        "pb200_fit_regressors_copy_device": fit_args[:10] + [vp, vp, vp] + fit_args[10:],
        "pb200_fit_regressors_host": fit_args[:10] + [vp, vp] + fit_args[10:] + [vp, i32],
        "pb200_objective_host": fit_args[:9] + [vp, vp, vp, vp],
        "pb200_objective_regressors_host": fit_args[:9] + [vp, vp, vp, vp, vp, vp],
        "pb200_predict_sums_anchored_device": pred_args + [i64, vp, vp, i32] + [vp] * 7,
        "pb200_predict_sums_anchored_quantiles_device": pred_args + [i64, vp, vp, i32] + [vp] * 7 + [i32, vp, vp],
        "pb200_period_host": [vp, i64, i32, i32, vp, vp],
        "pb200_make_future_device": [vp, vp, i64, i32, i64, vp],
        "pb200_outlier_counts_device": [vp, vp, i32, vp, i64, vp, vp, vp, vp],
        "pb200_outlier_compact_device": [vp, vp, vp, i32, vp, i64, vp, vp, vp, vp],
        "pb200_join_future_regressors_device": [vp, vp, vp, vp, i64, i32, vp, vp, i64, i32, vp, vp, vp],
        "pb200_regressor_scales_device": [vp, OP, vp, vp, i64, vp, vp],
        "pb200_cv_gather_regressors_device": [vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, i64, vp, i32, vp, vp],
        "pb200_forecast_csv_lengths_device": [vp, vp, vp, vp, i64, i32, vp],
        "pb200_forecast_csv_rows_device": [vp, vp, vp, vp, vp, i64, C.c_char_p, i32, vp, vp],
        "pb200_forecast_csv_row_host": [i32, i32, i64, i32, C.c_char_p, i32, C.c_char_p],
        "pb200_cv_plan_counts_device": [vp, OP, vp, vp, i64, i64, i64, i64, vp, vp, vp],
        "pb200_cv_plan_device": [vp, OP, vp, vp, i64, i64, i64, i64, vp, vp, vp, vp, vp, vp],
        "pb200_cv_gather_device": [vp, vp, vp, i32, vp, vp, vp, vp, vp, i64, vp, i32, vp, vp, vp],
        "pb200_cv_metrics_device": [vp, vp, vp, vp, vp, vp, vp, vp, i64, dbl] + [vp] * 8,
        "pb200_cv_windows_device": [vp, vp, vp, i32, vp, vp, vp, vp, i64, vp, i32, i64, i32, vp, vp, vp, vp, vp],
        "pb200_cv_quantile_metrics_device": [vp, vp, vp, vp, i64, i32, vp, vp, vp, i64, dbl, vp, vp, vp, vp, vp],
    })
    restypes = {"pb200_default_options": None, "pb200_destroy": None, "pb200_create": vp, "pb200_last_error": C.c_char_p,
                "pb200_stream": vp, "pb200_launch_count": i64, "pb200_tab_chunk": i32, "pb200_component_count": i32,
                "pb200_forecast_csv_row_host": i32}     # every other entry point returns an int status
    for name, args in prototypes.items():
        f = getattr(lib, name)
        f.argtypes = args
        f.restype = restypes.get(name, C.c_int)
    _lib = lib
    return lib


def default_options() -> Options:
    o = Options()
    load().pb200_default_options(C.byref(o))
    return o


def get_layout(opts: Options) -> Layout:
    lay = Layout()
    rc = load().pb200_get_layout(C.byref(opts), C.byref(lay))
    if rc != 0:
        raise ValueError(f"pb200_get_layout failed ({rc}): {last_error()}")
    return lay


def last_error() -> str:
    return (load().pb200_last_error() or b"").decode()


class Pb200Error(RuntimeError):
    pass


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise Pb200Error(f"{what} failed ({rc}): {last_error()}")


class Context:
    """pb200_ctx handle: one per process per GPU."""

    def __init__(self, device: int = 0):
        self._lib = load()
        self._h = self._lib.pb200_create(int(device))
        if not self._h:
            raise Pb200Error("pb200_create failed: " + last_error())
        self.device = int(device)

    @property
    def handle(self):
        return self._h

    @property
    def stream(self) -> int:
        return int(self._lib.pb200_stream(self._h) or 0)

    @property
    def launch_count(self) -> int:
        return int(self._lib.pb200_launch_count(self._h))

    def last_fit_variant_counts(self):
        """(4, 8) int32: series of the last fit per kernel variant (planes, rotation, week table, day table)
        x seasonality mask."""
        import numpy as np
        out = np.zeros(32, np.int32)
        check(self._lib.pb200_last_fit_variant_counts(self._h, out.ctypes.data), "pb200_last_fit_variant_counts")
        return out.reshape(4, 8)

    def synchronize(self) -> None:
        check(self._lib.pb200_synchronize(self._h), "pb200_synchronize")

    def close(self) -> None:
        if self._h:
            self._lib.pb200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
