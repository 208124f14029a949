/*
 * prophet_b200.h -- C ABI of the H100-native batched Prophet fitter / scorer.
 *
 * Drop-in boundary for the per-series hot path of mageky/time-series-spark:
 *
 *   pb200_fit_*      replaces  model_time_series_udf            src/jobs/prophet_modeler.py:41-85
 *                    (floor/cap prep :56-60, Prophet(...).fit(pdf) :65-66) run once per
 *                    (series_id, dim_id) group by groupby().apply()  src/jobs/prophet_modeler.py:139-141
 *   pb200_predict_*  replaces  forecast_time_series_udf         src/jobs/prophet_scorer.py:35-102
 *                    (make_future_dataframe :64-66, floor/cap :67-68, predict :70,
 *                    int truncation :73, floor clamp :76-84) run once per model row by
 *                    groupby().apply()                          src/jobs/prophet_scorer.py:159-161
 *
 * All series of a shard go through ONE call.  Plain pointers and sizes only; no
 * torch / Arrow types.  "d_" = device (HBM) pointer, "h_" = host pointer.
 * Every function returns 0 on success or a negative PB200_E_* code; per-series
 * solver outcomes are reported in the status array, never as a call failure
 * (the reference turns a per-series RuntimeError into "no output row",
 * prophet_modeler.py:81-85 / prophet_scorer.py:99-102).
 *
 * There is NO CPU fallback behind this ABI: every entry point launches sm_90a
 * kernels and fails with PB200_E_CUDA if no device is usable.
 */
#ifndef PROPHET_B200_H
#define PROPHET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB200_ABI_VERSION 1

#if defined(__GNUC__)
#define PB200_API __attribute__((visibility("default")))
#else
#define PB200_API
#endif

/* call-level error codes */
#define PB200_OK            0
#define PB200_E_ARG        -1   /* bad argument (null pointer, negative size, unsupported option) */
#define PB200_E_CUDA       -2   /* CUDA runtime error; see pb200_last_error() */
#define PB200_E_WORKSPACE  -3   /* workspace too small */
#define PB200_E_UNSUPPORTED -4  /* series too long / option outside the compiled kernels */

/* per-series status (status[] output of fit).  >= 0 : Stan L-BFGS TerminationCondition
 * (stan/optimization/bfgs.hpp), a model row is produced;  < 0 : no model row. */
/* pb200_options.algorithm */
#define PB200_ALG_LBFGS_NEWTON 0  /* optimizing(LBFGS); except RuntimeError: optimizing(Newton)  -- fbprophet 0.5 Prophet.fit */
#define PB200_ALG_LBFGS        1  /* L-BFGS only: a line-search failure is final (status PB200_ST_LSFAIL, row dropped) */
#define PB200_ALG_NEWTON       2  /* Newton only (tests; later fbprophet versions use it for short histories) */

#define PB200_ST_SUCCESS      0   /* only transient; never final */
#define PB200_ST_ABSX        10
#define PB200_ST_ABSF        20
#define PB200_ST_RELF        21
#define PB200_ST_ABSGRAD     30
#define PB200_ST_RELGRAD     31
#define PB200_ST_MAXIT       40
#define PB200_ST_CONST_LINEAR 50  /* fbprophet "nothing to fit" shortcut: params = init, sigma_obs = 1e-9 */
#define PB200_ST_NEWTON      60   /* model from fbprophet 0.5's Newton retry after an L-BFGS line-search failure */
#define PB200_ST_LSFAIL      -1   /* line search failed (PyStan raises RuntimeError -> fbprophet Newton retry) */
#define PB200_ST_INIT_ERROR  -2   /* objective not finite at the initial point */
#define PB200_ST_TOO_FEW     -3   /* < 2 rows  (fbprophet ValueError) */
#define PB200_ST_CAP_LE_FLOOR -4  /* cap <= floor (fbprophet ValueError) */
#define PB200_ST_BAD_INPUT   -5   /* unsorted timestamps / non-finite y / zero time span */
#define PB200_ST_BAD_PRIOR   -6   /* pb200_fit_prior_device: the series' prior scales are not finite and > 0 */
/* -7 PB200_ST_BAD_REGRESSOR: see the regressor entry points at the end of this header */

/* where a series of pb200_fit_warm_device started (d_warm) */
#define PB200_WARM_USED       1   /* from its previous model */
#define PB200_WARM_NONE       0   /* cold: no previous model, or the series is not optimised (prep error, constant linear) */
#define PB200_WARM_SHAPE     -1   /* cold: the previous model's S or seasonality mask differs from the new history's */
#define PB200_WARM_BAD       -2   /* cold: the previous model has a non-finite k, m, delta or beta, or sigma_obs <= 0 */

/* y element type */
#define PB200_Y_I32 0
#define PB200_Y_F32 1
#define PB200_Y_F64 2

/* growth */
#define PB200_GROWTH_LINEAR   0
#define PB200_GROWTH_LOGISTIC 1

/* seasonality switch: PB200_SEAS_AUTO follows Prophet.set_auto_seasonalities,
 * 0 disables, 1 forces that seasonality on.  Its Fourier order is the default
 * (yearly 10, weekly 3, daily 4) unless a pb200_options_v2 sets another. */
#define PB200_SEAS_AUTO (-1)

/* Options = Prophet.__init__ arguments the reference fixes at
 * prophet_modeler.py:65 plus fbprophet 0.5 / PyStan 2.19.1.1 defaults. */
typedef struct pb200_options {
    int32_t abi_version;            /* PB200_ABI_VERSION */
    int32_t growth;                 /* PB200_GROWTH_LOGISTIC (reference default) */
    int32_t multiplicative;         /* 1 = seasonality_mode='multiplicative' (reference default) */
    int32_t n_changepoints;         /* 25 */
    double  changepoint_range;      /* 0.8 */
    double  changepoint_prior_scale;/* 0.05 */
    double  seasonality_prior_scale;/* 10.0 */
    int32_t yearly;                 /* PB200_SEAS_AUTO | 0 | 1 */
    int32_t weekly;
    int32_t daily;
    int32_t max_iter;               /* 10000 (fbprophet passes iter=1e4) */
    int32_t history_size;           /* 5 */
    double  init_alpha;             /* 1e-3 */
    double  tol_obj;                /* 1e-12 */
    double  tol_rel_obj;            /* 1e4  (x machine epsilon) */
    double  tol_grad;               /* 1e-8 */
    double  tol_rel_grad;           /* 1e7  (x machine epsilon) */
    double  tol_param;              /* 1e-8 */
    double  interval_width;         /* 0.8; must be in [0, 1] when intervals are requested (else PB200_E_ARG, nothing launched) */
    int32_t uncertainty_samples;    /* 1000; 0 = skip yhat_lower / yhat_upper; else [2, 1024] (else PB200_E_UNSUPPORTED) */
    int32_t algorithm;              /* PB200_ALG_*: 0 = fbprophet 0.5's fit(): Stan L-BFGS, Newton retry after a line-search failure */
} pb200_options;

/* Fills *o with the reference's defaults. */
PB200_API void pb200_default_options(pb200_options* o);

/*
 * Seasonality table (DESIGN §18): fbprophet's add_seasonality(name, period, fourier_order, prior_scale) and non-default
 * built-in Fourier orders.  A pb200_options_v2 with v1.abi_version = PB200_ABI_VERSION_TABLE is accepted by every entry
 * point that takes a const pb200_options* (pass &o.v1); the tail is read only at that version.
 *   yearly_order / weekly_order / daily_order  Fourier order of the built-in when its switch (v1.yearly ...) is on or
 *                 AUTO; 0 = the default (10, 3, 4)
 *   seasonalities[n_seasonalities]  custom seasonalities in the order they were added: name (NUL-terminated, <= 15
 *                 bytes, unique), period in days > 0, fourier_order > 0, prior_scale > 0 or 0 for
 *                 v1.seasonality_prior_scale.  Never auto-disabled.  A name equal to a built-in's replaces it when that
 *                 built-in's switch is AUTO; with an explicit switch (0 or 1) it is refused.
 * The model's columns are the custom entries in order, then yearly, weekly and daily: at most PB200_MAX_SEASONALITIES
 * entries, K = sum of 2 * order <= 64 and 3 + max(1, n_changepoints) + K <= 96, else PB200_E_UNSUPPORTED before any
 * launch.  All seasonalities share v1.multiplicative.  A table that restates the defaults (no custom entry, orders
 * 0 or default) is the v1 model; any other is a table model: its series are fitted by a one-warp-per-series kernel
 * whatever their grid, meta_i32[3] holds one bit per table entry (bit j: entry j active), and the params row packs
 * the betas of the active entries in table order.
 * Components add one plane per custom entry (pb200_component_count).  The Newton retry and PB200_ALG_NEWTON evaluate
 * the table as the fit does.  Not yet for table models (PB200_E_UNSUPPORTED): per-series prior scales and warm starts
 * (pb200_fit_prior_device / pb200_fit_warm_* with a prior or an init).
 */
#define PB200_ABI_VERSION_TABLE 2
#define PB200_MAX_SEASONALITIES 8
typedef struct pb200_seasonality {
    char    name[16];
    double  period;                 /* days */
    double  prior_scale;            /* 0 = seasonality_prior_scale */
    int32_t fourier_order;
    int32_t reserved;
} pb200_seasonality;

typedef struct pb200_options_v2 {
    pb200_options v1;               /* v1.abi_version = PB200_ABI_VERSION_TABLE */
    int32_t yearly_order, weekly_order, daily_order;
    int32_t n_seasonalities;        /* 0 .. PB200_MAX_SEASONALITIES */
    const pb200_seasonality* seasonalities;
} pb200_options_v2;

/* Series of the context's LAST fit that went to the seasonality-table class (0 for a v1 model).  Synchronises. */
PB200_API int pb200_last_fit_table_count(struct pb200_ctx* ctx, int64_t* h_count);

/* Layout of one fitted-model record (the arrays fit writes and predict reads).
 * smax = max(1, n_changepoints); kmax = 2*(10+3+4) = 34 or fewer when
 * seasonalities are forced off, or the sum of 2 * order over a seasonality table;
 * params row = [k, m, sigma_obs, delta[smax], beta[kmax]]. */
typedef struct pb200_layout {
    int32_t smax;
    int32_t kmax;
    int32_t pstride;      /* doubles per params row = 3 + smax + kmax */
    int32_t meta_i32_stride; /* 8  : T, S, n_changepoints_real, seasonality mask (1 yearly|2 weekly|4 daily), status, iters, n_evals, reserved */
    int32_t meta_i64_stride; /* 2  : start_ns, t_scale_ns */
    int32_t meta_f64_stride; /* 4  : y_scale, floor, cap, neg_log_posterior */
} pb200_layout;

PB200_API int pb200_get_layout(const pb200_options* o, pb200_layout* out);

typedef struct pb200_ctx pb200_ctx;   /* owns a stream, device workspace and pinned staging */

/* Creates a context on CUDA device `device`.  Fails (NULL) when no GPU is present. */
PB200_API pb200_ctx* pb200_create(int device);
PB200_API void pb200_destroy(pb200_ctx* ctx);
PB200_API const char* pb200_last_error(void);
/* cudaStream_t the context launches on (as void*), for event timing by the caller. */
PB200_API void* pb200_stream(pb200_ctx* ctx);
/* number of kernel launches issued by this context so far */
PB200_API int64_t pb200_launch_count(pb200_ctx* ctx);
/* Diagnostics: how many series of the context's LAST fit went to each fit-kernel variant.
 * counts[v*8 + mask], summed over the CTA-width classes; v = 0 feature planes, 1 regular-grid rotation,
 * 2 week-period seasonal table, 3 day-period seasonal table; mask = bit0 yearly | bit1 weekly |
 * bit2 daily.  Synchronises the context's stream. */
/* Diagnostics (host arithmetic, no GPU needed): points per lane the seasonal-table kernel variants give a
 * series of T points whose table period is P grid steps -- the smallest chunk >= ceil(T / 32) for which the 64
 * residual bins the 32 lanes update in one loop step are pairwise distinct (what makes those updates race-free
 * and deterministic) -- or -1 if there is none within the slack the planes workspace allows. */
PB200_API int32_t pb200_tab_chunk(int32_t T, int32_t P);
#define PB200_N_VARIANT_COUNTS 32
PB200_API int pb200_last_fit_variant_counts(pb200_ctx* ctx, int32_t* h_counts);

/*
 * Batched fit: all series of a shard in one call.
 *
 * Input is the reference's (series_id, dim_id, ds, y) frame after grouping
 * (prophet_modeler.py:102-116,139-141) packed as a ragged batch: rows of series
 * i are [offsets[i], offsets[i+1]) of ds / y, sorted by ds ascending (the sort
 * fbprophet's setup_dataframe does), null y rows removed (fbprophet drops them).
 *   d_ds      int64 ns since epoch           [n_rows]
 *   d_y       y values, element type y_dtype [n_rows]
 *   h_offsets int64                          [n_series + 1]  (host copy; the
 *             device copy is made by the call)
 *   floor, cap_multiplier  config model.floor / model.cap_multiplier
 *             (prophet_modeler.py:56-60); cap_i = max(y_i) * cap_multiplier in double.
 *   d_cap     optional explicit per-series cap [n_series] (NULL = use cap_multiplier)
 * Outputs (device, caller-owned, sized per pb200_get_layout):
 *   d_params   double [n_series * pstride]
 *   d_tchange  double [n_series * smax]
 *   d_meta_i32 int32  [n_series * 8]
 *   d_meta_i64 int64  [n_series * 2]
 *   d_meta_f64 double [n_series * 4]
 * Stream-ordered on the context stream; returns after enqueueing.
 */
PB200_API int pb200_fit_device(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* d_cap,
                     double* d_params, double* d_tchange,
                     int32_t* d_meta_i32, int64_t* d_meta_i64, double* d_meta_f64);

/* pb200_fit_device with per-series prior scales (hyperparameter tuning fits each series with its own):
 *   d_prior   double [n_series][2] = (changepoint_prior_scale, seasonality_prior_scale) of series i
 *             at [2 i], [2 i + 1] (device); NULL = the options' scales for every series, which is
 *             exactly pb200_fit_device.  A series whose pair is not finite and > 0 gets status
 *             PB200_ST_BAD_PRIOR and no fit; the other series are not affected.  A pair equal to
 *             the options' gives the same bits as NULL. */
PB200_API int pb200_fit_prior_device(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* d_cap,
                     const double* d_prior, double* d_params, double* d_tchange,
                     int32_t* d_meta_i32, int64_t* d_meta_i64, double* d_meta_f64);

/* pb200_fit_prior_device started from each series' previous model (fbprophet's "updating fitted
 * models": m.fit(df, init=stan_init(m_old))):
 *   d_init_params   double [n_series][pstride] previous model records (layout of d_params), row i
 *                   for series i; NULL = exactly pb200_fit_prior_device (d_init_meta, d_warm ignored)
 *   d_init_meta     int32 [n_series][8] their meta_i32 (S at [1], mask at [3], status at [4]); a
 *                   status < 0 means "no previous model"
 *   d_warm          int32 [n_series] PB200_WARM_* per series, or NULL
 * A series starts from k, m, delta[0:S], log(sigma_obs), beta[0:K] of its record (raw values, no
 * rescaling to the new y_scale / t_scale / cap) when the record's status is >= 0, its S and mask are
 * the new history's, and those values are finite with sigma_obs > 0; otherwise from stan_init, bit for
 * bit as without an init.  The L-BFGS run, its Newton retry and PB200_ALG_NEWTON all start there; the
 * constant-linear shortcut ignores it.  A start point whose objective is not finite gives
 * PB200_ST_INIT_ERROR (L-BFGS).  The model record and its layout are those of pb200_fit_device. */
PB200_API int pb200_fit_warm_device(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* d_cap, const double* d_prior,
                     const double* d_init_params, const int32_t* d_init_meta_i32,
                     double* d_params, double* d_tchange,
                     int32_t* d_meta_i32, int64_t* d_meta_i64, double* d_meta_f64, int32_t* d_warm);

/* pb200_fit_warm_device on HOST buffers (h_cap, h_prior, h_init_params, h_warm may be NULL), plus
 * an optional trajectory: h_trace with trace_cap > 0 gets pb200_fit_trace_host's rows (NULL / 0: none). */
PB200_API int pb200_fit_warm_host(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* h_cap, const double* h_prior,
                     const double* h_init_params, const int32_t* h_init_meta_i32,
                     double* h_params, double* h_tchange,
                     int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64, int32_t* h_warm,
                     double* h_trace, int32_t trace_cap);

/* Same with HOST buffers in and out (pinned or pageable); the call stages
 * through the context's device workspace, copies results back and synchronises. */
PB200_API int pb200_fit_host(pb200_ctx* ctx, const pb200_options* opts,
                   const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                   const int64_t* h_offsets, int64_t n_series,
                   double floor, double cap_multiplier, const double* h_cap,
                   double* h_params, double* h_tchange,
                   int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64);

/*
 * Parity-test hook: evaluates the Prophet MAP objective (-log posterior up to constants,
 * the function Stan's L-BFGS minimises) and its gradient at caller-supplied points, through
 * the same kernel code the fit uses.  h_theta / h_grad rows have stride pstride and hold
 * Stan's unconstrained order: k, m, delta[S_i], log(sigma_obs), beta[K_i] packed from 0.
 * h_f[i] = objective, h_meta_i32 as in fit (status PB200_ST_INIT_ERROR when not finite).
 */
PB200_API int pb200_objective_host(pb200_ctx* ctx, const pb200_options* opts,
                   const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                   const int64_t* h_offsets, int64_t n_series,
                   double floor, double cap_multiplier, const double* h_theta,
                   double* h_f, double* h_grad, int32_t* h_meta_i32);

/*
 * Parity-test hook: pb200_fit_host that also records the optimiser's trajectory.  For every accepted
 * L-BFGS iteration it <= trace_cap of series i, h_trace[(i * trace_cap + it - 1) * 4 ...] =
 * (it, f_k, alpha_k, objective evaluations so far) -- the record oracle/prophet_oracle.py::stan_lbfgs(trace=...)
 * produces, so that the two can be compared step by step (a wrong line-search or update constant that still
 * converges shows up in the first rows).  Rows never written stay 0.
 */
PB200_API int pb200_fit_trace_host(pb200_ctx* ctx, const pb200_options* opts,
                   const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                   const int64_t* h_offsets, int64_t n_series,
                   double floor, double cap_multiplier,
                   double* h_params, double* h_tchange,
                   int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64,
                   double* h_trace, int32_t trace_cap);

/*
 * Batched predict over `horizon` future timestamps per model.
 *   d_future_ds int64 ns [n_models * horizon]  (make_future_dataframe output,
 *               prophet_scorer.py:64-66; built by pb200_make_future_device or the caller)
 *   d_floor / d_cap  per-model doubles as the scorer reads them back from the
 *               float32 model-table columns (prophet_scorer.py:46-47,67-68)
 * Outputs [n_models * horizon]:
 *   d_yhat        double  trend*(1+multiplicative)+additive
 *   d_yhat_lower / d_yhat_upper  double, MC interval (NULL or uncertainty_samples=0 to skip);
 *                 a function of the seed and the model's own record, not of its place in the batch
 *   d_yhat_int    int32   (int)yhat, then < floor -> floor   (prophet_scorer.py:73-84),
 *                 saturated to [INT32_MIN, INT32_MAX]
 * Models whose meta status < 0 produce no forecast: their rows are filled with
 * NaN / INT32_MIN and the caller drops them (empty frame in the reference).
 */
PB200_API int pb200_predict_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int);

PB200_API int pb200_predict_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int);

/*
 * pb200_predict_* plus fbprophet's component columns of Prophet.predict (DESIGN §12).  Same arguments and the same
 * yhat / yhat_lower / yhat_upper / yhat_int bits as pb200_predict_*, and:
 *   d_components  double [PB200_N_COMPONENTS][n_models * horizon], plane PB200_COMP_* (required):
 *     TREND           predict_trend: piecewise trend * y_scale + floor (floor 0 for linear growth)
 *     MULTIPLICATIVE  multiplicative_terms: yearly + weekly + daily in multiplicative mode, else 0;
 *                     yhat == trend * (1 + multiplicative_terms) exactly
 *     ADDITIVE        additive_terms: (yearly + weekly + daily) * y_scale in additive mode, else 0;
 *                     yhat == trend + additive_terms up to the rounding of additive_terms (yhat fuses the product)
 *     YEARLY / WEEKLY / DAILY  X_c beta_c of that seasonality: times y_scale in additive mode, the relative factor
 *                     in multiplicative mode; exactly 0 when the model's seasonality mask lacks it
 *   d_trend_lower / d_trend_upper  double [n_models * horizon] or both NULL: percentiles at 100(1 -+ w)/2 of the
 *     noise-free trend of the same draws as yhat_lower / yhat_upper; they need those intervals (both pointers and
 *     uncertainty_samples > 0, else PB200_E_ARG) and take their option checks.
 * Failed models (status < 0) get NaN in every plane and bound.
 */
#define PB200_N_COMPONENTS        6
#define PB200_COMP_TREND          0
#define PB200_COMP_MULTIPLICATIVE 1
#define PB200_COMP_ADDITIVE       2
#define PB200_COMP_YEARLY         3
#define PB200_COMP_WEEKLY         4
#define PB200_COMP_DAILY          5
/* Planes of pb200_predict_components_* for these options: PB200_N_COMPONENTS, plus one per custom seasonality of a
 * seasonality table not named like a built-in, in table order (a custom 'yearly' / 'weekly' / 'daily' fills that
 * built-in's plane); d_components holds that many planes.  Each is X_c beta_c of its seasonality as the built-ins' planes
 * are (0 where the model's mask lacks it), and in table order they add up to multiplicative_terms (multiplicative mode)
 * or to additive_terms / y_scale's unrounded sum.  A negative PB200_E_* for bad options. */
PB200_API int32_t pb200_component_count(const pb200_options* o);
PB200_API int pb200_predict_components_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, double* d_components, double* d_trend_lower, double* d_trend_upper);

PB200_API int pb200_predict_components_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int, double* h_components, double* h_trend_lower, double* h_trend_upper);

/*
 * pb200_predict_* plus forecast totals over fixed-width time windows with joint-draw intervals: fbprophet's
 * predictive_samples(future)['yhat'] summed per window, then percentiles of the sums (DESIGN §13).  Same arguments and the
 * same yhat / yhat_lower / yhat_upper / yhat_int bits as pb200_predict_* (d_yhat_lower / d_yhat_upper optional as there), and:
 *   width_ns > 0, origin_ns   the window of a point is floor((ds - origin_ns) / width_ns); a model's windows are the
 *                 maximal runs of equal window index in its (ascending) frame, in order
 *   wmax > 0      slots per model in the arrays below
 *   d_n_windows   int32 [n_models]  the model's number of windows -- the true count also when it exceeds wmax, in which
 *                 case only the first wmax windows are written: the caller checks
 * and, each [n_models * wmax], slot j of model i at i * wmax + j:
 *   d_win_start     int64   origin_ns + index * width_ns of window j
 *   d_win_points    int32   frame points in it (the first and last window of a frame may be partial)
 *   d_yhat_sum      double  s = 0.0; s = s + yhat[h] over the window's points in frame order
 *   d_quantity_sum  int64   sum of yhat_int over them
 *   d_sum_lower / d_sum_upper  double  numpy linear-interpolation percentiles at 100(1 -+ interval_width)/2 over the
 *                 uncertainty_samples sums of the draws behind yhat_lower / yhat_upper, each draw summed like yhat_sum
 * Slots at or past n_windows hold INT64_MIN / 0 / NaN / INT64_MIN / NaN / NaN.  Failed models (status < 0) have no window.
 * uncertainty_samples must be in [2, 1024] (PB200_E_UNSUPPORTED) and interval_width in [0, 1], width_ns and wmax > 0 and
 * the window outputs non-null (PB200_E_ARG): nothing is launched otherwise.
 */
PB200_API int pb200_predict_sums_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                         double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper);

PB200_API int pb200_predict_sums_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax,
                       int32_t* h_n_windows, int64_t* h_win_start, int32_t* h_win_points,
                       double* h_yhat_sum, int64_t* h_quantity_sum, double* h_sum_lower, double* h_sum_upper);

/*
 * pb200_predict_sums_device with a window origin and a frame length per model (DESIGN §14): model i's windows are
 * floor((ds - d_origin_ns[i]) / width_ns) over its first d_frame_len[i] points; the points after them (a frame padded by
 * repeating its last timestamp) are predicted as usual but summed into no window.  The draws are those of the whole
 * frame, so with every origin equal to origin_ns and every length equal to horizon the outputs are
 * pb200_predict_sums_device's, byte for byte; the pointwise outputs are always pb200_predict_device's.  win_start is
 * d_origin_ns[i] + w * width_ns.  d_origin_ns / d_frame_len: [n_models] device arrays, both required.
 */
PB200_API int pb200_predict_sums_anchored_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int64_t width_ns, const int64_t* d_origin_ns,
                         const int32_t* d_frame_len, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                         double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper);

/*
 * pb200_predict_sums_* over calendar periods (DESIGN §17): months, quarters and years of any anchor.  The arguments and
 * outputs are pb200_predict_sums_*'s with (months, month_shift) in place of (width_ns, origin_ns):
 *   months in {1, 3, 12}, 0 <= month_shift < months   the period of a point is floor((mi + month_shift) / months), mi the
 *                 months of ds's proleptic Gregorian civil date since 1970-01 (mathematical floor: also before 1970); a
 *                 model's windows are the maximal runs of equal period in its (ascending) frame, in order
 *   d_win_start   the period's start: 00:00 on day 1 of month p * months - month_shift since 1970-01
 * pandas' 'M' is (1, 0), 'Q-<MON>' (3, (12 - E) mod 3) and 'Y-<MON>' (12, (12 - E) mod 12), E the end month (1..12).  A
 * period start before the int64-ns minimum is not representable: such a slot holds the start taken mod 2^64 (the callers
 * refuse such frames).  A bad rule is PB200_E_ARG; the other checks are pb200_predict_sums_*'s.  Nothing is launched on
 * an error.
 */
PB200_API int pb200_predict_period_sums_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int32_t months, int32_t month_shift, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                         double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper);

PB200_API int pb200_predict_period_sums_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int, int32_t months, int32_t month_shift, int32_t wmax,
                       int32_t* h_n_windows, int64_t* h_win_start, int32_t* h_win_points,
                       double* h_yhat_sum, int64_t* h_quantity_sum, double* h_sum_lower, double* h_sum_upper);

/*
 * The period of each of n timestamps under (months, month_shift) and its start, by the very __host__ __device__ functions
 * the calendar kernel runs (csrc/calendar.cuh); host arrays.  Needs no context or device.  PB200_E_ARG on a bad rule.
 */
PB200_API int pb200_period_host(const int64_t* ds, int64_t n, int32_t months, int32_t month_shift, int64_t* period,
                                int64_t* start);

/*
 * pb200_predict_* plus forecast quantiles at n_q levels from the same draws (DESIGN §15): fbprophet's
 * np.percentile(predictive_samples(future)['yhat'], p, axis=1) for each p of h_percentiles, in one pass over the draws.
 * Same arguments and the same yhat / yhat_lower / yhat_upper / yhat_int bits as pb200_predict_* (the bounds optional as
 * there), and:
 *   n_q            levels, in [1, 32]
 *   h_percentiles  host double [n_q], each in [0, 100]; any order, repeats allowed
 *   d_quantiles    double [n_q * n_models * horizon]: plane q, model i, point h at (q * n_models + i) * horizon + h
 * Plane q at a point is s_i + (s_{min(i+1, n-1)} - s_i) * f over the sorted draws s, with x = p_q / 100.0 * (n - 1),
 * i = floor(x), f = x - i, n = uncertainty_samples: the expression of the interval bounds, so a plane at
 * 100 (1 -+ interval_width) / 2 (computed as written) is yhat_lower / yhat_upper bit for bit.  Failed models get NaN.
 * uncertainty_samples must be in [2, 1024] (PB200_E_UNSUPPORTED) and interval_width in [0, 1]; n_q, a NaN or
 * out-of-range percentile, or a null h_percentiles / d_quantiles give PB200_E_ARG.  Nothing is launched on an error.
 */
PB200_API int pb200_predict_quantiles_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int32_t n_q, const double* h_percentiles, double* d_quantiles);

PB200_API int pb200_predict_quantiles_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int, int32_t n_q, const double* h_percentiles, double* h_quantiles);

/* future_ds[i*horizon + j] = last_ds[i] + (j+1)*freq_ns  -- make_future_dataframe
 * (include_history=False) for a fixed-width pandas frequency. */
PB200_API int pb200_make_future_device(pb200_ctx* ctx, const int64_t* d_last_ds, int64_t n_models,
                             int32_t horizon, int64_t freq_ns, int64_t* d_future_ds);

PB200_API int pb200_synchronize(pb200_ctx* ctx);

/*
 * Forecast CSV rows formatted on the device: the row formatting of convert_forecasts + write_forecasts
 * (src/jobs/prophet_scorer.py:131-150 -- extract_date per row :107-108, created_timestamp :134, Spark's CSV writer
 * :147-150) for the standard frame
 *     "created_timestamp",series_id,dim_id,"forecast_date","forecast_timestamp",forecast_quantity
 * Two passes: row lengths, then -- given the exclusive scan of the lengths as byte offsets -- the bytes
 * (d_out holds the sum of the lengths).  ds in [1970-01-01, 10000-01-01); created_timestamp at most 64 bytes.
 * pb200_forecast_csv_row_host runs the same row formatter on the host for ONE row (tests; returns the row's
 * length, out must hold 160 bytes).
 */
PB200_API int pb200_forecast_csv_lengths_device(pb200_ctx* ctx, const int32_t* d_series_id, const int32_t* d_dim_id,
                                                const int32_t* d_quantity, int64_t n_rows, int32_t created_len,
                                                int64_t* d_row_len);
PB200_API int pb200_forecast_csv_rows_device(pb200_ctx* ctx, const int32_t* d_series_id, const int32_t* d_dim_id,
                                             const int64_t* d_ds_ns, const int32_t* d_quantity, int64_t n_rows,
                                             const char* h_created, int32_t created_len, const int64_t* d_row_off,
                                             uint8_t* d_out);
PB200_API int32_t pb200_forecast_csv_row_host(int32_t series_id, int32_t dim_id, int64_t ds_ns, int32_t quantity,
                                              const char* created, int32_t created_len, char* out);

/*
 * Backtest (fbprophet.diagnostics.cross_validation / performance_metrics) of a batch of series; DESIGN §9.
 *
 * Cutoff plan, two passes over the series (d_ds sorted ascending per series, rows [d_offsets[i], d_offsets[i+1])):
 *   pb200_cv_plan_counts_device  d_n_cutoffs[i] = cutoffs of generate_cutoffs(horizon, period, initial) (0 on error),
 *                                d_mask[i] = the full history's seasonality mask (1 yearly | 2 weekly | 4 daily, the rule
 *                                of the fit's set_auto_seasonalities under opts->yearly / weekly / daily), d_err[i] =
 *                                PB200_CV_ERR_* bits.
 *   pb200_cv_plan_device         given d_pair_off = exclusive scan of d_n_cutoffs ([n_series + 1]), writes per
 *                                (series, cutoff) pair, cutoffs ascending within a series: d_pair_series, d_cutoff (ns),
 *                                d_hist_end (first row > cutoff: the history is [offsets[i], hist_end)), d_win_end (first
 *                                row > cutoff + horizon: the held-out window is [hist_end, win_end)); ORs
 *                                PB200_CV_ERR_FEW into d_err.
 * horizon / period / initial: int64 ns, > 0.
 */
#define PB200_CV_ERR_HORIZON 1   /* "Less data than horizon" */
#define PB200_CV_ERR_INITIAL 2   /* "Less data than horizon after initial window" */
#define PB200_CV_ERR_FEW     4   /* "Less than two datapoints before cutoff" at some cutoff */
PB200_API int pb200_cv_plan_counts_device(pb200_ctx* ctx, const pb200_options* opts, const int64_t* d_ds,
                                          const int64_t* d_offsets, int64_t n_series, int64_t horizon_ns, int64_t period_ns,
                                          int64_t initial_ns, int32_t* d_n_cutoffs, int32_t* d_mask, int32_t* d_err);
PB200_API int pb200_cv_plan_device(pb200_ctx* ctx, const pb200_options* opts, const int64_t* d_ds, const int64_t* d_offsets,
                                   int64_t n_series, int64_t horizon_ns, int64_t period_ns, int64_t initial_ns,
                                   const int64_t* d_pair_off, int32_t* d_err, int32_t* d_pair_series, int64_t* d_cutoff,
                                   int64_t* d_hist_end, int64_t* d_win_end);

/*
 * Truncated-history fit batch of n plan pairs d_pairs[k]: entry k's history rows (ds, and y in its element type y_dtype)
 * go to [d_fit_off[k], d_fit_off[k+1]) of d_ds_out / d_y_out (d_fit_off = exclusive scan of hist_end - offsets[series]),
 * its held-out timestamps to row k of d_future_ds [n * hmax], a window shorter than hmax padded by repeating its last
 * timestamp (so that pb200_predict_device runs on the frame as it is; hmax >= every window's length).
 */
PB200_API int pb200_cv_gather_device(pb200_ctx* ctx, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                                     const int64_t* d_offsets, const int32_t* d_pair_series, const int64_t* d_hist_end,
                                     const int64_t* d_win_end, const int64_t* d_pairs, int64_t n, const int64_t* d_fit_off,
                                     int32_t hmax, int64_t* d_ds_out, void* d_y_out, int64_t* d_future_ds);

/*
 * performance_metrics per series over held-out rows: d_horizon (ns, ds - cutoff), d_y, d_yhat and optionally
 * d_yhat_lower / d_yhat_upper (both or neither) of n_rows rows; d_order lists the rows sorted by (series, horizon) and
 * series i owns d_order[d_srow_off[i] .. d_srow_off[i+1]).  With w = min(n_i, max(1, (int)(rolling_window * n_i))) the
 * metrics of a distinct horizon h are means over w rows: every row of h, then rows of smaller horizons nearest first, the
 * group where the window stops contributing its mean times the rows still needed (rolling_mean_by_h).  Outputs per slot
 * q = d_srow_off[i] + g for the g-th distinct horizon of series i (slots past the last horizon and horizons with fewer
 * than w rows at or below them get d_valid[q] = 0): d_out_horizon, d_mse, d_rmse, d_mae, d_mape (NaN for every horizon
 * of a series with some |y| < 1e-8), d_coverage (NaN without intervals).  d_scratch: int64 [rows].  Sums run in the
 * rows' listed order, one thread per series: bit-reproducible and independent of the other series.
 */
PB200_API int pb200_cv_metrics_device(pb200_ctx* ctx, const int64_t* d_horizon, const double* d_y, const double* d_yhat,
                                      const double* d_yhat_lower, const double* d_yhat_upper, const int64_t* d_order,
                                      const int64_t* d_srow_off, int64_t n_series, double rolling_window,
                                      int64_t* d_out_horizon, int64_t* d_scratch, double* d_mse, double* d_rmse,
                                      double* d_mae, double* d_mape, double* d_coverage, int32_t* d_valid);

/*
 * Backtest window totals (DESIGN §14) of n gathered entries: entry k is plan pair d_pairs[k], its held-out rows
 * [d_hist_end[p], d_win_end[p]) of d_ds / d_y (y_dtype as pb200_cv_gather_device) and row k of d_yhat [n * hmax] (the
 * predict frame of pb200_cv_gather_device's d_future_ds).  Window j of cutoff c is (c + j W, c + (j + 1) W], W =
 * width_ns > 0: row r lies in j = (ds_r - c - 1) / W.  Per entry, its non-empty windows in ascending j go to slots
 * k * wmax + i: d_win_start (c + j W), d_win_points, d_y_sum and d_yhat_sum (the rows' float64 y / yhat summed in
 * ascending row order, plain fp64 adds); d_n_windows[k] is the count (slots at or past it hold INT64_MIN / 0 / NaN; a
 * count above wmax writes the first wmax).  One warp per entry, no floating-point atomics: an entry's outputs depend
 * on that entry only.
 */
PB200_API int pb200_cv_windows_device(pb200_ctx* ctx, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                                      const int64_t* d_cutoff, const int64_t* d_hist_end, const int64_t* d_win_end,
                                      const int64_t* d_pairs, int64_t n, const double* d_yhat, int32_t hmax,
                                      int64_t width_ns, int32_t wmax, int32_t* d_n_windows, int64_t* d_win_start,
                                      int32_t* d_win_points, double* d_y_sum, double* d_yhat_sum);

/*
 * Calibration of held-out quantiles by horizon (DESIGN §15): pb200_cv_metrics_device's rows, order, slots and rolling
 * window rule over two per-row values of each level tau_q = h_levels[q] (host double [n_q], each in [0, 1], n_q in
 * [1, 32]) with the held-out quantile d_yq[q * n_rows + r] and e = y - yq:
 *   pinball loss  max(tau e, (tau - 1) e)
 *   below         1 if y <= yq else 0
 * The means over the window go to d_pinball / d_share_below [n_q * n_rows] at q * n_rows + slot, with d_out_horizon and
 * d_valid as pb200_cv_metrics_device's; d_scratch: int64 [n_rows].  One thread per series, no atomics.
 */
PB200_API int pb200_cv_quantile_metrics_device(pb200_ctx* ctx, const int64_t* d_horizon, const double* d_y,
                                               const double* d_yq, int64_t n_rows, int32_t n_q, const double* h_levels,
                                               const int64_t* d_order, const int64_t* d_srow_off, int64_t n_series,
                                               double rolling_window, int64_t* d_out_horizon, int64_t* d_scratch,
                                               double* d_pinball, double* d_share_below, int32_t* d_valid);

/*
 * In-sample predict over ragged frames (DESIGN §16): fbprophet's m.predict() with no frame, for every model's own history.
 * The arguments of pb200_predict_device, with the fixed (d_future_ds, horizon) replaced by a ragged frame: model i's rows
 * are [h_offsets[i], h_offsets[i + 1]) of d_ds (int64 ns, ascending per model), h_offsets a host int64 array
 * [n_models + 1] as pb200_fit_device's (the call makes the device copy).  Outputs, each indexed like d_ds:
 *   d_yhat                       double, pb200_predict_device's yhat
 *   d_yhat_lower / d_yhat_upper  double, the interval (NULL or uncertainty_samples = 0 to skip)
 * The key, the counters and Tmax are those of the model's own frame, so every value is bit-identical to what
 * pb200_predict_device gives when that model's rows are its frame, padded to any longer horizon by repeating its last
 * timestamp.  Failed models (status < 0) get NaN rows.  Argument checks are pb200_predict_device's, plus monotone
 * offsets; nothing is launched on an error.  The _host form takes host arrays (h_ds [h_offsets[n_models]]).
 */
PB200_API int pb200_predict_history_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_ds, const int64_t* h_offsets,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper);

PB200_API int pb200_predict_history_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_ds, const int64_t* h_offsets,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper);

/*
 * Outlier flags and the kept rows (DESIGN §16), two passes over series i's rows [d_offsets[i], d_offsets[i + 1]):
 *   pb200_outlier_counts_device   d_flag[r] = (double)y[r] < d_lower[r] || (double)y[r] > d_upper[r] (uint8; a NaN
 *                                 bound never flags), d_kept[i] = the series' rows not flagged (int32)
 *   pb200_outlier_compact_device  given d_kept_off = exclusive scan of d_kept ([n_series + 1], int64), writes the kept
 *                                 rows' ds and y (y in its element type y_dtype) to [d_kept_off[i], d_kept_off[i + 1]) of
 *                                 d_ds_out / d_y_out in their order: a packed batch pb200_fit_device takes as it is.
 * One warp per series, no atomics: a series' outputs depend on its own rows only.
 */
PB200_API int pb200_outlier_counts_device(pb200_ctx* ctx, const void* d_y, int32_t y_dtype, const int64_t* d_offsets,
                                          int64_t n_series, const double* d_lower, const double* d_upper, uint8_t* d_flag,
                                          int32_t* d_kept);
PB200_API int pb200_outlier_compact_device(pb200_ctx* ctx, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                                           const int64_t* d_offsets, int64_t n_series, const uint8_t* d_flag,
                                           const int64_t* d_kept_off, int64_t* d_ds_out, void* d_y_out);

/*
 * Extra regressors (DESIGN §19): fbprophet 0.5's add_regressor(name, prior_scale, standardize, mode).  A
 * pb200_options_v3 with v2.v1.abi_version = PB200_ABI_VERSION_REGRESSORS embeds a pb200_options_v2 (its table may
 * restate the defaults) and adds:
 *   holidays_prior_scale  the prior scale of a regressor whose prior_scale is 0 (fbprophet's default 10.0)
 *   regressors[n_regressors]  in the order they were added, at most PB200_MAX_REGRESSORS: name (NUL-terminated, <= 15
 *                 bytes, unique, not a seasonality's), prior_scale > 0 or 0, standardize PB200_STD_AUTO / 0 / 1.  Every
 *                 regressor takes v1.multiplicative.
 * With n_regressors = 0 a v3 options is exactly its v2 part.  With n_regressors = R > 0 the model is a table model
 * (even when its seasonalities restate the defaults) whose columns are the active seasonal columns, then the R
 * regressors: regressor r of series i is beta[K_seas(mask_i) + r] of its params row and of the objective hook's theta.
 * Limits: K_seas + R <= 64 and 3 + max(1, n_changepoints) + K_seas + R <= 96, else PB200_E_UNSUPPORTED before any
 * launch.  pb200_get_layout counts R in kmax.  Only the entry points below take such options; every other entry point
 * that takes options refuses them with PB200_E_UNSUPPORTED before any launch (components, window and period sums,
 * quantiles, in-sample predict, the backtest, per-series prior scales and warm start have no regressor values).
 *
 * Standardisation (fbprophet's initialize_scales, on the rows the fit sees): a regressor with fewer than 2 distinct
 * values, or under PB200_STD_AUTO one whose values are exactly {0, 1}, is used as it is (mu = 0, std = 1); any other is
 * (x - mu) / std with mu its mean and std its sample standard deviation (ddof = 1).
 */
#define PB200_ABI_VERSION_REGRESSORS 3
#define PB200_MAX_REGRESSORS 16
#define PB200_STD_AUTO (-1)
#define PB200_ST_BAD_REGRESSOR -7  /* a regressor value of the series' history is not finite (fbprophet: "Found NaN") */

typedef struct pb200_regressor {
    char    name[16];
    double  prior_scale;            /* 0 = holidays_prior_scale */
    int32_t standardize;            /* PB200_STD_AUTO | 0 | 1 */
    int32_t reserved;
} pb200_regressor;

typedef struct pb200_options_v3 {
    pb200_options_v2 v2;            /* v2.v1.abi_version = PB200_ABI_VERSION_REGRESSORS */
    double  holidays_prior_scale;   /* 10.0 */
    int32_t n_regressors;           /* 0 .. PB200_MAX_REGRESSORS */
    int32_t reserved;
    const pb200_regressor* regressors;
} pb200_options_v3;

/* pb200_fit_device with the regressors' values:
 *   d_reg        double [R][n_rows] (device), plane r aligned with d_ds (n_rows = h_offsets[n_series])
 *   d_reg_scale  double [n_series][R][2] (device, out): (mu, std) of each regressor of each series; (0, 1) where it is
 *                not standardised.  A series with a non-finite value gets status PB200_ST_BAD_REGRESSOR and no fit; the
 *                other series are not affected. */
PB200_API int pb200_fit_regressors_device(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* d_cap,
                     const double* d_reg, double* d_reg_scale,
                     double* d_params, double* d_tchange,
                     int32_t* d_meta_i32, int64_t* d_meta_i64, double* d_meta_f64);

/* The same on host buffers, plus pb200_fit_trace_host's trajectory rows when h_trace != NULL and trace_cap > 0. */
PB200_API int pb200_fit_regressors_host(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* h_cap,
                     const double* h_reg, double* h_reg_scale,
                     double* h_params, double* h_tchange,
                     int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64,
                     double* h_trace, int32_t trace_cap);

/* pb200_objective_host with the regressors' values (h_reg as h_ds); h_reg_scale [n_series][R][2] receives the
 * standardisation the objective used. */
PB200_API int pb200_objective_regressors_host(pb200_ctx* ctx, const pb200_options* opts,
                     const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series,
                     double floor, double cap_multiplier, const double* h_reg, double* h_reg_scale,
                     const double* h_theta, double* h_f, double* h_grad, int32_t* h_meta_i32);

/* pb200_predict_* with the regressors' future values:
 *   d_future_reg  double [R][n_models * horizon], plane r aligned with d_future_ds
 *   d_reg_scale   double [n_models][R][2], the fit's (mu, std)
 * yhat adds sum_r beta_r (x_r - mu_r) / std_r to the seasonal term.  A model with a non-finite future regressor value
 * gets the rows of a failed model (NaN, INT32_MIN). */
PB200_API int pb200_predict_regressors_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         const double* d_future_reg, const double* d_reg_scale,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int);

PB200_API int pb200_predict_regressors_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       const double* h_future_reg, const double* h_reg_scale,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int);

/*
 * The regressors' future values of every model's forecast grid, joined on the device (DESIGN §20).  The table: n_rows
 * rows packed by group, group g owning rows [d_tab_offsets[g], d_tab_offsets[g + 1]) of d_tab_ds (int64 ns, ascending
 * within a group) and of each plane of d_tab_reg (double [n_regressors][n_rows]).  d_model_group [n_models] (int64) is
 * each model's group, -1 for none; d_future_ds [n_models][horizon] its grid.  For every grid point the row of the
 * model's group with exactly its timestamp gives the point's values in d_future_reg (double [n_regressors][n_models *
 * horizon], the layout pb200_predict_regressors_* reads); a point without one gets NaN.  d_missing [n_models] (int32)
 * receives the model's points without a row, d_first_missing [n_models] (int64) the timestamp of the first of them
 * (INT64_MIN when there is none).  Rows that are no grid point are ignored.  The group's timestamps must be distinct:
 * with a repeated one, which of its rows is taken is not specified.  One warp per model, no atomics.
 */
PB200_API int pb200_join_future_regressors_device(pb200_ctx* ctx, const int64_t* d_tab_ds, const int64_t* d_tab_offsets,
                                                  const double* d_tab_reg, int64_t n_rows, int32_t n_regressors,
                                                  const int64_t* d_model_group, const int64_t* d_future_ds,
                                                  int64_t n_models, int32_t horizon, double* d_future_reg,
                                                  int32_t* d_missing, int64_t* d_first_missing);

/*
 * The backtest with regressors (DESIGN §20), fbprophet 0.5's cross_validation: the cutoff fits take the full history's
 * standardised values z = (x - mu_full) / std_full and keep the full model's (mu_full, std_full) where they do not
 * standardise (prophet_copy copies extra_regressors; initialize_scales overwrites mu / std only where it standardises).
 *   pb200_regressor_scales_device      reg_scale_kernel alone over full histories (h_offsets as pb200_fit_device's):
 *                                      d_reg_scale [n_series][R][2] (mu, std) as pb200_fit_regressors_device gives
 *                                      them, d_bad [n_series] (uint8) 1 where a value is not finite.
 *   pb200_cv_gather_regressors_device  beside pb200_cv_gather_device, for the same entries: z of each truncated history
 *                                      as d_reg_fit [R][d_fit_off[n]] and of each held-out window as d_reg_future
 *                                      [R][n * hmax] (pb200_predict_regressors_*'s layout), short windows padded with
 *                                      0.0; d_reg_scale_full [n_series][R][2].
 *   pb200_fit_regressors_copy_device   pb200_fit_regressors_device whose regressors keep d_reg_scale_copy
 *                                      [n_series][R][2] where they are not standardised, instead of (0, 1).
 */
PB200_API int pb200_regressor_scales_device(pb200_ctx* ctx, const pb200_options* opts, const double* d_reg,
                                            const int64_t* h_offsets, int64_t n_series, double* d_reg_scale,
                                            uint8_t* d_bad);
PB200_API int pb200_cv_gather_regressors_device(pb200_ctx* ctx, const double* d_reg, int64_t n_rows, int32_t n_regressors,
                                                const double* d_reg_scale_full, const int64_t* d_offsets,
                                                const int32_t* d_pair_series, const int64_t* d_hist_end,
                                                const int64_t* d_win_end, const int64_t* d_pairs, int64_t n,
                                                const int64_t* d_fit_off, int32_t hmax, double* d_reg_fit,
                                                double* d_reg_future);
PB200_API int pb200_fit_regressors_copy_device(pb200_ctx* ctx, const pb200_options* opts, const int64_t* d_ds,
                                               const void* d_y, int32_t y_dtype, const int64_t* h_offsets,
                                               int64_t n_series, double floor, double cap_multiplier, const double* d_cap,
                                               const double* d_reg, const double* d_reg_scale_copy, double* d_reg_scale,
                                               double* d_params, double* d_tchange, int32_t* d_meta_i32,
                                               int64_t* d_meta_i64, double* d_meta_f64);

#ifdef __cplusplus
}
#endif
#endif /* PROPHET_B200_H */
