/*
 * Quantiles of window and calendar-period totals (DESIGN §21): the entry points that extend pb200_predict_sums_*,
 * pb200_predict_sums_anchored_device and pb200_predict_period_sums_* (prophet_b200.h) with n_q levels.  The same
 * library exports them; prophet_b200.h keeps the interface every other call uses.
 */
#ifndef PROPHET_B200_WINDOW_QUANTILES_H
#define PROPHET_B200_WINDOW_QUANTILES_H

#include "prophet_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/*
 * Quantiles of the window totals at n_q levels (DESIGN §21): pb200_predict_sums_*, pb200_predict_sums_anchored_device and
 * pb200_predict_period_sums_* with n_q percentiles and their planes after the sums arguments.  Plane q of a window is the
 * expression of pb200_predict_quantiles_* at h_percentiles[q] over the uncertainty_samples window sums whose percentiles
 * are d_sum_lower / d_sum_upper (the same draws, the same adds), so a plane at 100 (1 -+ interval_width) / 2 is
 * d_sum_lower / d_sum_upper bit for bit.  Every other output is the sums call's, byte for byte, and:
 *   n_q              levels, in [1, 32]
 *   h_percentiles    host double [n_q], each in [0, 100]; any order, repeats allowed
 *   d_sum_quantiles  double [n_q * n_models * wmax]: plane q, model i, slot j at (q * n_models + i) * wmax + j; slots at
 *                    or past n_windows and every slot of a failed model are NaN
 * The checks are the sums call's, then pb200_predict_quantiles_*'s: n_q, a NaN or out-of-range percentile, or a null
 * h_percentiles / d_sum_quantiles give PB200_E_ARG.  Options with regressors are refused (PB200_E_UNSUPPORTED) as by
 * every sums call.  Nothing is launched on an error.
 */
PB200_API int pb200_predict_sums_quantiles_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                         double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper,
                         int32_t n_q, const double* h_percentiles, double* d_sum_quantiles);

PB200_API int pb200_predict_sums_quantiles_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax,
                       int32_t* h_n_windows, int64_t* h_win_start, int32_t* h_win_points,
                       double* h_yhat_sum, int64_t* h_quantity_sum, double* h_sum_lower, double* h_sum_upper,
                       int32_t n_q, const double* h_percentiles, double* h_sum_quantiles);

PB200_API int pb200_predict_sums_anchored_quantiles_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int64_t width_ns, const int64_t* d_origin_ns,
                         const int32_t* d_frame_len, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                         double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper,
                         int32_t n_q, const double* h_percentiles, double* d_sum_quantiles);

PB200_API int pb200_predict_period_sums_quantiles_device(pb200_ctx* ctx, const pb200_options* opts,
                         const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed,
                         double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int32_t months, int32_t month_shift, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                         double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper,
                         int32_t n_q, const double* h_percentiles, double* d_sum_quantiles);

PB200_API int pb200_predict_period_sums_quantiles_host(pb200_ctx* ctx, const pb200_options* opts,
                       const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed,
                       double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int, int32_t months, int32_t month_shift, int32_t wmax,
                       int32_t* h_n_windows, int64_t* h_win_start, int32_t* h_win_points,
                       double* h_yhat_sum, int64_t* h_quantity_sum, double* h_sum_lower, double* h_sum_upper,
                       int32_t n_q, const double* h_percentiles, double* h_sum_quantiles);

#ifdef __cplusplus
}
#endif

#endif /* PROPHET_B200_WINDOW_QUANTILES_H */
