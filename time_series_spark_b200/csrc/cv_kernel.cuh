// Backtest (fbprophet.diagnostics cross_validation / performance_metrics) over a whole batch of series.  Four pieces, the
// fit / predict / MC kernels being reused unchanged in between:
//   cv_plan_kernel     per series: the cutoffs of generate_cutoffs, each cutoff's history end and held-out window, the
//                      full history's seasonality mask and the error flags.  Two passes, like csv_kernel.cuh: counts,
//                      then (given the exclusive scan of the counts) the (series, cutoff) pairs.
//   cv_gather_kernel   the truncated histories of a list of pairs packed into one ragged fit batch, and the held-out
//                      timestamps as a [pairs, hmax] frame for predict (short windows padded by their last timestamp).
//   cv_metrics_kernel  performance_metrics per series: per-horizon trailing-window means of the squared / absolute /
//                      relative errors and of the interval coverage.
//   cv_window_kernel   per gathered entry: the held-out rows' totals over fixed-width windows anchored at the cutoff
//                      (DESIGN §14), the window rows cv_metrics_kernel then reduces like pointwise rows.
//   cv_quantile_metrics_kernel  cv_metrics_kernel's trailing-window means of the pinball loss and of [y <= quantile]
//                      per level of held-out quantiles (DESIGN §15).
// Every series is one warp (plan, windows) or one thread (metrics) and every sum runs in one fixed order with no
// floating-point atomics: a series' plan, metrics and windows do not depend on the other series of the batch.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "fit_kernel.cuh"

namespace pb200 {
namespace cv {

// error flags of a series (cv_plan err[]); the fbprophet exceptions they stand for
constexpr int ERR_HORIZON = 1;   // "Less data than horizon"
constexpr int ERR_INITIAL = 2;   // "Less data than horizon after initial window"
constexpr int ERR_FEW = 4;       // "Less than two datapoints before cutoff" (some cutoff)

// first index in [lo, hi) whose timestamp is > v (hi if none)
__device__ __forceinline__ long long upper_bound(const long long* ds, long long lo, long long hi, const long long v) {
    while (lo < hi) {
        const long long mid = lo + ((hi - lo) >> 1);
        if (ds[mid] <= v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// generate_cutoffs over the sorted rows [a, b): returns the number of cutoffs (< 0: an ERR_* flag, negated) and, when
// out != nullptr, writes them in ascending order to out[0 .. n).  The walk produces them in descending order, so the
// writing pass is told n (from the counting pass) and fills out from the back.
// H, P and I may be any positive int64 (pandas Timedeltas reach ~106 751 days), so no sum or difference below is formed
// before it is known to stay in int64: a timestamp minus a duration that would fall below INT64_MIN lies before every
// row, and first + I beyond INT64_MAX after every cutoff.  (A wrapped last - H or prev - P would otherwise land after
// the rows and send the walk back to the same cutoff forever.)  Every cutoff c satisfies c <= last - H, so c + H does
// not overflow.
__device__ __forceinline__ int cutoff_walk(const long long* ds, const long long a, const long long b, const long long H,
                                           const long long P, const long long I, long long* out, const int n_known) {
    const long long first = ds[a], last = ds[b - 1];
    if (last < INT64_MIN + H || last - H < first) return -ERR_HORIZON;
    long long prev = last - H;
    const bool can_start = first <= INT64_MAX - I;             // else first + I is after every cutoff
    int n = 0;
    while (can_start && prev >= first + I) {
        long long c = 0;
        bool stop = false;
        if (prev < INT64_MIN + P) {
            // prev - P lies before every row: whichever branch fbprophet takes, the next cutoff ends the loop
            stop = true;
        } else {
            c = prev - P;
            const long long u = upper_bound(ds, a, b, c);     // first row > c
            if (!(u < b && ds[u] <= c + H)) {
                // no row in (c, c + H]: the next cutoff is (latest row <= c) - H.  With no such row fbprophet's cutoff
                // becomes NaT, which ends the loop and is the element dropped: prev is kept.  So does a next cutoff
                // before every row
                if (u == a || ds[u - 1] < INT64_MIN + H) stop = true;
                else c = ds[u - 1] - H;
            }
        }
        if (out) out[n_known - 1 - n] = prev;
        ++n;
        if (stop) return n;
        prev = c;
    }
    return n > 0 ? n : -ERR_INITIAL;                           // prev, the last element, is dropped
}

struct PlanArgs {
    const long long* ds;
    const long long* offsets;    // [n_series + 1]
    long long n_series;
    long long horizon, period, initial;
    int yearly, weekly, daily;   // pb200_options switches
    // counting pass (pair_off == nullptr)
    int* n_cut;                  // [n_series] cutoffs (0 on error)
    int* mask;                   // [n_series] full-history seasonality mask
    int* err;                    // [n_series] ERR_* bits
    // writing pass
    const long long* pair_off;   // [n_series + 1] exclusive scan of n_cut
    int* pair_series;            // [pairs]
    long long* cutoff;           // [pairs] ns
    long long* hist_end;         // [pairs] first row > cutoff
    long long* win_end;          // [pairs] first row > cutoff + horizon
};

__global__ void __launch_bounds__(256) cv_plan_kernel(const PlanArgs a) {
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long s = gw; s < a.n_series; s += nw) {
        const long long off = a.offsets[s], end = a.offsets[s + 1];
        if (a.pair_off == nullptr) {
            // the full history's smallest non-zero step, as prep_kernel measures it
            long long mindt = INT64_MAX;
            for (long long i = off + 1 + lane; i < end; i += 32) {
                const long long dt = a.ds[i] - a.ds[i - 1];
                if (dt != 0 && dt < mindt) mindt = dt;
            }
            mindt = wminll(mindt);
            if (lane == 0) {
                int err = 0, n = 0;
                if (end - off < 1) {
                    err = ERR_HORIZON;
                } else {
                    n = cutoff_walk(a.ds, off, end, a.horizon, a.period, a.initial, nullptr, 0);
                    if (n < 0) {
                        err = -n;
                        n = 0;
                    }
                }
                a.mask[s] = end - off < 1 ? 0 : auto_seasonality_mask(a.ds[end - 1] - a.ds[off], mindt, a.yearly, a.weekly, a.daily);
                a.n_cut[s] = n;
                a.err[s] = err;
            }
        } else if (lane == 0) {
            const long long p0 = a.pair_off[s];
            const int n = (int)(a.pair_off[s + 1] - p0);
            if (n <= 0) continue;
            cutoff_walk(a.ds, off, end, a.horizon, a.period, a.initial, a.cutoff + p0, n);
            int few = 0;
            for (int j = 0; j < n; ++j) {
                const long long c = a.cutoff[p0 + j];
                const long long he = upper_bound(a.ds, off, end, c);
                a.pair_series[p0 + j] = (int)s;
                a.hist_end[p0 + j] = he;
                a.win_end[p0 + j] = upper_bound(a.ds, he, end, c + a.horizon);
                if (he - off < 2) few = 1;
            }
            if (few) a.err[s] |= ERR_FEW;
        }
    }
}

struct GatherArgs {
    const long long* ds;
    const void* y;
    int y_dtype;
    const long long* offsets;    // [n_series + 1] of ds / y
    const int* pair_series;      // [pairs] (plan)
    const long long* hist_end;
    const long long* win_end;
    const long long* pairs;      // [n] the pair of each entry of the gathered batch
    long long n;
    const long long* fit_off;    // [n + 1] exclusive scan of the entries' history lengths
    int hmax;
    long long* ds_out;           // [fit_off[n]]
    void* y_out;                 // [fit_off[n]], element type y_dtype
    long long* fut;              // [n * hmax]
};

// one CTA per entry: its history prefix, then its held-out timestamps
__global__ void __launch_bounds__(256) cv_gather_kernel(const GatherArgs a) {
    for (long long k = blockIdx.x; k < a.n; k += gridDim.x) {
        const long long p = a.pairs[k];
        const long long off = a.offsets[a.pair_series[p]], he = a.hist_end[p], we = a.win_end[p];
        const long long dst = a.fit_off[k], len = he - off;
        for (long long i = threadIdx.x; i < len; i += blockDim.x) a.ds_out[dst + i] = a.ds[off + i];
        if (a.y_dtype == PB200_Y_F64) {
            const double* ys = (const double*)a.y;
            double* yd = (double*)a.y_out;
            for (long long i = threadIdx.x; i < len; i += blockDim.x) yd[dst + i] = ys[off + i];
        } else {   // int32 / float32: moved as 32-bit words
            const uint32_t* ys = (const uint32_t*)a.y;
            uint32_t* yd = (uint32_t*)a.y_out;
            for (long long i = threadIdx.x; i < len; i += blockDim.x) yd[dst + i] = ys[off + i];
        }
        for (int j = threadIdx.x; j < a.hmax; j += blockDim.x) {
            const long long r = he + j < we ? he + j : we - 1;
            a.fut[k * a.hmax + j] = a.ds[r];
        }
    }
}

struct MetricsArgs {
    const long long* horizon;    // [n_rows] ns (ds - cutoff)
    const double* y;             // [n_rows]
    const double* yhat;
    const double* lo;            // nullable (no coverage)
    const double* hi;
    const long long* order;      // [n_rows] the rows sorted by (series, horizon), stable
    const long long* srow_off;   // [n_series + 1] into order
    long long n_series;
    double rolling_window;
    // outputs, slot srow_off[s] + g for the g-th distinct horizon of series s
    long long* out_h;
    long long* out_n;            // scratch: rows of the horizon
    double* out_mse;
    double* out_rmse;
    double* out_mae;
    double* out_mape;
    double* out_cov;
    int* out_valid;              // 1 where the horizon has a metrics row
};

__global__ void __launch_bounds__(128) cv_metrics_kernel(const MetricsArgs a) {
    for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < a.n_series; s += (long long)gridDim.x * blockDim.x) {
        const long long r0 = a.srow_off[s], r1 = a.srow_off[s + 1], n = r1 - r0;
        if (n <= 0) continue;
        // group sums per distinct horizon, rows in their sorted order
        long long G = 0;
        bool tiny_y = false;
        for (long long r = r0; r < r1;) {
            const long long h = a.horizon[a.order[r]];
            double se = 0.0, ae = 0.0, ape = 0.0, cv = 0.0;
            long long c = 0;
            for (; r < r1 && a.horizon[a.order[r]] == h; ++r, ++c) {
                const long long i = a.order[r];
                const double yv = a.y[i], e = yv - a.yhat[i], ay = fabs(yv);
                if (ay < 1e-8) tiny_y = true;
                se += e * e;
                ae += fabs(e);
                ape += fabs(e) / ay;
                if (a.lo) cv += (a.lo[i] <= yv && yv <= a.hi[i]) ? 1.0 : 0.0;
            }
            const long long g = r0 + G++;
            a.out_h[g] = h;
            a.out_n[g] = c;
            a.out_mse[g] = se;
            a.out_mae[g] = ae;
            a.out_mape[g] = ape;
            a.out_cov[g] = cv;
        }
        long long w = (long long)(a.rolling_window * (double)n);
        if (w < 1) w = 1;
        if (w > n) w = n;
        // horizon k: the mean over w rows -- all of k's, then smaller horizons nearest first, the group where the
        // window stops contributing its mean times the rows still needed.  Descending k: slot k is overwritten with
        // its result only once no larger horizon needs its sums
        for (long long k = G - 1; k >= 0; --k) {
            double se = 0.0, ae = 0.0, ape = 0.0, cv = 0.0;
            long long need = w;
            for (long long g = k; g >= 0 && need > 0; --g) {
                const long long q = r0 + g, c = a.out_n[q];
                if (c >= need) {
                    const double f = (double)need / (double)c;
                    se += a.out_mse[q] * f;
                    ae += a.out_mae[q] * f;
                    ape += a.out_mape[q] * f;
                    cv += a.out_cov[q] * f;
                    need = 0;
                } else {
                    se += a.out_mse[q];
                    ae += a.out_mae[q];
                    ape += a.out_mape[q];
                    cv += a.out_cov[q];
                    need -= c;
                }
            }
            const long long q = r0 + k;
            a.out_valid[q] = need == 0 ? 1 : 0;
            const double mse = se / (double)w;
            a.out_mse[q] = mse;
            a.out_rmse[q] = sqrt(mse);
            a.out_mae[q] = ae / (double)w;
            a.out_mape[q] = tiny_y ? NAN : ape / (double)w;
            a.out_cov[q] = a.lo ? cv / (double)w : NAN;
        }
        for (long long q = r0 + G; q < r1; ++q) a.out_valid[q] = 0;
    }
}

// ---- held-out quantiles (DESIGN §15): pinball loss and the share of y at or below the quantile, per level ----
constexpr int CV_QMAX = 32;

struct QuantMetricsArgs {
    const long long* horizon;    // [n_rows] ns, as MetricsArgs
    const double* y;             // [n_rows]
    const double* yq;            // [nq][n_rows] the held-out quantile of each level
    long long n_rows;
    int nq;
    double level[CV_QMAX];       // tau in [0, 1]
    const long long* order;      // as MetricsArgs
    const long long* srow_off;
    long long n_series;
    double rolling_window;
    long long* out_h;            // slots as MetricsArgs
    long long* out_n;            // scratch
    double* out_pinball;         // [nq][n_rows]
    double* out_below;           // [nq][n_rows]
    int* out_valid;
};

// cv_metrics_kernel's groups and rolling window over, per level, max(tau e, (tau - 1) e) and [y <= yq]
__global__ void __launch_bounds__(128) cv_quantile_metrics_kernel(const QuantMetricsArgs a) {
    for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < a.n_series; s += (long long)gridDim.x * blockDim.x) {
        const long long r0 = a.srow_off[s], r1 = a.srow_off[s + 1], n = r1 - r0;
        if (n <= 0) continue;
        long long G = 0;
        for (long long r = r0; r < r1;) {
            const long long h = a.horizon[a.order[r]];
            long long re = r;
            while (re < r1 && a.horizon[a.order[re]] == h) ++re;
            const long long g = r0 + G++;
            a.out_h[g] = h;
            a.out_n[g] = re - r;
            for (int q = 0; q < a.nq; ++q) {
                const double tau = a.level[q];
                const double* yq = a.yq + (size_t)q * a.n_rows;
                double pin = 0.0, below = 0.0;
                for (long long j = r; j < re; ++j) {
                    const long long i = a.order[j];
                    const double yv = a.y[i], e = yv - yq[i];
                    pin += fmax(tau * e, (tau - 1.0) * e);
                    below += yv <= yq[i] ? 1.0 : 0.0;
                }
                a.out_pinball[(size_t)q * a.n_rows + g] = pin;
                a.out_below[(size_t)q * a.n_rows + g] = below;
            }
            r = re;
        }
        long long w = (long long)(a.rolling_window * (double)n);
        if (w < 1) w = 1;
        if (w > n) w = n;
        // descending k, as cv_metrics_kernel: slot k is overwritten only once no larger horizon needs its sums
        for (long long k = G - 1; k >= 0; --k) {
            long long need = w;
            long long gl = k;                      // the last group the window reaches
            for (; gl >= 0; --gl) {
                const long long c = a.out_n[r0 + gl];
                if (c >= need) break;
                need -= c;
            }
            a.out_valid[r0 + k] = gl >= 0 ? 1 : 0;
            for (int q = 0; q < a.nq; ++q) {
                double* pin = a.out_pinball + (size_t)q * a.n_rows + r0;
                double* below = a.out_below + (size_t)q * a.n_rows + r0;
                double sp = 0.0, sb = 0.0;
                long long nd = w;
                for (long long g = k; g >= 0 && nd > 0; --g) {
                    const long long c = a.out_n[r0 + g];
                    if (c >= nd) {
                        const double f = (double)nd / (double)c;
                        sp += pin[g] * f;
                        sb += below[g] * f;
                        nd = 0;
                    } else {
                        sp += pin[g];
                        sb += below[g];
                        nd -= c;
                    }
                }
                pin[k] = sp / (double)w;
                below[k] = sb / (double)w;
            }
        }
        for (long long q = r0 + G; q < r1; ++q) a.out_valid[q] = 0;
    }
}

struct WindowArgs {
    const long long* ds;
    const void* y;
    int y_dtype;
    const long long* cutoff;     // [pairs] (plan)
    const long long* hist_end;
    const long long* win_end;
    const long long* pairs;      // [n] the pair of each gathered entry
    long long n;
    const double* yhat;          // [n * hmax] the predict frame of the gathered entries
    int hmax;
    long long width;             // W > 0
    int wmax;
    // outputs: n_windows [n]; from here on [n * wmax], slot k * wmax + i for entry k's i-th non-empty window
    int* n_windows;
    long long* win_start;        // c + j W: window j is (c + j W, c + (j + 1) W]
    int* points;
    double* y_sum;
    double* yhat_sum;
};

// One warp per entry.  The held-out rows [hist_end, win_end) of the pair are read 32 at a time, one per lane (coalesced),
// then broadcast in row order so that every lane keeps the same running sums: s = s + v in ascending row order, plain
// fp64 adds, the order of tests/window_backtest_oracle.window_rows.  Row r lies in window j = (ds_r - (c + 1)) / W:
// every held-out row has c < ds_r <= c + H, so the quotient is a non-negative floor and no term overflows.  Lane 0 writes a window when
// the next row's differs; windows at or past wmax are counted and not written; slots past the count hold INT64_MIN / 0 /
// NaN, as mc_sum_kernel's.
__global__ void __launch_bounds__(256) cv_window_kernel(const WindowArgs a) {
    const int lane = threadIdx.x & 31;
    const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long k = gw; k < a.n; k += nwarps) {
        const long long p = a.pairs[k];
        const long long he = a.hist_end[p], we = a.win_end[p], c = a.cutoff[p];
        const double* yh = a.yhat + (size_t)k * a.hmax;
        const size_t wb = (size_t)k * a.wmax;
        int nw = 0, pts = 0;
        long long cur = 0;
        double ys = 0.0, fs = 0.0;
        auto close_window = [&]() {
            if (lane == 0 && nw < a.wmax) {
                a.win_start[wb + nw] = c + cur * a.width;
                a.points[wb + nw] = pts;
                a.y_sum[wb + nw] = ys;
                a.yhat_sum[wb + nw] = fs;
            }
            ++nw;
            pts = 0; ys = 0.0; fs = 0.0;
        };
        for (long long r0 = he; r0 < we; r0 += 32) {
            const long long r = r0 + lane;
            long long wv = 0;
            double yv = 0.0, fv = 0.0;
            if (r < we) {
                wv = (a.ds[r] - c - 1) / a.width;
                if (a.y_dtype == PB200_Y_F64) yv = ((const double*)a.y)[r];
                else if (a.y_dtype == PB200_Y_F32) yv = (double)((const float*)a.y)[r];
                else yv = (double)((const int*)a.y)[r];
                fv = yh[r - he];
            }
            const int m = we - r0 < 32 ? (int)(we - r0) : 32;
            for (int i = 0; i < m; ++i) {
                const long long wi = __shfl_sync(0xffffffffu, wv, i);
                const double yi = __shfl_sync(0xffffffffu, yv, i), fi = __shfl_sync(0xffffffffu, fv, i);
                if (pts > 0 && wi != cur) close_window();
                cur = wi;
                ++pts;
                ys = __dadd_rn(ys, yi);
                fs = __dadd_rn(fs, fi);
            }
        }
        if (pts > 0) close_window();
        if (lane == 0) a.n_windows[k] = nw;
        for (int i = (nw < a.wmax ? nw : a.wmax) + lane; i < a.wmax; i += 32) {
            a.win_start[wb + i] = INT64_MIN;
            a.points[wb + i] = 0;
            a.y_sum[wb + i] = NAN;
            a.yhat_sum[wb + i] = NAN;
        }
    }
}

}  // namespace cv
}  // namespace pb200
