// fbprophet's initialize_scales for the extra regressors (DESIGN §19): the kernel that standardises them per series before
// the fit
#pragma once
#include "fit_kernel.cuh"
#include "regressors.cuh"

namespace pb200 {
struct RegScaleArgs {
    const double* reg;           // [R][n_rows]
    long long n_rows;
    const long long* offsets;    // [n_series + 1] (device)
    int n_series;
    RegSpec spec;
    double* reg_scale;           // [n_series][R][2] out
    unsigned char* bad;          // [n_series] out: 1 if a value of the series' history is not finite
    const double* scale_copy;    // [n_series][R][2]: the (mu, std) a regressor keeps where it is not standardised
                                 // (fbprophet's prophet_copy of the full model's scales, DESIGN §20); null: (0, 1)
};

// fbprophet's initialize_scales for the regressors, one warp per series: a first pass for min, max, the {0, 1} test,
// non-finite values and the sum, a second for sum (x - mu)^2 (the two-pass form of pandas' nanvar).  Fewer than two
// distinct values, or a binary column under 'auto', or standardize = 0: (mu, std) = (0, 1), or the series' scale_copy
// entry when there is one (initialize_scales overwrites mu / std only where it standardises).  A non-finite value: (NaN,
// NaN) and the series is flagged, so that prep_kernel gives it PB200_ST_BAD_REGRESSOR
__global__ void __launch_bounds__(256) reg_scale_kernel(const RegScaleArgs a) {
    const int lane = threadIdx.x & 31;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int nw = (gridDim.x * blockDim.x) >> 5;
    const int R = a.spec.R;
    for (int s = gw; s < a.n_series; s += nw) {
        const long long off = a.offsets[s];
        const int T = (int)(a.offsets[s + 1] - off);
        int bad_any = 0;
        for (int r = 0; r < R; ++r) {
            const double* x = a.reg + (size_t)r * a.n_rows + off;
            double mn = INFINITY, mx = -INFINITY, sum = 0.0;
            int nonfin = 0, binary = 1;
            for (int i = lane; i < T; i += 32) {
                const double v = x[i];
                if (!isfinite(v)) nonfin = 1;
                if (!(v == 0.0 || v == 1.0)) binary = 0;
                mn = fmin(mn, v);
                mx = fmax(mx, v);
                sum += v;
            }
            nonfin = __any_sync(FULL, nonfin);
            binary = __all_sync(FULL, binary);
            mn = wmin(mn);
            mx = wmax(mx);
            sum = wsum(sum);
            double mu = 0.0, sd = 1.0;
            if (a.scale_copy) {
                mu = a.scale_copy[((size_t)s * R + r) * 2];
                sd = a.scale_copy[((size_t)s * R + r) * 2 + 1];
            }
            const int st = a.spec.standardize[r];
            if (nonfin) {
                mu = sd = NAN;
            } else if (T >= 2 && mn != mx && (st == 1 || (st == PB200_STD_AUTO && !binary))) {
                mu = sum / (double)T;
                double ss = 0.0;
                for (int i = lane; i < T; i += 32) {
                    const double d = x[i] - mu;
                    ss = fma(d, d, ss);
                }
                ss = wsum(ss);
                sd = sqrt(ss / (double)(T - 1));
            }
            bad_any |= nonfin;
            if (lane == 0) {
                a.reg_scale[((size_t)s * R + r) * 2] = mu;
                a.reg_scale[((size_t)s * R + r) * 2 + 1] = sd;
            }
        }
        if (lane == 0) a.bad[s] = (unsigned char)bad_any;
    }
}

// The backtest's regressor values (DESIGN §20): fbprophet 0.5's cross_validation slices model.history, whose regressor
// columns setup_dataframe has replaced by z = (x - mu_full) / std_full.  For each gathered entry (a plan pair, as
// cv_gather_kernel's), z of its truncated history packed as the fit batch's planes and z of its held-out rows as
// [n][hmax] frames; a short window's padding is 0.0, a finite value (a non-finite one would fail the whole model in
// predict).  One CTA per entry.
struct CvRegGatherArgs {
    const double* reg;           // [R][n_rows] the original values
    long long n_rows;
    int R;
    const double* scale_full;    // [n_series][R][2] (mu_full, std_full) of the full histories
    const long long* offsets;    // [n_series + 1]
    const int* pair_series;      // [pairs] (plan)
    const long long* hist_end;
    const long long* win_end;
    const long long* pairs;      // [n]
    long long n;
    const long long* fit_off;    // [n + 1]
    int hmax;
    double* reg_fit;             // [R][fit_off[n]]
    double* reg_fut;             // [R][n * hmax]
};

__global__ void __launch_bounds__(256) cv_gather_regressors_kernel(const CvRegGatherArgs a) {
    const long long fit_rows = a.fit_off[a.n];
    for (long long k = blockIdx.x; k < a.n; k += gridDim.x) {
        const long long p = a.pairs[k];
        const int s = a.pair_series[p];
        const long long off = a.offsets[s], he = a.hist_end[p], we = a.win_end[p];
        const long long dst = a.fit_off[k], len = he - off;
        for (int r = 0; r < a.R; ++r) {
            const double mu = a.scale_full[((size_t)s * a.R + r) * 2], sd = a.scale_full[((size_t)s * a.R + r) * 2 + 1];
            const double* x = a.reg + (size_t)r * a.n_rows;
            for (long long i = threadIdx.x; i < len; i += blockDim.x)
                a.reg_fit[(size_t)r * fit_rows + dst + i] = reg_value(x[off + i], mu, sd);
            for (int j = threadIdx.x; j < a.hmax; j += blockDim.x)
                a.reg_fut[(size_t)r * a.n * a.hmax + k * a.hmax + j] = he + j < we ? reg_value(x[he + j], mu, sd) : 0.0;
        }
    }
}

}  // namespace pb200
