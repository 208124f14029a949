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
};

// fbprophet's initialize_scales for the regressors, one warp per series: a first pass for min, max, the {0, 1} test,
// non-finite values and the sum, a second for sum (x - mu)^2 (the two-pass form of pandas' nanvar).  Fewer than two
// distinct values, or a binary column under 'auto', or standardize = 0: (mu, std) = (0, 1).  A non-finite value: (NaN,
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

}  // namespace pb200
