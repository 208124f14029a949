// Outlier flags and the compaction of the kept rows for sm_90a (DESIGN §16): after the in-sample predict, a history row
// is an outlier when its y lies outside [yhat_lower, yhat_upper]; the rows that are not make a packed batch that the fit
// takes as it is.  Two passes, as the backtest plan's: counts per series, the caller's exclusive scan, the rows.
//
// One warp per series, 32 consecutive rows per step: the flags of a step are one ballot, a kept row's place is the popc
// of the kept rows before it in the step plus those of the earlier steps.  No atomics: a series' outputs depend on that
// series' rows only, in their order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/prophet_b200.h"

namespace pb200 {
namespace insample {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

struct FlagArgs {
    const void* y;              // [rows], element type y_dtype (PB200_Y_*)
    int y_dtype;
    const long long* offsets;   // [n_series + 1]: series i owns rows [offsets[i], offsets[i + 1])
    long long n_series;
    const double* lower;        // [rows]
    const double* upper;
    unsigned char* flag;        // [rows]: 1 when (double)y < lower or (double)y > upper (a NaN bound never flags)
    int* kept;                  // [n_series]: rows not flagged
};

struct CompactArgs {
    const long long* ds;        // [rows]
    const void* y;
    int y_dtype;
    const long long* offsets;
    long long n_series;
    const unsigned char* flag;
    const long long* kept_off;  // [n_series + 1]: exclusive scan of FlagArgs::kept
    long long* ds_out;          // [kept_off[n_series]]
    void* y_out;                // [kept_off[n_series]], element type y_dtype
};

__device__ __forceinline__ double y_value(const void* y, const int dt, const long long r) {
    if (dt == PB200_Y_F64) return ((const double*)y)[r];
    if (dt == PB200_Y_F32) return (double)((const float*)y)[r];
    return (double)((const int*)y)[r];
}

__global__ void __launch_bounds__(THREADS) outlier_counts_kernel(const FlagArgs a) {
    const int lane = threadIdx.x & 31;
    const long long step = (long long)gridDim.x * WARPS;
    for (long long s = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5); s < a.n_series; s += step) {
        const long long r1 = a.offsets[s + 1];
        int kept = 0;
        for (long long b = a.offsets[s]; b < r1; b += 32) {
            const long long r = b + lane;
            bool keep = false;
            if (r < r1) {
                const double v = y_value(a.y, a.y_dtype, r);
                const bool out = v < a.lower[r] || v > a.upper[r];
                a.flag[r] = out ? 1 : 0;
                keep = !out;
            }
            kept += __popc(__ballot_sync(0xffffffffu, keep));
        }
        if (lane == 0) a.kept[s] = kept;
    }
}

__global__ void __launch_bounds__(THREADS) outlier_compact_kernel(const CompactArgs a) {
    const int lane = threadIdx.x & 31;
    const unsigned before = (1u << lane) - 1u;
    const long long step = (long long)gridDim.x * WARPS;
    for (long long s = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5); s < a.n_series; s += step) {
        const long long r1 = a.offsets[s + 1];
        long long w = a.kept_off[s];
        for (long long b = a.offsets[s]; b < r1; b += 32) {
            const long long r = b + lane;
            const bool keep = r < r1 && a.flag[r] == 0;
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                const long long o = w + __popc(m & before);
                a.ds_out[o] = a.ds[r];
                if (a.y_dtype == PB200_Y_F64) ((double*)a.y_out)[o] = ((const double*)a.y)[r];
                else ((int*)a.y_out)[o] = ((const int*)a.y)[r];     // int32 and float32: the 4 bytes as they are
            }
            w += __popc(m);
        }
    }
}

}  // namespace insample
}  // namespace pb200
