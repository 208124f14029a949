// The scorer's join of the regressors' future values onto the forecast grid for sm_90a (DESIGN §20): for every model and
// every point of its future grid, the row of the model's group in a packed table whose timestamp is exactly the point's.
//
// One warp per model, lane l takes the grid points l, l + 32, ...: each binary-searches its timestamp among the group's
// rows (ascending within a group, as the pack leaves them), so a point costs log2(rows) loads and the R values of its row.
// Table rows that are no point of the grid are never read.  A point without a row gets NaN in every plane and counts as
// missing; the model's count and its first missing timestamp (the grid is ascending, so the least missing index) come
// from one warp reduction.  No atomics: a model's outputs depend on its own grid and group only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb200 {
namespace join {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;

struct JoinArgs {
    const long long* tab_ds;       // [rows] int64 ns, ascending within a group
    const long long* tab_offsets;  // [n_groups + 1]: group g owns rows [tab_offsets[g], tab_offsets[g + 1])
    const double* tab_reg;         // [R][rows]
    long long rows;
    int R;
    const long long* model_group;  // [n_models]: the model's group, -1 when the table has none
    const long long* future_ds;    // [n_models][horizon]
    long long n_models;
    int horizon;
    double* future_reg;            // [R][n_models * horizon]: pb200_predict_regressors_*'s d_future_reg
    int* missing;                  // [n_models]: grid points without a row
    long long* first_missing;      // [n_models]: timestamp of the first of them, INT64_MIN when there is none
};

__global__ void __launch_bounds__(THREADS) join_future_regressors_kernel(const JoinArgs a) {
    const int lane = threadIdx.x & 31;
    const long long plane = a.n_models * (long long)a.horizon;
    const long long step = (long long)gridDim.x * WARPS;
    for (long long m = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5); m < a.n_models; m += step) {
        const long long g = a.model_group[m];
        const long long lo0 = g >= 0 ? a.tab_offsets[g] : 0;
        const long long hi0 = g >= 0 ? a.tab_offsets[g + 1] : 0;
        int miss = 0;
        int first = a.horizon;                       // least missing grid index of this lane
        for (int h = lane; h < a.horizon; h += 32) {
            const long long p = m * (long long)a.horizon + h;
            const long long t = a.future_ds[p];
            long long lo = lo0, hi = hi0;            // lower bound of t in [lo0, hi0)
            while (lo < hi) {
                const long long mid = lo + ((hi - lo) >> 1);
                if (a.tab_ds[mid] < t) lo = mid + 1;
                else hi = mid;
            }
            const bool hit = lo < hi0 && a.tab_ds[lo] == t;
            for (int r = 0; r < a.R; ++r)
                a.future_reg[r * plane + p] = hit ? a.tab_reg[r * a.rows + lo] : __longlong_as_double(0x7ff8000000000000ll);
            if (!hit) {
                ++miss;
                first = min(first, h);
            }
        }
        for (int o = 16; o > 0; o >>= 1) {
            miss += __shfl_xor_sync(0xffffffffu, miss, o);
            first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
        }
        if (lane == 0) {
            a.missing[m] = miss;
            a.first_missing[m] = miss ? a.future_ds[m * (long long)a.horizon + first] : (long long)INT64_MIN;
        }
    }
}

}  // namespace join
}  // namespace pb200
