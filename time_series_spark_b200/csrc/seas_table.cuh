// A model's seasonality table (pb200_options_v2, DESIGN §18): fbprophet's add_seasonality entries and non-default
// built-in orders, normalised on the host into the column order fbprophet's make_all_seasonality_features gives --
// the custom seasonalities in the order they were added, then yearly, weekly and daily.  Passed by value in the
// kernel arguments (at most 8 entries).  n == 0 is the default model: the compiled-in orders, today's kernels.
#pragma once
#include <cuda_runtime.h>

namespace pb200 {

constexpr int SEAS_TMAX = 8;     // entries per table
constexpr int SEAS_KMAX = 64;    // sum of 2 * order over the table
constexpr int SEAS_PMAX = 96;    // 3 + S + K: three vector elements per lane of the optimiser warp

struct SeasTab {
    int n;
    int order[SEAS_TMAX];
    // 0: always on (a custom seasonality, never auto-disabled); 1 | 2 | 4: the built-in (yearly | weekly | daily) whose
    // switch and set_auto_seasonalities rule decide, read from the series' built-in mask
    int kind[SEAS_TMAX];
    double period[SEAS_TMAX];        // days
    double inv_sig2[SEAS_TMAX];      // 1 / prior_scale^2, correctly rounded on the host
    // component plane of each entry (pb200_predict_components_*): PB200_COMP_YEARLY / WEEKLY / DAILY for a built-in or a
    // custom entry of that name, else PB200_N_COMPONENTS + its rank among the other custom entries
    int plane[SEAS_TMAX];
    int nplanes;                     // PB200_N_COMPONENTS + the custom entries not named like a built-in
};

// the table mask of a history (bit j: entry j is active) given its built-in mask (auto_seasonality_mask)
__host__ __device__ __forceinline__ int tab_mask(const SeasTab& t, const int builtin_mask) {
    int m = 0;
    for (int e = 0; e < t.n; ++e)
        if (t.kind[e] == 0 || (builtin_mask & t.kind[e])) m |= 1 << e;
    return m;
}

// Fourier columns of the active entries (0: none; the fit then carries fbprophet's single zero column)
__host__ __device__ __forceinline__ int tab_k(const SeasTab& t, const int mask) {
    int k = 0;
    for (int e = 0; e < t.n; ++e)
        if ((mask >> e) & 1) k += 2 * t.order[e];
    return k;
}

}  // namespace pb200
