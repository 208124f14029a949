// Extra regressors (pb200_options_v3, DESIGN §19): fbprophet 0.5's add_regressor.  A regressor is one more column of a
// table model's design matrix, after the active seasonal columns; its values come from the caller (one plane of
// [n_rows] doubles per regressor) and are standardised per series as fbprophet's initialize_scales does.
#pragma once
#include <cuda_runtime.h>

namespace pb200 {

constexpr int REG_MAX = 16;      // PB200_MAX_REGRESSORS

// the model's regressors as the host normalised them, passed by value
struct RegSpec {
    int R;
    int standardize[REG_MAX];    // PB200_STD_AUTO, 0 or 1
    double inv_sig2[REG_MAX];    // 1 / prior_scale^2, correctly rounded on the host
};

// the one form of a standardised value: the fit, the Newton retry and predict all evaluate it so
__host__ __device__ __forceinline__ double reg_value(const double x, const double mu, const double sd) { return (x - mu) / sd; }

}  // namespace pb200
