// One translation unit per seasonality class (compile with -DPB200_MASK=0..7):
// bit0 yearly (order 10), bit1 weekly (order 3), bit2 daily (order 4) -- the Fourier
// orders Prophet.set_auto_seasonalities uses.  Instantiates fit_kernel for
// NT in {32, 128} x growth in {linear, logistic}.
#include "fit_kernel.cuh"
#include "launch.h"

#ifndef PB200_MASK
#error "compile with -DPB200_MASK=<0..7>"
#endif

namespace pb200 {

constexpr int YO = (PB200_MASK & 1) ? 10 : 0;
constexpr int WO = (PB200_MASK & 2) ? 3 : 0;
constexpr int DO = (PB200_MASK & 4) ? 4 : 0;

template <int NT, bool LOGI, int REG>
static cudaError_t launch_one(const FitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ) {
    auto kern = fit_kernel<NT, LOGI, YO, WO, DO, REG>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (occ) {
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, kern, NT, smem);
        return e;
    }
    kern<<<grid, NT, smem, st>>>(a);
    return cudaGetLastError();
}

#define PB200_CAT_(a, b) a##b
#define PB200_CAT(a, b) PB200_CAT_(a, b)

template <int NT>
static cudaError_t launch_nt(int logi, int reg, const FitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ) {
    if constexpr (PB200_MASK == 6 && NT == 32) {   // seasonal-table variants: weekly + daily, warp per series
        if (reg == 2) return logi ? launch_one<NT, true, 2>(a, grid, smem, st, occ) : launch_one<NT, false, 2>(a, grid, smem, st, occ);
        if (reg == 3) return logi ? launch_one<NT, true, 3>(a, grid, smem, st, occ) : launch_one<NT, false, 3>(a, grid, smem, st, occ);
    }
    if (reg >= 2) return cudaErrorInvalidValue;
    if constexpr (PB200_MASK != 0) {        // the regular-grid variant only differs when there are Fourier features
        if (reg) return logi ? launch_one<NT, true, 1>(a, grid, smem, st, occ) : launch_one<NT, false, 1>(a, grid, smem, st, occ);
    }
    return logi ? launch_one<NT, true, 0>(a, grid, smem, st, occ) : launch_one<NT, false, 0>(a, grid, smem, st, occ);
}

cudaError_t PB200_CAT(launch_fit_mask, PB200_MASK)(int nt, int logi, int reg, const FitArgs& a, int grid, size_t smem,
                                                   cudaStream_t st, int* occ) {
    if (nt == 32) return launch_nt<32>(logi, reg, a, grid, smem, st, occ);
    if (nt == 128) return launch_nt<128>(logi, reg, a, grid, smem, st, occ);
    return cudaErrorInvalidValue;
}

}  // namespace pb200
