// Instantiations of the grouped-lanes fit kernel (fit_group.cuh): G in {8, 16} lanes per series x growth x
// seasonality mode for the weekly + daily day-table class, x growth for the class without seasonality.
#include <cstdlib>

#include "fit_group.cuh"
#include "launch.h"

namespace pb200 {

template <int G, bool LOGI, bool MULT, bool SEAS>
static cudaError_t launch_group_one(const FitArgs& a, int grid, cudaStream_t st, int* occ) {
    auto kern = grp::fit_group_kernel<G, LOGI, MULT, SEAS>;
    // PB200_GRP_PAD (A/B runs only): extra dynamic shared memory per CTA, i.e. fewer resident warps per SM
    static const size_t pad = getenv("PB200_GRP_PAD") ? (size_t)atoi(getenv("PB200_GRP_PAD")) : 0;
    const size_t smem = grp::group_smem_bytes<G, SEAS>() + pad;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (occ) return cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, kern, 32, smem);
    kern<<<grid, 32, smem, st>>>(a);
    return cudaGetLastError();
}

template <int G>
static cudaError_t launch_group_g(int logi, int mult, int seas, const FitArgs& a, int grid, cudaStream_t st, int* occ) {
    if (!seas) return logi ? launch_group_one<G, true, false, false>(a, grid, st, occ) : launch_group_one<G, false, false, false>(a, grid, st, occ);
    if (logi) return mult ? launch_group_one<G, true, true, true>(a, grid, st, occ) : launch_group_one<G, true, false, true>(a, grid, st, occ);
    return mult ? launch_group_one<G, false, true, true>(a, grid, st, occ) : launch_group_one<G, false, false, true>(a, grid, st, occ);
}

cudaError_t launch_fit_group(int g, int logi, int mult, int seas, const FitArgs& a, int grid, cudaStream_t st, int* occ) {
    if (g == 8) return launch_group_g<8>(logi, mult, seas, a, grid, st, occ);
    if (g == 16) return launch_group_g<16>(logi, mult, seas, a, grid, st, occ);
    return cudaErrorInvalidValue;
}

size_t fit_group_plane_doubles(int tmax, int g) {
    size_t d = grp::group_plane_doubles(tmax, g) + grp::GHIST;
    return (d + 1) & ~(size_t)1;
}

}  // namespace pb200

#ifdef PB200_PHASE_CLOCKS
// dev builds only (-DPB200_PHASE_CLOCKS): the grouped kernel's per-phase warp cycles summed since the last reset, in
// pb200::grp::PhaseClock order (n <= PC_N entries); waits for the device first.  Returns the number of entries, < 0 on error
extern "C" PB200_API int pb200_dev_phase_clocks(unsigned long long* h_out, int n, int reset) {
    if (n > pb200::grp::PC_N) n = pb200::grp::PC_N;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (h_out && n > 0 && cudaMemcpyFromSymbol(h_out, pb200::grp::g_phase_cycles, (size_t)n * sizeof(unsigned long long)) != cudaSuccess)
        return -1;
    if (reset) {
        static const unsigned long long zero[pb200::grp::PC_N] = {};
        if (cudaMemcpyToSymbol(pb200::grp::g_phase_cycles, zero, sizeof(zero)) != cudaSuccess) return -1;
    }
    return n;
}
#endif
