// Launch entry points of the per-seasonality-class translation units (fit_inst.cu).
#pragma once
#include <cuda_runtime.h>

namespace pb200 {
struct FitArgs;
#define PB200_DECL(m) \
    cudaError_t launch_fit_mask##m(int nt, int logi, int reg, const FitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ);
PB200_DECL(0) PB200_DECL(1) PB200_DECL(2) PB200_DECL(3) PB200_DECL(4) PB200_DECL(5) PB200_DECL(6) PB200_DECL(7)
#undef PB200_DECL
}  // namespace pb200

namespace pb200 {
// grouped-lanes day-table kernel (fit_group_inst.cu): g = lanes per series (8 | 16)
cudaError_t launch_fit_group(int g, int logi, int mult, int seas, const FitArgs& a, int grid, cudaStream_t st, int* occ);
size_t fit_group_plane_doubles(int tmax, int g);      // global workspace per series slot (y pairs + L-BFGS history)
}  // namespace pb200

namespace pb200 {
// fit class of the models with a seasonality table (fit_table.cu): one warp per series, dynamic shared memory of
// fit_table_smem(ppad) bytes
struct TableFitArgs;
cudaError_t launch_fit_table(int logi, const TableFitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ);
size_t fit_table_smem(int ppad);
// ... with regressors (DESIGN §19): fit_table_reg_smem(ppad) bytes of dynamic shared memory
struct RegTableFitArgs;
cudaError_t launch_fit_table_reg(int logi, const RegTableFitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ);
size_t fit_table_reg_smem(int ppad);
}  // namespace pb200
