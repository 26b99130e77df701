// qmm_moe.cuh -- the MUL_MAT_ID grouped GEMM's router as a launch of its own (defined in gemm_tcgen05.cu), for the test entry
// points of include/b200_moe.h.  Declared here, not in qmm_kernels.cuh: the plugin's C++ objects are compiled against that header.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace qmm {

constexpr int MOE_TILE_COLS = 128;                 // columns per tile of the grouped GEMM (its GEMM_NT)

// tiles a launch covers: every expert may leave one partial tile
inline int64_t moe_max_tiles(int64_t jobs, int64_t n_expert) { return (jobs + MOE_TILE_COLS - 1) / MOE_TILE_COLS + n_expert; }

// moe_route_kernel: tile_expert [max_tiles], col_src / col_dst [max_tiles * MOE_TILE_COLS]; n_expert <= 256
cudaError_t launch_moe_route(const int32_t * ids, int64_t ids_stride, int T, int n_used, int nb1, int n_expert, int max_tiles,
                             int * tile_expert, int * col_src, int * col_dst, cudaStream_t st);

}  // namespace qmm
