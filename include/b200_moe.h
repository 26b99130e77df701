/*
 * b200_moe.h -- the MUL_MAT_ID test entry points of libb200qmm.so (conventions, B200_API and the B200_E_* codes: b200_qmm.h).
 *
 * b200_mul_mat_id_path and b200_moe_route expose the kernels the ggml backend runs for GGML_OP_MUL_MAT_ID -- the routed decode
 * GEMV, the grouped wgmma GEMM and the device router that feeds it -- so that tests can check each of them against the oracle.
 * They call the code the backend calls and compute nothing it does not.
 *
 * They live in a header of their own for the reason b200_attn.h does: the plugin's C++ objects compile against b200_qmm.h, and a
 * checkout without the reference sources links objects built elsewhere only when the headers they were compiled against are
 * unchanged.
 */
#ifndef B200_MOE_H
#define B200_MOE_H

#include "b200_qmm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- MUL_MAT_ID on a chosen kernel ----
 * Arguments and semantics as for b200_mul_mat_id in b200_qmm.h: dst[:, s, t] = as[:, :, ids[s, t]] . b[:, s % nb1, t], ids row t at
 * ids_dev + t * ids_stride (int32 elements; llama passes the first n_used rows of an [n_expert, T] argsort, ids_stride = n_expert).
 * path: 0 = what the backend runs for the node (the grouped GEMM for a K-quant with T * n_used >= 32 and n_expert <= 256, the
 *           routed GEMV otherwise, and also when the GEMM cannot take the operands' alignment),
 *       1 = the routed GEMV (token chunks of 65535 / n_used, the grid's y limit),
 *       2 = the grouped GEMM: B200_E_UNSUPPORTED for Q4_0 / Q8_0, n_expert > 256 or weights / activations it cannot align;
 *           there is no fall-back to the GEMV.
 * *taken (may be NULL) receives the kernel that ran: 1 GEMV, 2 grouped GEMM (0 when nothing ran).
 * ws_dev >= b200_mul_mat_id_path_workspace_bytes() (enough for either kernel). */
B200_API size_t b200_mul_mat_id_path_workspace_bytes(int type, int64_t M, int64_t K, int64_t n_expert, int64_t n_used, int64_t T, int64_t nb1);
B200_API int    b200_mul_mat_id_path(int type, const void * w_dev, int64_t row_stride, int64_t expert_stride, int64_t n_expert,
                       int64_t M, int64_t K, const float * b_dev, int64_t nb1, const int32_t * ids_dev, int64_t ids_stride,
                       int64_t n_used, int64_t T, float * dst_dev, void * ws_dev, size_t ws_bytes, int path, int * taken, void * stream);

/* ---- the grouped GEMM's router on its own ----
 * Sorts the T * n_used (token, slot) jobs j = t * n_used + s by expert into column tiles of 128: experts in ascending order, each
 * expert's tiles contiguous, its jobs in the first slots of its run (in no fixed order; the rest of the run is -1).
 * tile_expert_dev int32 [max_tiles]: the expert of each tile, -1 past the live tiles; col_src_dev / col_dst_dev int32 [max_tiles * 128]:
 * per column slot, the activation column t * nb1 + (nb1 == 1 ? 0 : s) and the job j, -1 in unused slots.  Jobs whose id is outside
 * [0, n_expert) are left out.  max_tiles = b200_moe_route_max_tiles(n_expert, n_used, T) = ceil(T * n_used / 128) + n_expert.
 * Returns max_tiles, or a negative B200_E_* code (B200_E_UNSUPPORTED for n_expert > 256). */
B200_API int64_t b200_moe_route_max_tiles(int64_t n_expert, int64_t n_used, int64_t T);
B200_API int64_t b200_moe_route(const int32_t * ids_dev, int64_t ids_stride, int64_t n_expert, int64_t n_used, int64_t T, int64_t nb1,
                       int32_t * tile_expert_dev, int32_t * col_src_dev, int32_t * col_dst_dev, void * stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_MOE_H */
