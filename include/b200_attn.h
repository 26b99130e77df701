/*
 * b200_attn.h -- the attention entry points of libb200qmm.so (conventions, B200_API and the B200_E_* codes: b200_qmm.h).
 *
 * b200_flash_attn and b200_attn_program expose the attention kernels the ggml backend runs -- the prefill kernels of
 * FLASH_ATTN_EXT and the decode kernel's attention phase -- so that tests can check them against a float64 reference.
 * They call the code the backend calls and compute nothing it does not.
 *
 * They live in a header of their own: the plugin's C++ objects (backend/) compile against b200_qmm.h, and a checkout
 * without the reference sources links objects built elsewhere only when the headers they were compiled against are
 * unchanged.  The plugin does not use these two entry points, so declaring them here leaves those objects valid.
 */
#ifndef B200_ATTN_H
#define B200_ATTN_H

#include "b200_qmm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- FLASH_ATTN_EXT on the prefill kernels ----
 * Each tensor is a device pointer with ggml's ne[4] / nb[4] (byte strides), so views and permuted layouts are given exactly
 * as llama builds them: q f32 [DK, N, H, B], k f16 [DK, n_kv, Hkv, Bk], v f16 [DV, n_kv, Hkv, Bv], mask f16
 * [>= n_kv, >= N, H / r, B / r'] or NULL, dst f32 [DV, H, N, B].  H must be a multiple of Hkv and B of Bk, Bv (broadcast).
 * Semantics of ggml_compute_forward_flash_attn_ext_f16 (ggml/src/ggml-cpu/ops.cpp): q is rounded to f16, s = scale * q.k
 * (softcap != 0: softcap * tanh(s / softcap)) + mask, softmax over the keys whose mask is not -inf, a row with none gives 0.
 * path: 0 = what the backend runs (tensor-core kernel for >= 16 rows where the shape fits, else the scalar kernel),
 * 1 = the scalar kernel (D a multiple of 32, <= 256), 2 = the tensor-core kernel (D in {64, 128}, >= 16 rows).  A shape the
 * requested kernel does not handle returns B200_E_UNSUPPORTED; there is no fall-back to the other kernel.
 * ws_dev: scratch for the tile-activity pre-pass of the tensor-core kernel (>= b200_flash_attn_workspace_bytes(); NULL = no
 * pre-pass, every kv tile is visited). */
B200_API size_t b200_flash_attn_workspace_bytes(const int64_t * q_ne, const int64_t * k_ne, const int64_t * mask_ne);
B200_API int    b200_flash_attn(const float * q_dev, const int64_t * q_ne, const int64_t * q_nb,
                       const void * k_dev, const int64_t * k_ne, const int64_t * k_nb,
                       const void * v_dev, const int64_t * v_ne, const int64_t * v_nb,
                       const void * mask_dev, const int64_t * mask_ne, const int64_t * mask_nb,
                       float * dst_dev, const int64_t * dst_ne, const int64_t * dst_nb,
                       float scale, float softcap, void * ws_dev, size_t ws_bytes, int path, void * stream);

/* ---- the decode kernel's attention phase ----
 * One launch of the persistent decode kernel holding the attention phase of one token (ROPE(q), ROPE(k), K/V cache store,
 * FLASH_ATTN_EXT over the cache), optionally preceded by the fused q|k|v mat-vec phase that feeds it through tagged slots --
 * the phases the ggml backend records for a Llama layer (FlowBuilder::add_matvec / add_attn).  Pointers are device pointers. */
typedef struct b200_attn_args {
    /* w_qkv[0] == NULL: q, k, v are read from the plain vectors below.  Otherwise q | k | v = W_i . q8_K(rms_norm(x) * norm_w)
     * (K-quant weights, [n_embd] -> [head_dim * n_head | n_head_kv | n_head_kv]) are computed in the same launch and also
     * written to q, k, v. */
    int           type_qkv[3];
    const void *  w_qkv[3];
    int64_t       row_stride_qkv[3];
    const float * x;                    /* f32 [n_embd] */
    const float * norm_w;               /* f32 [n_embd] or NULL */
    int64_t       n_embd;
    float         eps;
    float *       q;                    /* f32 [head_dim * n_head], before ROPE */
    float *       k;                    /* f32 [head_dim * n_head_kv], before ROPE */
    float *       v;                    /* f32 [head_dim * n_head_kv] */
    /* ROPE (ggml_rope_ext's parameters; mode 0 or 2) */
    int           n_head, n_head_kv, head_dim, n_dims, rope_mode, n_ctx_orig;
    float         freq_base, freq_scale, ext_factor, attn_factor, beta_fast, beta_slow;
    const float * freq_factors;         /* f32 [n_dims / 2] or NULL */
    const int32_t * pos;                /* i32 [1] */
    /* the cache rows the new k / v are stored to (f16, head after head): row kpos[0] / vpos[0] */
    void *        k_cache;
    int64_t       k_row_bytes;
    void *        v_cache;
    int64_t       v_row_bytes;
    const int64_t * kpos;
    const int64_t * vpos;
    /* the K / V views attention reads: f16 [head_dim, n_kv, n_head_kv], byte strides of a key and of a kv head */
    const void *  kview;
    int64_t       k_nb1, k_nb2;
    const void *  vview;
    int64_t       v_nb1, v_nb2;
    int           n_kv;
    const void *  mask;                 /* f16 [n_kv] or NULL */
    float         scale, softcap;
    float *       dst;                  /* f32 [head_dim * n_head] */
} b200_attn_args;
/* head_dim must be 128.  *nsplit (may be NULL) receives the number of CTAs each head was split over. */
B200_API int    b200_attn_program(const b200_attn_args * args, int * nsplit, void * stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_ATTN_H */
