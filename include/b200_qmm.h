/*
 * b200_qmm.h -- C ABI of libb200qmm.so: the H100 (sm_90a) implementation of ggml's quantised mat-mul hot path.
 *
 * This is the kernel-level boundary.  The reference-facing drop-in boundary (the ggml backend plugin that stock
 * llama.cpp binaries dlopen through GGML_BACKEND_PATH) is declared in include/ggml-b200.h and is a thin C++ layer
 * over these entry points.
 *
 * Conventions
 *   - plain C: pointers, sizes, ints.  No torch / ggml types.  `type` is the numeric value of enum ggml_type
 *     (ggml/include/ggml.h:388-410): Q4_0=2, Q8_0=8, Q4_K=12, Q5_K=13, Q6_K=14.
 *   - *_dev pointers are CUDA device pointers on the current device; `stream` is a cudaStream_t passed as void*
 *     (NULL = default stream).  All calls are asynchronous on `stream` unless stated otherwise.
 *   - return value: 0 on success, otherwise a negative B200_E_* code; b200_qmm_last_error() gives the text.
 *     There is no CPU fallback: without a usable sm_90 device every compute call fails with B200_E_NO_DEVICE.
 *   - matrix layout is ggml's (ggml/include/ggml.h:1425-1431): weight src0 = [K, M] quantised along K, row m at
 *     w + m*row_stride bytes; activation src1 = [K, N] f32, column n at x + n*ldx floats; dst = [M, N] f32,
 *     column n at dst + n*ldd floats.
 *   - weight buffers must be readable up to the next 16-byte boundary after their last byte (cudaMalloc and the
 *     ggml buffer type guarantee this); Q4_K/Q5_K weights must be 16-byte aligned, the others 2-byte aligned.
 */
#ifndef B200_QMM_H
#define B200_QMM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#define B200_QMM_ABI_VERSION 1

#define B200_OK              0
#define B200_E_INVALID      -1   /* bad type / shape (K not a multiple of the block size, N < 0, ...)            */
#define B200_E_MISALIGNED   -2   /* pointer or stride violates the alignment contract above                        */
#define B200_E_WORKSPACE    -3   /* workspace too small                                                            */
#define B200_E_CUDA         -4   /* a CUDA call failed; see b200_qmm_last_error()                                  */
#define B200_E_NO_DEVICE    -5   /* no sm_90 device / driver                                                       */
#define B200_E_UNSUPPORTED  -6

B200_API int          b200_qmm_abi_version(void);
B200_API const char * b200_qmm_last_error(void);
/* number of usable sm_90 devices (0 if none); never fails */
B200_API int          b200_qmm_device_count(void);

/* ggml_row_size(type, k) (ggml/src/ggml.c): bytes of one quantised row of k weights; 0 if unsupported */
B200_API int64_t      b200_row_bytes(int type, int64_t k);

/* ---- replaces dequantize_row_{q4_0,q8_0,q4_K,q5_K,q6_K} (ggml/src/ggml-quants.c:459,553,1529,1731,1939) ----
 * Bit-exact fp32 output.  nrows rows of k weights; row r read at w_dev + r*row_stride, written at y_dev + r*ldy. */
B200_API int b200_dequantize_rows(int type, const void * w_dev, int64_t row_stride, float * y_dev, int64_t ldy,
                         int64_t nrows, int64_t k, void * stream);

/* ---- replaces from_float = quantize_row_q8_0 / quantize_row_q8_K applied to src1 in
 *      ggml_compute_forward_mul_mat (ggml/src/ggml-cpu/ggml-cpu.c:1322-1357; ggml-quants.c:276,2768) ----
 * Quantises n f32 rows of k activations to the activation format the CPU backend pairs with `weight_type`
 * (Q8_K for K-quants, Q8_0 otherwise), writing our device layout into ws_dev (>= b200_act_workspace_bytes()).
 * b200_act_layout() reports where the three planes live so a caller can inspect them:
 *   qs int8 [n][qs_stride], d f32 [n][d_stride], bsums int16 [n][bs_stride]        (see DESIGN.md "ActQ8").       */
B200_API size_t b200_act_workspace_bytes(int weight_type, int64_t n, int64_t k);
B200_API int    b200_quantize_act(int weight_type, const float * x_dev, int64_t ldx, int64_t n, int64_t k,
                         void * ws_dev, size_t ws_bytes, void * stream);
B200_API int    b200_act_layout(int weight_type, void * ws_dev, int64_t n, int64_t k,
                       void ** qs, void ** d, void ** bsums, int64_t * qs_stride, int64_t * d_stride, int64_t * bs_stride);
/* 0 = quantize_row_q8_0_ref rounding (default, oracle-pinned); 1 = the x86 AVX2 from_float variant
 * (ggml-cpu/arch/x86/quants.c:302-345).  Affects Q4_0/Q8_0 weights only. */
B200_API void   b200_set_q8_0_rounding(int mode);

/* ---- replaces ggml_compute_forward_mul_mat for quantised src0 (ggml/src/ggml-cpu/ggml-cpu.c:1254-1452) ----
 * dst[M,N] = W[M,K] . X[K,N].  N <= 8 runs the decode GEMV (mmvq regime, ggml-cuda/mmvq.cu), N > 8 the wgmma
 * prefill GEMM (mmq regime, ggml-cuda/mmq.cu).  ws_dev >= b200_mul_mat_workspace_bytes(). */
B200_API size_t b200_mul_mat_workspace_bytes(int type, int64_t M, int64_t N, int64_t K);
B200_API int    b200_mul_mat(int type, const void * w_dev, int64_t row_stride, int64_t M, int64_t K,
                    const float * x_dev, int64_t ldx, int64_t N, float * dst_dev, int64_t ldd,
                    void * ws_dev, size_t ws_bytes, void * stream);
/* The decode GEMV alone, on activations already quantised into ws_dev by b200_quantize_act(type, ..., n, k, ws_dev)
 * (n <= 8).  Lets a caller quantise once and reuse it for several weight matrices (attn_q/k/v, ffn_gate/up), and
 * lets the bench time the HBM-bound kernel in isolation. */
B200_API int    b200_gemv_q8(int type, const void * w_dev, int64_t row_stride, int64_t M, int64_t K,
                    void * ws_dev, int64_t n, float * dst_dev, int64_t ldd, void * stream);
/* The fused decode mat-vec the backend launches for a Llama layer (csrc/gemv3.cu): up to 3 same-type K-quant matrices that
 * share ONE f32 activation vector x[K].  If norm_w != NULL, x is first RMS-normalised and multiplied by norm_w (ggml
 * RMS_NORM + MUL, eps); the vector is quantised to Q8_K inside the kernel.  mode 0: dst[i] = W_i x;  mode 1: dst[0] = W_0 x +
 * residual[0] (ggml ADD);  mode 2 (nmat == 2, M equal): dst[0] = silu(W_0 x) * (W_1 x) (ggml GLU SWIGLU). */
B200_API int    b200_fused_matvec(int type, int nmat, const void * const * w_dev, const int64_t * row_stride, const int64_t * M, int64_t K,
                    const float * x_dev, const float * norm_w_dev, float eps, int mode, const float * const * residual_dev,
                    float * const * dst_dev, void * stream);
/* A chain of n fused mat-vecs (each with the semantics of one b200_fused_matvec call; arrays of length n, per-matrix arrays --
 * type, w_dev, row_stride, M, dst_dev -- of length 3n; the up-to-3 matrices of a phase may have different K-quant types)
 * executed as ONE launch of the persistent dataflow decode kernel (csrc/decode_flow.cu): one resident CTA per SM, no grid
 * barrier -- a phase whose x or residual is the dst of an earlier phase reads it through tagged slots as soon as it is
 * produced -- and one weight stream per CTA that runs ahead across phases.  This is the mat-vec part of what the ggml backend
 * records from a one-token llama graph.  Every dst is also written to its plain buffer (visible after the launch). */
B200_API int    b200_matvec_program(int n, const int * type, const int * nmat, const void * const * w_dev, const int64_t * row_stride, const int64_t * M,
                    const int64_t * K, const float * const * x_dev, const float * const * norm_w_dev, const float * eps, const int * mode,
                    const float * const * residual_dev, float * const * dst_dev, void * stream);
/* Host-only introspection of the persistent kernel's work plan for one mat-vec phase (no GPU needed): plan[0..7] = k-segments per
 * row, blocks per segment, rows per warp step, rows per ring piece of matrix 0/1/2, hidden-state flag, ring slot bytes. */
B200_API int    b200_flow_plan(int nmat, const int * type, const int64_t * M, int64_t K, const int64_t * row_stride, int mode, int has_norm,
                    int grid, int * plan);
/* host-only self-test of the decode-program recorder for the meta backend's node order (-sm tensor): 0 = the attention phase names the q vector
   remembered when ROPE(q) was postponed, not a later vector at the same address (ggml-alloc recycles the q mat-mul's buffer there) */
B200_API int    b200_flow_selftest_postponed_rope(void);
B200_API size_t b200_flow_slot_bytes(void);
/* path control for tests/benchmarks: 0 = auto, 1 = always GEMV (column chunks of 8), 2 = always GEMM */
B200_API void   b200_set_mul_mat_path(int path);
/* decode kernel generation: 2 = block-per-lane bulk-copy kernel where it applies (default), 1 = first generation */
B200_API void   b200_set_gemv_variant(int variant);

/* ---- replaces ggml_compute_forward_mul_mat_id (ggml/src/ggml-cpu/ggml-cpu.c:1534-1707) ----
 * as = [K, M, n_expert] (expert e at w_dev + e*expert_stride), b = [K, nb1, T] f32 contiguous (nb1 = n_used or 1),
 * ids = [n_used, T] int32 on the device (row t at ids_dev + t*ids_stride), dst = [M, n_used, T] f32 contiguous:
 * dst[:, s, t] = as[:, :, ids[s, t]] . b[:, s % nb1, t].  Routing happens on the device (no host sync). */
B200_API size_t b200_mul_mat_id_workspace_bytes(int type, int64_t M, int64_t K, int64_t n_used, int64_t T, int64_t nb1);
B200_API int    b200_mul_mat_id(int type, const void * w_dev, int64_t row_stride, int64_t expert_stride, int64_t n_expert,
                       int64_t M, int64_t K, const float * b_dev, int64_t nb1, const int32_t * ids_dev, int64_t ids_stride,
                       int64_t n_used, int64_t T, float * dst_dev, void * ws_dev, size_t ws_bytes, void * stream);

/* ---- end-to-end convenience: HOST activations in, HOST result out (weights stay resident in HBM) ----
 * Copies x_host (pinned or pageable) H2D, runs b200_mul_mat, copies dst D2H and synchronises `stream`.
 * scratch_dev >= N*K*4 + M*N*4 + b200_mul_mat_workspace_bytes() bytes. */
B200_API size_t b200_mul_mat_host_scratch_bytes(int type, int64_t M, int64_t N, int64_t K);
B200_API int    b200_mul_mat_host(int type, const void * w_dev, int64_t row_stride, int64_t M, int64_t K,
                         const float * x_host, int64_t N, float * dst_host,
                         void * scratch_dev, size_t scratch_bytes, void * stream);

/* number of kernels this library has launched since load (for the bench's gpu_launches claim) */
B200_API uint64_t b200_qmm_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_QMM_H */
