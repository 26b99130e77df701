// qmm_kernels.cuh -- launch-side declarations shared by the .cu files and the C-ABI (c_abi.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace qmm {

void note_launch(int n = 1);          // bump the library-wide kernel launch counter (c_abi.cu)
void set_q8_0_mode(int m);            // act_quant.cu
int  get_q8_0_mode();
bool pdl_attr_always();           // GGML_B200_PDL_ATTR_ALWAYS (diagnosis): pass the attribute (value 0) even when PDL is off
void set_pdl(bool on);                // programmatic dependent launch for the small decode kernels (default on)
bool pdl_enabled();
void set_gemv_variant(int v);         // gemv.cu: 1 = first-generation kernel only, 2 = gemv2.cu where it applies

// Quantised activation operand in HBM (see qmm_formats.cuh for the field meaning).  Column n of a batch lives at
// qs + n*qs_stride, d + n*d_stride, bsums + n*bs_stride.
struct ActQ8 {
    int8_t  * qs;
    float   * d;
    int16_t * bsums;
    int64_t   qs_stride, d_stride, bs_stride;
};

// Workspace carving for N columns of K activations paired with weight type t.
size_t act_workspace_bytes(int weight_type, int64_t N, int64_t K);
ActQ8  act_carve(int weight_type, void * ws, int64_t N, int64_t K);

// f32 rows -> ActQ8 (bit-exact quantize_row_q8_K_ref / quantize_row_q8_0_ref values).  x row n at x + n*ldx floats.
cudaError_t launch_quantize_act(int weight_type, const float * x, int64_t ldx, int64_t N, int64_t K, const ActQ8 & out, cudaStream_t st);

// Fused decode prologue: y = rms_norm(x) * w_norm (ggml RMS_NORM + MUL), then quantise y.  x is one row of K floats.
cudaError_t launch_rmsnorm_quantize_act(int weight_type, const float * x, const float * w_norm, float eps, float * y_out /*nullable*/,
                                        int64_t K, const ActQ8 & out, cudaStream_t st);

// Bit-exact dequantize_row_*: nrows rows of k weights, row r at w + r*row_stride bytes -> y + r*ldy floats.
cudaError_t launch_dequantize(int type, const void * w, int64_t row_stride, float * y, int64_t ldy, int64_t nrows, int64_t k, cudaStream_t st);

struct GemvArgs {
    const uint8_t * w;          // weights; row m of matrix z at w + expert(z)*expert_stride + m*row_stride
    int64_t row_stride;         // bytes
    int64_t expert_stride;      // bytes (0 when ids == nullptr)
    int     M, K;
    int     ncols;              // activation columns handled per z (1..8); 1 when ids != nullptr
    int     nz;                 // gridDim.y: 1 for MUL_MAT; n_used*T for MUL_MAT_ID
    ActQ8   act;
    float * dst;                // dst[(z*ncols_z + n)*ldd + m]
    int64_t ldd;
    const float * residual;     // optional: added to dst (same indexing); nullptr = none
    // MUL_MAT_ID routing (device pointers); ids == nullptr -> plain MUL_MAT
    const int32_t * ids;        // ids[t*ids_stride + s]
    int64_t ids_stride;
    int     n_used, nb1, n_expert;
};
cudaError_t launch_gemv(int type, const GemvArgs & a, cudaStream_t st);

// Fused decode mat-vec (gemv3.cu): up to 3 same-type matrices sharing one activation vector, activation given as f32
// (optionally RMS-normalised and multiplied by norm_w first) and quantised in the kernel prologue, or pre-quantised.
struct FusedGemvArgs {
    int             nmat;
    const uint8_t * w[3];
    int64_t         row_stride[3];
    int             M[3];
    float *         dst[3];
    const float *   residual[3];      // mode 1
    int             K;
    const float *   x;                // f32 activation (K floats); nullptr -> use `act`
    const float *   norm_w;           // RMS_NORM weight (has_norm)
    float           eps;
    int             has_norm;
    ActQ8           act;
    int             mode;             // 0 store, 1 + residual, 2 SwiGLU pair (dst[0] = silu(W0 x) * (W1 x))
    int             pdl;              // launch with programmatic stream serialisation
    unsigned *      counter;          // zeroed ticket counter for dynamic row-group distribution (nullptr = static split)
    const uint8_t * next_w[3];        // weights of the NEXT fused launch: prefetched into the 50 MB L2 while this launch runs
    int64_t         next_bytes[3];
};
cudaError_t launch_fused_gemv(int type, const FusedGemvArgs & a, cudaStream_t st);

// Prefill GEMM (wgmma): dst[M,N] = W[M,K] . X[K,N] with X pre-quantised to ActQ8-derived fp16 integer operands.
struct GemmArgs {
    const uint8_t * w; int64_t row_stride; int M, K, N;
    const float * x; int64_t ldx;
    float * dst; int64_t ldd;
    void * workspace; size_t workspace_bytes;
    bool reuse_operands;   // the workspace still holds the operand images of the same (x, N, K): skip the activation pre-pass
};
size_t      gemm_workspace_bytes(int type, int64_t M, int64_t N, int64_t K);
cudaError_t launch_gemm(int type, const GemmArgs & a, cudaStream_t st);
// Q4_0 / Q8_0 (gemm_legacy_wgmma.cu); launch_gemm and gemm_workspace_bytes dispatch to these
size_t      gemm_legacy_workspace_bytes(int type, int64_t M, int64_t N, int64_t K);
cudaError_t launch_gemm_legacy(int type, const GemmArgs & a, cudaStream_t st);
// grouped GEMM for MUL_MAT_ID with many tokens: w [K, M, n_expert], x columns [K] at x + (t * nb1 + (nb1 == 1 ? 0 : s)) * ldx, ids[t * ids_stride + s],
// dst column (t * n_used + s) at dst + column * ldd
struct GemmGroupedArgs {
    const uint8_t * w; int64_t row_stride, expert_stride; int M, K, n_expert;
    const float * x; int64_t ldx; int nb1;
    const int32_t * ids; int64_t ids_stride; int T, n_used;
    float * dst; int64_t ldd;
    void * workspace; size_t workspace_bytes;
};
size_t      gemm_grouped_workspace_bytes(int type, int64_t M, int64_t jobs, int64_t n_expert, int64_t K);
cudaError_t launch_gemm_grouped(int type, const GemmGroupedArgs & a, cudaStream_t st);

// ---- one-shot NVLink all-reduce (allreduce.cu), used by the backend's ggml_backend_comm_* hooks
constexpr int ONESHOT_MAX_DEV = 8;
struct OneShotComm {
    int      n = 0;
    int      devs[ONESHOT_MAX_DEV] = {};
    float *  buf[ONESHOT_MAX_DEV] = {};      // per device: 2 sets x n slots x slot_floats
    unsigned * ctl[ONESHOT_MAX_DEV] = {};    // per device: flags[0..n) | seq @32 | block_counter @33 | finish_counter @34
    size_t   slot_floats = 0, set_floats = 0;
};
struct OneShotDev {
    int n, rank;
    size_t slot_floats, set_floats;
    float * buf;
    unsigned * flags;
    unsigned * seq, * block_counter, * finish_counter;
};
struct OneShotPeers {
    float *    buf[ONESHOT_MAX_DEV];
    unsigned * flags[ONESHOT_MAX_DEV];
};
cudaError_t oneshot_init(OneShotComm & c, const int * devs, int n, size_t max_bytes);
void        oneshot_free(OneShotComm & c);
cudaError_t oneshot_allreduce(OneShotComm & c, float * const * data, size_t count, const cudaStream_t * streams);


// Launch helper: programmatic stream serialisation lets kernel N+1 be scheduled while kernel N drains; kernels launched
// through it start with griddepcontrol.wait (pdl_prologue()) before touching their inputs.
#if defined(__CUDACC__)
__device__ __forceinline__ void pdl_prologue() {
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    asm volatile("griddepcontrol.wait;\n" ::: "memory");
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args &&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = at; cfg.numAttrs = (pdl_enabled() || pdl_attr_always()) ? 1 : 0;     // PDL off: a plain launch, no attribute at all
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

}  // namespace qmm
