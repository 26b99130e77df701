// c_abi.cu -- the extern "C" surface declared in include/b200_qmm.h.  Thin: argument checks, workspace carving,
// regime selection (decode GEMV vs prefill GEMM), error text.  No compute happens on the host and there is no CPU
// fallback: if CUDA is unusable every compute entry point fails loudly.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "../../include/b200_qmm.h"
#include "qmm_formats.cuh"
#include <vector>
#include <string.h>
#include "qmm_kernels.cuh"
#include "decode_flow.cuh"

namespace qmm {
static std::atomic<uint64_t> g_launches{0};
void note_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
static bool g_pdl = false;
void set_pdl(bool on) { g_pdl = on; }
bool pdl_enabled() { return g_pdl; }
bool pdl_attr_always() { static const bool v = getenv("GGML_B200_PDL_ATTR_ALWAYS") != nullptr; return v; }
}  // namespace qmm

using namespace qmm;

static thread_local char g_err[512] = "";
static int g_path = 0;

static int fail(int code, const char * what, cudaError_t e = cudaSuccess) {
    if (e != cudaSuccess) snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
    else snprintf(g_err, sizeof(g_err), "%s", what);
    return code;
}
static int from_cuda(cudaError_t e, const char * what) {
    if (e == cudaSuccess) return B200_OK;
    if (e == cudaErrorInvalidValue) return fail(B200_E_INVALID, what, e);
    if (e == cudaErrorMisalignedAddress) { cudaGetLastError(); return fail(B200_E_MISALIGNED, what, e); }
    if (e == cudaErrorNotSupported) return fail(B200_E_UNSUPPORTED, what, e);
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) return fail(B200_E_NO_DEVICE, what, e);
    return fail(B200_E_CUDA, what, e);
}
static bool type_ok(int t) { return block_bytes(t) != 0; }

extern "C" {

int b200_qmm_abi_version(void) { return B200_QMM_ABI_VERSION; }
const char * b200_qmm_last_error(void) { return g_err; }
uint64_t b200_qmm_launch_count(void) { return g_launches.load(); }

int b200_qmm_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    int ok = 0;
    for (int i = 0; i < n; i++) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess && major == 9) ok++;
    }
    return ok;
}

int64_t b200_row_bytes(int type, int64_t k) {
    if (!type_ok(type) || k < 0 || k % block_elems(type)) return 0;
    return k / block_elems(type) * block_bytes(type);
}

int b200_dequantize_rows(int type, const void * w, int64_t row_stride, float * y, int64_t ldy, int64_t nrows, int64_t k, void * stream) {
    if (!type_ok(type) || nrows < 0 || k < 0 || k % block_elems(type)) return fail(B200_E_INVALID, "b200_dequantize_rows: bad type/shape");
    return from_cuda(launch_dequantize(type, w, row_stride, y, ldy, nrows, k, (cudaStream_t)stream), "b200_dequantize_rows");
}

size_t b200_act_workspace_bytes(int wt, int64_t n, int64_t k) { return type_ok(wt) ? act_workspace_bytes(wt, n, k) : 0; }

int b200_quantize_act(int wt, const float * x, int64_t ldx, int64_t n, int64_t k, void * ws, size_t ws_bytes, void * stream) {
    if (!type_ok(wt) || n < 0 || k < 0 || k % block_elems(wt)) return fail(B200_E_INVALID, "b200_quantize_act: bad type/shape");
    if (ws_bytes < act_workspace_bytes(wt, n, k)) return fail(B200_E_WORKSPACE, "b200_quantize_act: workspace too small");
    return from_cuda(launch_quantize_act(wt, x, ldx, n, k, act_carve(wt, ws, n, k), (cudaStream_t)stream), "b200_quantize_act");
}

int b200_act_layout(int wt, void * ws, int64_t n, int64_t k, void ** qs, void ** d, void ** bsums, int64_t * qss, int64_t * ds, int64_t * bss) {
    if (!type_ok(wt)) return fail(B200_E_INVALID, "b200_act_layout: bad type");
    const ActQ8 a = act_carve(wt, ws, n, k);
    *qs = a.qs; *d = a.d; *bsums = a.bsums; *qss = a.qs_stride; *ds = a.d_stride; *bss = a.bs_stride;
    return B200_OK;
}

void b200_set_q8_0_rounding(int mode) { set_q8_0_mode(mode); }
void b200_set_mul_mat_path(int path) { g_path = path; }
void b200_set_gemv_variant(int v) { set_gemv_variant(v); }

size_t b200_mul_mat_workspace_bytes(int type, int64_t M, int64_t N, int64_t K) {
    if (!type_ok(type)) return 0;
    size_t a = act_workspace_bytes(type, N, K);
    size_t g = gemm_workspace_bytes(type, M, N, K);
    return (a > g ? a : g) + 256;
}

int b200_mul_mat(int type, const void * w, int64_t row_stride, int64_t M, int64_t K, const float * x, int64_t ldx, int64_t N,
                 float * dst, int64_t ldd, void * ws, size_t ws_bytes, void * stream) {
    if (!type_ok(type) || M < 0 || N < 0 || K <= 0 || K % block_elems(type)) return fail(B200_E_INVALID, "b200_mul_mat: bad type/shape");
    if (M == 0 || N == 0) return B200_OK;
    if (M > INT32_MAX || K > INT32_MAX || N > INT32_MAX) return fail(B200_E_INVALID, "b200_mul_mat: dimension too large");
    if (ws_bytes < b200_mul_mat_workspace_bytes(type, M, N, K)) return fail(B200_E_WORKSPACE, "b200_mul_mat: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const bool use_gemm = g_path == 2 || (g_path == 0 && N > 8 && gemm_workspace_bytes(type, M, N, K) != 0);
    if (use_gemm) {
        GemmArgs g{};
        g.w = (const uint8_t *)w; g.row_stride = row_stride; g.M = (int)M; g.K = (int)K; g.N = (int)N;
        g.x = x; g.ldx = ldx; g.dst = dst; g.ldd = ldd; g.workspace = ws; g.workspace_bytes = ws_bytes;
        return from_cuda(launch_gemm(type, g, st), "b200_mul_mat(gemm)");
    }
    const ActQ8 act = act_carve(type, ws, N, K);
    cudaError_t e = launch_quantize_act(type, x, ldx, N, K, act, st);
    if (e != cudaSuccess) return from_cuda(e, "b200_mul_mat(quantize)");
    for (int64_t n0 = 0; n0 < N; n0 += 8) {
        GemvArgs a{};
        a.w = (const uint8_t *)w; a.row_stride = row_stride; a.expert_stride = 0; a.M = (int)M; a.K = (int)K;
        a.ncols = (int)(N - n0 < 8 ? N - n0 : 8); a.nz = 1;
        a.act = act; a.act.qs += n0 * act.qs_stride; a.act.d += n0 * act.d_stride; a.act.bsums += n0 * act.bs_stride;
        a.dst = dst + n0 * ldd; a.ldd = ldd; a.residual = nullptr; a.ids = nullptr;
        e = launch_gemv(type, a, st);
        if (e != cudaSuccess) return from_cuda(e, "b200_mul_mat(gemv)");
    }
    return B200_OK;
}

int b200_gemv_q8(int type, const void * w, int64_t row_stride, int64_t M, int64_t K, void * ws, int64_t n, float * dst, int64_t ldd, void * stream) {
    if (!type_ok(type) || M < 0 || n < 1 || n > 8 || K <= 0 || K % block_elems(type)) return fail(B200_E_INVALID, "b200_gemv_q8: bad type/shape");
    if (M == 0) return B200_OK;
    GemvArgs a{};
    a.w = (const uint8_t *)w; a.row_stride = row_stride; a.expert_stride = 0; a.M = (int)M; a.K = (int)K;
    a.ncols = (int)n; a.nz = 1; a.act = act_carve(type, ws, n, K);
    a.dst = dst; a.ldd = ldd; a.residual = nullptr; a.ids = nullptr;
    return from_cuda(launch_gemv(type, a, (cudaStream_t)stream), "b200_gemv_q8");
}

int b200_fused_matvec(int type, int nmat, const void * const * w, const int64_t * row_stride, const int64_t * M, int64_t K, const float * x,
                      const float * norm_w, float eps, int mode, const float * const * residual, float * const * dst, void * stream) {
    if (!(type == T_Q4_K || type == T_Q5_K || type == T_Q6_K) || nmat < 1 || nmat > 3 || K <= 0 || K % 256 || K > 8192 || !x)
        return fail(B200_E_INVALID, "b200_fused_matvec: bad type/shape");
    FusedGemvArgs a{};
    a.nmat = nmat; a.K = (int)K; a.x = x; a.norm_w = norm_w; a.eps = eps; a.has_norm = norm_w ? 1 : 0; a.mode = mode; a.pdl = 0; a.counter = nullptr;
    for (int i = 0; i < nmat; i++) {
        a.w[i] = (const uint8_t *)w[i]; a.row_stride[i] = row_stride[i]; a.M[i] = (int)M[i]; a.dst[i] = dst[i];
        a.residual[i] = residual ? residual[i] : nullptr;
    }
    return from_cuda(launch_fused_gemv(type, a, (cudaStream_t)stream), "b200_fused_matvec");
}

int b200_matvec_program(int n, const int * type, const int * nmat, const void * const * w, const int64_t * row_stride, const int64_t * M,
                        const int64_t * K, const float * const * x, const float * const * norm_w, const float * eps, const int * mode,
                        const float * const * residual, float * const * dst, void * stream) {
    if (n <= 0 || n > 1024) return fail(B200_E_INVALID, "b200_matvec_program: bad phase count");
    // per-device program buffer, tagged-slot pool and zeroed sync words; the previous program may still be running on another
    // stream: callers serialise on the device
    static FlowPhase * d_ph[64] = {};
    static unsigned * d_sync[64] = {};
    static uint64_t * d_ll[64] = {};
    constexpr size_t LL_ELEMS = 512 * 1024;
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!d_ph[dev]) {
        if (cudaMalloc(&d_ph[dev], 1024 * sizeof(FlowPhase)) != cudaSuccess || cudaMalloc(&d_sync[dev], flow_sync_bytes()) != cudaSuccess ||
            cudaMalloc(&d_ll[dev], LL_ELEMS * sizeof(uint64_t)) != cudaSuccess) return from_cuda(cudaGetLastError(), "b200_matvec_program(alloc)");
        cudaMemset(d_sync[dev], 0, flow_sync_bytes());
        cudaMemset(d_ll[dev], 0, LL_ELEMS * sizeof(uint64_t));
        cudaDeviceSynchronize();                               // the caller's stream may be non-blocking: order the zeroing before its first launch
    }
    // the same builder the ggml backend uses: a phase whose input is an earlier phase's output reads it through tagged slots
    FlowBuilder fb;
    fb.reset(d_ll[dev], LL_ELEMS, flow_grid(dev));
    for (int i = 0; i < n; i++) {
        FlowBuilder::MatvecDesc d;
        d.nmat = nmat[i]; d.K = (int)K[i]; d.mode = mode[i]; d.x = x[i]; d.norm_w = norm_w[i]; d.eps = eps[i]; d.residual = residual[i];
        for (int j = 0; j < 3 && j < nmat[i]; j++) {
            d.w[j] = (const uint8_t *)w[3 * i + j]; d.row_stride[j] = row_stride[3 * i + j]; d.M[j] = (int)M[3 * i + j]; d.dst[j] = dst[3 * i + j]; d.type[j] = type[3 * i + j];
        }
        if (!fb.add_matvec(d)) return fail(B200_E_INVALID, "b200_matvec_program: phase not supported");
    }
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemcpyAsync(d_ph[dev], fb.phases().data(), (size_t)n * sizeof(FlowPhase), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return from_cuda(e, "b200_matvec_program(upload)");
    FlowProgram prog{d_ph[dev], n, d_sync[dev], 0, nullptr};
    return from_cuda(launch_decode_flow(prog, st), "b200_matvec_program");
}

size_t b200_flow_slot_bytes(void) { return flow_slot_bytes(); }

int b200_flow_plan(int nmat, const int * type, const int64_t * M, int64_t K, const int64_t * row_stride, int mode, int has_norm, int grid, int * plan) {
    // host-only: how the persistent kernel would cut this mat-vec phase into ring pieces (no device memory is touched)
    if (nmat < 1 || nmat > 3 || plan == nullptr) return fail(B200_E_INVALID, "b200_flow_plan: bad arguments");
    FlowBuilder fb;
    fb.reset(nullptr, 0, grid);
    FlowBuilder::MatvecDesc d;
    d.nmat = nmat; d.K = (int)K; d.mode = mode;
    static float dummy[4];
    const uintptr_t fake = 0x10000;                            // aligned, never dereferenced on the host
    for (int j = 0; j < nmat; j++) { d.w[j] = (const uint8_t *)(fake * (j + 1)); d.row_stride[j] = row_stride[j]; d.M[j] = (int)M[j]; d.type[j] = type[j]; d.dst[j] = (float *)(fake * (8 + j)); }
    d.x = (const float *)(fake * 16); d.norm_w = has_norm ? (const float *)(fake * 17) : nullptr; d.residual = mode == 1 ? (const float *)(fake * 18) : nullptr;
    (void)dummy;
    if (!fb.add_matvec(d)) return fail(B200_E_UNSUPPORTED, "b200_flow_plan: phase not representable");
    const FlowMatvec & m = fb.phases().back().mv;
    plan[0] = m.S; plan[1] = m.seg; plan[2] = m.RP; plan[3] = m.R[0]; plan[4] = m.R[1]; plan[5] = m.R[2]; plan[6] = m.keep_h; plan[7] = (int)b200_flow_slot_bytes();
    return B200_OK;
}

int b200_flow_selftest_postponed_rope(void) {
    // host-only regression check of the program recorder (no device memory is touched): the meta backend's node order records the q mat-vec,
    // postpones ROPE(q), records the v | k mat-vecs -- whose outputs may land in the q mat-mul's recycled buffer -- and only then the attention
    // phase.  The recorder names vectors by address, so the attention phase must be given the q vector remembered at the postponement
    // (rounds 2's leases W / Y / Z: without it the phase read v's slots as q).  Returns 0 when the phase names the right slots.
    static uint64_t pool[1 << 16];
    const uintptr_t fake = 0x100000;
    FlowBuilder fb;
    fb.reset(pool, sizeof(pool) / sizeof(pool[0]), 132);
    float * A = (float *)(fake * 1), * C = (float *)(fake * 2), * X = (float *)(fake * 3), * OUT = (float *)(fake * 4);
    FlowBuilder::MatvecDesc q;
    q.nmat = 1; q.K = 4096; q.mode = 0; q.w[0] = (const uint8_t *)(fake * 8); q.row_stride[0] = 16 * 144; q.M[0] = 4096; q.type[0] = T_Q4_K; q.dst[0] = A;
    q.x = X; q.norm_w = (const float *)(fake * 9); q.eps = 1e-5f;
    if (!fb.add_matvec(q)) return 1;
    const FlowVec qv = fb.vec(A);                               // what the backend remembers when it postpones ROPE(q)
    if (qv.ll == nullptr) return 2;
    FlowBuilder::MatvecDesc vk = q;
    vk.nmat = 2; vk.w[1] = (const uint8_t *)(fake * 10); vk.row_stride[1] = 16 * 144; vk.M[0] = 1024; vk.M[1] = 1024; vk.type[1] = T_Q4_K;
    vk.dst[0] = A;                                              // v lands in the q mat-mul's recycled buffer
    vk.dst[1] = C;
    if (!fb.add_matvec(vk)) return 3;
    if (fb.vec(A).ll == qv.ll) return 4;                        // (the by-address lookup now names v: the hazard this test documents)
    FlowAttn a;
    memset(&a, 0, sizeof(a));
    a.n_head = 32; a.n_head_kv = 8; a.head_dim = 128; a.n_dims = 128; a.rope_mode = 0; a.n_kv = 256;
    a.kview = (const void *)(fake * 11); a.vview = (const void *)(fake * 12); a.k_nb1 = 2048; a.k_nb2 = 256; a.v_nb1 = 2048; a.v_nb2 = 256;
    if (!fb.add_attn(a, A, C, A, OUT, &qv)) return 5;
    const FlowAttn & at = fb.phases().back().at;
    if (at.q.ll != qv.ll || at.q.tag != qv.tag) return 6;       // q: the slots of the FIRST phase
    if (at.v.ll == qv.ll || at.v.ll != fb.phases()[1].mv.out[0].ll) return 7;   // v: the slots of the second phase's first matrix
    if (at.k.ll != fb.phases()[1].mv.out[1].ll) return 8;
    return 0;
}

size_t b200_mul_mat_id_workspace_bytes(int type, int64_t M, int64_t K, int64_t n_used, int64_t T, int64_t nb1) {
    (void)M; (void)n_used;
    return type_ok(type) ? act_workspace_bytes(type, nb1 * T, K) + 256 : 0;
}

int b200_mul_mat_id(int type, const void * w, int64_t row_stride, int64_t expert_stride, int64_t n_expert, int64_t M, int64_t K,
                    const float * b, int64_t nb1, const int32_t * ids, int64_t ids_stride, int64_t n_used, int64_t T,
                    float * dst, void * ws, size_t ws_bytes, void * stream) {
    if (!type_ok(type) || M < 0 || T < 0 || n_used <= 0 || n_expert <= 0 || K <= 0 || K % block_elems(type) || (nb1 != 1 && nb1 != n_used))
        return fail(B200_E_INVALID, "b200_mul_mat_id: bad type/shape");
    if (M == 0 || T == 0) return B200_OK;
    if (ws_bytes < b200_mul_mat_id_workspace_bytes(type, M, K, n_used, T, nb1)) return fail(B200_E_WORKSPACE, "b200_mul_mat_id: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const ActQ8 act = act_carve(type, ws, nb1 * T, K);
    cudaError_t e = launch_quantize_act(type, b, K, nb1 * T, K, act, st);
    if (e != cudaSuccess) return from_cuda(e, "b200_mul_mat_id(quantize)");
    // gridDim.y <= 65535: chunk the (slot, token) pairs by whole tokens
    const int64_t t_chunk = 65535 / n_used;
    for (int64_t t0 = 0; t0 < T; t0 += t_chunk) {
        const int64_t nt = T - t0 < t_chunk ? T - t0 : t_chunk;
        GemvArgs a{};
        a.w = (const uint8_t *)w; a.row_stride = row_stride; a.expert_stride = expert_stride; a.M = (int)M; a.K = (int)K;
        a.ncols = 1; a.nz = (int)(nt * n_used);
        a.act = act; a.act.qs += t0 * nb1 * act.qs_stride; a.act.d += t0 * nb1 * act.d_stride; a.act.bsums += t0 * nb1 * act.bs_stride;
        a.dst = dst + t0 * n_used * M; a.ldd = M; a.residual = nullptr;
        a.ids = ids + t0 * ids_stride; a.ids_stride = ids_stride; a.n_used = (int)n_used; a.nb1 = (int)nb1; a.n_expert = (int)n_expert;
        e = launch_gemv(type, a, st);
        if (e != cudaSuccess) return from_cuda(e, "b200_mul_mat_id(gemv)");
    }
    return B200_OK;
}

size_t b200_mul_mat_host_scratch_bytes(int type, int64_t M, int64_t N, int64_t K) {
    if (!type_ok(type)) return 0;
    return (size_t)(N * K * 4 + 256) + (size_t)(M * N * 4 + 256) + b200_mul_mat_workspace_bytes(type, M, N, K) + 256;
}

int b200_mul_mat_host(int type, const void * w, int64_t row_stride, int64_t M, int64_t K, const float * x_host, int64_t N,
                      float * dst_host, void * scratch, size_t scratch_bytes, void * stream) {
    if (scratch_bytes < b200_mul_mat_host_scratch_bytes(type, M, N, K)) return fail(B200_E_WORKSPACE, "b200_mul_mat_host: scratch too small");
    cudaStream_t st = (cudaStream_t)stream;
    uint8_t * p = (uint8_t *)(((uintptr_t)scratch + 255) & ~(uintptr_t)255);
    float * x_dev = (float *)p;   p += ((size_t)(N * K * 4) + 255) & ~(size_t)255;
    float * d_dev = (float *)p;   p += ((size_t)(M * N * 4) + 255) & ~(size_t)255;
    const size_t ws_bytes = scratch_bytes - (size_t)(p - (uint8_t *)scratch);
    cudaError_t e = cudaMemcpyAsync(x_dev, x_host, (size_t)(N * K * 4), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return from_cuda(e, "b200_mul_mat_host(h2d)");
    int rc = b200_mul_mat(type, w, row_stride, M, K, x_dev, K, N, d_dev, M, p, ws_bytes, stream);
    if (rc) return rc;
    e = cudaMemcpyAsync(dst_host, d_dev, (size_t)(M * N * 4), cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) return from_cuda(e, "b200_mul_mat_host(d2h)");
    return from_cuda(cudaStreamSynchronize(st), "b200_mul_mat_host(sync)");
}

}  // extern "C"
