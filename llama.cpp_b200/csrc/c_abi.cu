// c_abi.cu -- the extern "C" surface declared in include/b200_qmm.h, include/b200_attn.h, include/b200_moe.h and include/b200_flow.h.  Thin: argument checks, workspace carving,
// regime selection (decode GEMV vs prefill GEMM), error text.  No compute happens on the host and there is no CPU
// fallback: if CUDA is unusable every compute entry point fails loudly.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "../../include/b200_qmm.h"
#include "../../include/b200_attn.h"
#include "../../include/b200_moe.h"
#include "../../include/b200_flow.h"
#include "qmm_formats.cuh"
#include <vector>
#include <string.h>
#include "qmm_kernels.cuh"
#include "qmm_ops.cuh"
#include "qmm_attn.cuh"
#include "qmm_moe.cuh"
#include "decode_flow.cuh"

namespace qmm {
static std::atomic<uint64_t> g_launches{0};
void note_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
// decode_flow.cu: the Q8_K hand-over as the recorded phases carry it (b200_flow_q8k_plan, b200_flow_q8k_reuse)
int    flow_q8k_block_of(const FlowMatvec & p, int cta);          // the block CTA `cta` quantises, -1: none (or the phase emits no Q8_K blocks)
size_t flow_q8k_words(const FlowMatvec & p);                      // tagged words of the phase's Q8_K blocks (out[1].ll), 0: none
bool   flow_reads_q8k(const FlowMatvec & p);                      // the phase's input is a Q8_K vector
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

// Per-device program buffer, tagged-slot pool and zeroed sync words of the programs launched through this C ABI
// (b200_matvec_program, b200_attn_program).  The previous program may still be running on another stream: callers serialise
// on the device.
struct FlowBuffers { FlowPhase * ph; unsigned * sync; uint64_t * ll; int dev; };
constexpr int FLOW_ABI_PHASES = 1024;
constexpr size_t FLOW_ABI_LL_ELEMS = 512 * 1024;

static cudaError_t flow_buffers(FlowBuffers & fbuf) {
    static FlowPhase * d_ph[64] = {};
    static unsigned * d_sync[64] = {};
    static uint64_t * d_ll[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!d_ph[dev]) {
        if (cudaMalloc(&d_ph[dev], FLOW_ABI_PHASES * sizeof(FlowPhase)) != cudaSuccess || cudaMalloc(&d_sync[dev], flow_sync_bytes()) != cudaSuccess ||
            cudaMalloc(&d_ll[dev], FLOW_ABI_LL_ELEMS * sizeof(uint64_t)) != cudaSuccess) return cudaGetLastError();
        cudaMemset(d_sync[dev], 0, flow_sync_bytes());
        cudaMemset(d_ll[dev], 0, FLOW_ABI_LL_ELEMS * sizeof(uint64_t));
        cudaDeviceSynchronize();                               // the caller's stream may be non-blocking: order the zeroing before its first launch
    }
    fbuf.ph = d_ph[dev]; fbuf.sync = d_sync[dev]; fbuf.ll = d_ll[dev]; fbuf.dev = dev;
    return cudaSuccess;
}

static cudaError_t flow_launch(const FlowBuffers & fbuf, const FlowBuilder & fb, cudaStream_t st) {
    const int n = (int)fb.size();
    cudaError_t e = cudaMemcpyAsync(fbuf.ph, fb.phases().data(), (size_t)n * sizeof(FlowPhase), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    FlowProgram prog{fbuf.ph, n, fbuf.sync, 0, nullptr};
    return launch_decode_flow(prog, st);
}

int b200_matvec_program(int n, const int * type, const int * nmat, const void * const * w, const int64_t * row_stride, const int64_t * M,
                        const int64_t * K, const float * const * x, const float * const * norm_w, const float * eps, const int * mode,
                        const float * const * residual, float * const * dst, void * stream) {
    if (n <= 0 || n > FLOW_ABI_PHASES) return fail(B200_E_INVALID, "b200_matvec_program: bad phase count");
    FlowBuffers fbuf;
    cudaError_t e = flow_buffers(fbuf);
    if (e != cudaSuccess) return from_cuda(e, "b200_matvec_program(alloc)");
    // the same builder the ggml backend uses: a phase whose input is an earlier phase's output reads it through tagged slots
    FlowBuilder fb;
    fb.reset(fbuf.ll, FLOW_ABI_LL_ELEMS, flow_grid(fbuf.dev));
    for (int i = 0; i < n; i++) {
        FlowBuilder::MatvecDesc d;
        d.nmat = nmat[i]; d.K = (int)K[i]; d.mode = mode[i]; d.x = x[i]; d.norm_w = norm_w[i]; d.eps = eps[i]; d.residual = residual[i];
        for (int j = 0; j < 3 && j < nmat[i]; j++) {
            d.w[j] = (const uint8_t *)w[3 * i + j]; d.row_stride[j] = row_stride[3 * i + j]; d.M[j] = (int)M[3 * i + j]; d.dst[j] = dst[3 * i + j]; d.type[j] = type[3 * i + j];
        }
        if (!fb.add_matvec(d)) return fail(B200_E_INVALID, "b200_matvec_program: phase not supported");
    }
    return from_cuda(flow_launch(fbuf, fb, (cudaStream_t)stream), "b200_matvec_program");
}

int b200_attn_program(const b200_attn_args * a, int * nsplit, void * stream) {
    if (a == nullptr) return fail(B200_E_INVALID, "b200_attn_program: no arguments");
    if (a->head_dim != 128) return fail(B200_E_UNSUPPORTED, "b200_attn_program: head_dim must be 128");
    if (a->n_head <= 0 || a->n_head_kv <= 0 || a->n_head % a->n_head_kv) return fail(B200_E_INVALID, "b200_attn_program: n_head must be a multiple of n_head_kv");
    if (a->n_kv <= 0 || a->n_dims <= 0 || a->n_dims > a->head_dim || a->n_dims % 2 || (a->rope_mode != 0 && a->rope_mode != 2))
        return fail(B200_E_INVALID, "b200_attn_program: bad n_kv / n_dims / rope mode");
    if (!a->q || !a->k || !a->v || !a->dst || !a->pos || !a->kpos || !a->vpos || !a->k_cache || !a->v_cache || !a->kview || !a->vview)
        return fail(B200_E_INVALID, "b200_attn_program: missing pointer");
    const bool fused = a->w_qkv[0] != nullptr;
    if (fused && (!a->w_qkv[1] || !a->w_qkv[2] || !a->x || a->n_embd <= 0 || a->n_embd > INT32_MAX))
        return fail(B200_E_INVALID, "b200_attn_program: incomplete q|k|v mat-vec");
    FlowBuffers fbuf;
    cudaError_t e = flow_buffers(fbuf);
    if (e != cudaSuccess) return from_cuda(e, "b200_attn_program(alloc)");
    FlowBuilder fb;
    fb.reset(fbuf.ll, FLOW_ABI_LL_ELEMS, flow_grid(fbuf.dev));
    if (fused) {
        FlowBuilder::MatvecDesc d;
        d.nmat = 3; d.K = (int)a->n_embd; d.mode = 0; d.x = a->x; d.norm_w = a->norm_w; d.eps = a->eps;
        float * outs[3] = {a->q, a->k, a->v};
        const int64_t rows[3] = {(int64_t)a->head_dim * a->n_head, (int64_t)a->head_dim * a->n_head_kv, (int64_t)a->head_dim * a->n_head_kv};
        for (int j = 0; j < 3; j++) {
            d.w[j] = (const uint8_t *)a->w_qkv[j]; d.row_stride[j] = a->row_stride_qkv[j]; d.M[j] = (int)rows[j]; d.type[j] = a->type_qkv[j]; d.dst[j] = outs[j];
        }
        if (!fb.add_matvec(d)) return fail(B200_E_UNSUPPORTED, "b200_attn_program: q|k|v mat-vec not representable");
    }
    // FlowAttn as the backend fills it for a ROPE pair + SET_ROWS pair + FLASH_ATTN_EXT (backend/ggml_b200.cpp, fuse_rope_pair)
    ops::RopeKVArgs r{};
    r.n_dims = a->n_dims; r.n_ctx_orig = a->n_ctx_orig; r.freq_base = a->freq_base; r.beta_fast = a->beta_fast; r.beta_slow = a->beta_slow;
    FlowAttn m;
    memset(&m, 0, sizeof(m));
    m.k_cache = a->k_cache; m.k_row_bytes = a->k_row_bytes; m.v_cache = a->v_cache; m.v_row_bytes = a->v_row_bytes;
    m.k_idx = a->kpos; m.v_idx = a->vpos; m.pos = a->pos; m.freq_factors = a->freq_factors;
    m.kview = a->kview; m.k_nb1 = a->k_nb1; m.k_nb2 = a->k_nb2;
    m.vview = a->vview; m.v_nb1 = a->v_nb1; m.v_nb2 = a->v_nb2;
    m.mask = a->mask;
    m.n_head = a->n_head; m.n_head_kv = a->n_head_kv; m.head_dim = a->head_dim; m.n_dims = a->n_dims; m.rope_mode = a->rope_mode; m.n_kv = a->n_kv;
    m.freq_scale = a->freq_scale; m.ext_factor = a->ext_factor; m.attn_factor = a->attn_factor;
    ops::rope_derived(r, m.theta_scale, m.corr0, m.corr1);
    m.softcap = a->softcap; m.scale = a->softcap != 0.0f ? a->scale / a->softcap : a->scale;
    if (!fb.add_attn(m, a->q, a->k, a->v, a->dst)) return fail(B200_E_UNSUPPORTED, "b200_attn_program: attention phase not representable");
    if (nsplit) *nsplit = fb.phases().back().at.nsplit;
    return from_cuda(flow_launch(fbuf, fb, (cudaStream_t)stream), "b200_attn_program");
}

static ops::TensorView tview(const void * p, const int64_t * ne, const int64_t * nb, int type) {
    ops::TensorView t;
    t.data = const_cast<void *>(p);
    for (int i = 0; i < 4; i++) { t.ne[i] = ne[i]; t.nb[i] = nb ? nb[i] : 0; }
    t.type = type;
    return t;
}

size_t b200_flash_attn_workspace_bytes(const int64_t * q_ne, const int64_t * k_ne, const int64_t * mask_ne) {
    if (!q_ne || !k_ne) return 0;
    const ops::TensorView q = tview(nullptr, q_ne, nullptr, 0), k = tview(nullptr, k_ne, nullptr, 1);
    if (!mask_ne) return ops::flash_attn_workspace_bytes(q, k, nullptr);
    const ops::TensorView m = tview(nullptr, mask_ne, nullptr, 1);
    return ops::flash_attn_workspace_bytes(q, k, &m);
}

int b200_flash_attn(const float * q, const int64_t * q_ne, const int64_t * q_nb, const void * k, const int64_t * k_ne, const int64_t * k_nb,
                    const void * v, const int64_t * v_ne, const int64_t * v_nb, const void * mask, const int64_t * mask_ne, const int64_t * mask_nb,
                    float * dst, const int64_t * dst_ne, const int64_t * dst_nb, float scale, float softcap, void * ws, size_t ws_bytes, int path, void * stream) {
    if (!q_ne || !q_nb || !k_ne || !k_nb || !v_ne || !v_nb || !dst_ne || !dst_nb || (mask && (!mask_ne || !mask_nb)) || path < 0 || path > 2)
        return fail(B200_E_INVALID, "b200_flash_attn: bad arguments");
    for (int i = 0; i < 4; i++)
        if (q_ne[i] <= 0 || k_ne[i] <= 0 || v_ne[i] <= 0 || (mask && mask_ne[i] <= 0)) return fail(B200_E_INVALID, "b200_flash_attn: empty dimension");
    const int64_t DK = q_ne[0], N = q_ne[1], H = q_ne[2], B = q_ne[3], n_kv = k_ne[1], DV = v_ne[0];
    if (k_ne[0] != DK || v_ne[1] != n_kv || H % k_ne[2] || H % v_ne[2] || B % k_ne[3] || B % v_ne[3])
        return fail(B200_E_INVALID, "b200_flash_attn: q / k / v shapes do not broadcast");
    if (dst_ne[0] != DV || dst_ne[1] != H || dst_ne[2] != N || dst_ne[3] != B) return fail(B200_E_INVALID, "b200_flash_attn: dst must be [DV, H, N, B]");
    if (q_nb[0] != 4 || k_nb[0] != 2 || v_nb[0] != 2 || dst_nb[0] != 4 || (mask && mask_nb[0] != 2)) return fail(B200_E_INVALID, "b200_flash_attn: rows must be contiguous");
    if (mask && (mask_ne[0] < n_kv || mask_ne[1] < N || H % mask_ne[2] || B % mask_ne[3])) return fail(B200_E_INVALID, "b200_flash_attn: mask shape");
    if (path == 1 && (DK != DV || DK % 32 || DK > 256)) return fail(B200_E_UNSUPPORTED, "b200_flash_attn: the scalar kernel needs D = DV, a multiple of 32 up to 256");
    if (path == 2 && (DK != DV || (DK != 64 && DK != 128) || N < ops::FA_MIN_ROWS_MMA))
        return fail(B200_E_UNSUPPORTED, "b200_flash_attn: the tensor-core kernel needs D = DV in {64, 128} and >= 16 rows");
    const ops::TensorView tq = tview(q, q_ne, q_nb, 0), tk = tview(k, k_ne, k_nb, 1), tv = tview(v, v_ne, v_nb, 1), td = tview(dst, dst_ne, dst_nb, 0);
    const ops::TensorView tm = mask ? tview(mask, mask_ne, mask_nb, 1) : tq;
    const ops::TensorView * pm = mask ? &tm : nullptr;
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e;
    if (path == 0) e = ops::flash_attn(tq, tk, tv, pm, td, scale, softcap, st, ws, ws_bytes);
    else if (path == 1) e = ops::flash_attn_scalar(tq, tk, tv, pm, td, scale, softcap, st);
    else e = ops::flash_attn_prefill(tq, tk, tv, pm, td, scale, softcap, ws, ws_bytes, st);
    return from_cuda(e, "b200_flash_attn");
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

int b200_flow_q8k_plan(int producer_mode, int64_t M, int64_t K_in, int consumer_norm, int grid, int * block_of_cta) {
    if ((producer_mode != 0 && producer_mode != 2) || M <= 0 || M > FLOW_MAX_K || K_in <= 0 || K_in > FLOW_MAX_K || grid <= 0 || grid > 4096 || !block_of_cta)
        return fail(B200_E_INVALID, "b200_flow_q8k_plan: bad arguments");
    const uintptr_t fake = 0x100000;                           // aligned, never dereferenced on the host
    FlowBuilder fb;
    fb.reset(reinterpret_cast<uint64_t *>(fake * 64), 1 << 20, grid);
    FlowBuilder::MatvecDesc up;
    up.nmat = producer_mode == 2 ? 2 : 1; up.K = (int)K_in; up.mode = producer_mode; up.x = (const float *)(fake * 1);
    up.norm_w = (const float *)(fake * 2); up.eps = 1e-5f; up.dst[0] = (float *)(fake * 3);
    for (int j = 0; j < up.nmat; j++) { up.w[j] = (const uint8_t *)(fake * (8 + j)); up.row_stride[j] = K_in / 256 * 144; up.M[j] = (int)M; up.type[j] = T_Q4_K; }
    FlowBuilder::MatvecDesc down;
    down.nmat = 1; down.K = (int)M; down.mode = 0; down.x = up.dst[0]; down.norm_w = consumer_norm ? (const float *)(fake * 4) : nullptr; down.eps = 1e-5f;
    down.w[0] = (const uint8_t *)(fake * 10); down.row_stride[0] = M / 256 * 144; down.M[0] = 4096; down.type[0] = T_Q4_K; down.dst[0] = (float *)(fake * 5);
    if (!fb.add_matvec(up) || !fb.add_matvec(down)) return fail(B200_E_UNSUPPORTED, "b200_flow_q8k_plan: phase not representable");
    const bool q8k = flow_reads_q8k(fb.phases()[1].mv);
    for (int c = 0; c < grid; c++) block_of_cta[c] = flow_q8k_block_of(fb.phases()[0].mv, c);
    return q8k ? 1 : 0;
}

int b200_flow_q8k_reuse(int n_layers, int64_t n_ff, int64_t pool_elems, int grid, int * n_q8k, int * min_phases) {
    if (n_layers <= 0 || n_layers > 256 || n_ff <= 0 || n_ff > FLOW_MAX_K || pool_elems <= 0 || grid < 32 || grid > 4096 || !n_q8k || !min_phases)
        return fail(B200_E_INVALID, "b200_flow_q8k_reuse: bad arguments");
    const uintptr_t fake = 0x100000;                           // aligned, never dereferenced on the host
    uint64_t * const pool = reinterpret_cast<uint64_t *>(fake * 4096);
    FlowBuilder fb;
    fb.reset(pool, (size_t)pool_elems, grid);
    const int E = 4096, D = 128, H = 32, HKV = 8;
    auto vecp = [&](int l, int j) { return (float *)(fake * (16 + 16 * (size_t)l + j)); };
    auto mv = [&](int nmat, int K, int mode, const float * x, const float * norm_w, const float * resid, const int * M, float * d0, float * d1, float * d2) {
        FlowBuilder::MatvecDesc d;
        d.nmat = nmat; d.K = K; d.mode = mode; d.x = x; d.norm_w = norm_w; d.residual = resid; d.eps = 1e-5f;
        float * dst[3] = {d0, d1, d2};
        for (int j = 0; j < nmat; j++) { d.w[j] = (const uint8_t *)(fake * 8); d.row_stride[j] = K / 256 * 144; d.M[j] = M[j]; d.type[j] = T_Q4_K; d.dst[j] = dst[j]; }
        return fb.add_matvec(d);
    };
    const float * h = (const float *)(fake * 1), * nw = (const float *)(fake * 2);
    for (int l = 0; l < n_layers; l++) {
        const int mqkv[3] = {H * D, HKV * D, HKV * D}, me[1] = {E}, mff[2] = {(int)n_ff, (int)n_ff};
        FlowAttn a;
        memset(&a, 0, sizeof(a));
        a.n_head = H; a.n_head_kv = HKV; a.head_dim = D; a.n_dims = D; a.rope_mode = 0; a.n_kv = 256;
        a.kview = (const void *)(fake * 11); a.vview = (const void *)(fake * 12); a.k_nb1 = 2048; a.k_nb2 = 256; a.v_nb1 = 2048; a.v_nb2 = 256;
        if (!mv(3, E, 0, h, nw, nullptr, mqkv, vecp(l, 0), vecp(l, 1), vecp(l, 2)) || !fb.add_attn(a, vecp(l, 0), vecp(l, 1), vecp(l, 2), vecp(l, 3)) ||
            !mv(1, E, 1, vecp(l, 3), nullptr, h, me, vecp(l, 4), nullptr, nullptr) || !mv(2, E, 2, vecp(l, 4), nw, nullptr, mff, vecp(l, 5), nullptr, nullptr) ||
            !mv(1, (int)n_ff, 1, vecp(l, 5), nullptr, vecp(l, 4), me, vecp(l, 6), nullptr, nullptr))
            return fail(B200_E_UNSUPPORTED, "b200_flow_q8k_reuse: phase not representable");
        h = vecp(l, 6);
    }
    // the slot ranges every phase writes, then the fewest phases between two writes of one slot
    struct Range { size_t lo, hi; int phase; };
    std::vector<Range> rs;
    const auto & ph = fb.phases();
    int nq = 0;
    auto add = [&](const uint64_t * ll, size_t n, int i) { if (ll && n) rs.push_back(Range{(size_t)(ll - pool), (size_t)(ll - pool) + n, i}); };
    for (int i = 0; i < (int)ph.size(); i++) {
        if (ph[i].kind == FLOW_MATVEC) {
            const FlowMatvec & m = ph[i].mv;
            for (int j = 0; j < (m.mode == 2 ? 1 : m.nmat); j++) add(m.out[j].ll, (size_t)m.M[j], i);
            add(m.out[1].ll, flow_q8k_words(m), i);
            nq += flow_reads_q8k(m) ? 1 : 0;
        } else if (ph[i].kind == FLOW_ATTN) {
            const FlowAttn & at = ph[i].at;
            add(at.out.ll, (size_t)at.n_head * at.head_dim, i);
            add(at.part_ll, (size_t)at.n_head * at.nsplit * (at.head_dim + 2), i);
        }
    }
    int dist = (int)ph.size();
    for (size_t x = 0; x < rs.size(); x++)
        for (size_t y = x + 1; y < rs.size(); y++)
            if (rs[x].lo < rs[y].hi && rs[y].lo < rs[x].hi && rs[x].phase != rs[y].phase) dist = std::min(dist, std::abs(rs[y].phase - rs[x].phase));
    *n_q8k = nq;
    *min_phases = dist;
    return B200_OK;
}

size_t b200_mul_mat_id_workspace_bytes(int type, int64_t M, int64_t K, int64_t n_used, int64_t T, int64_t nb1) {
    (void)M; (void)n_used;
    return type_ok(type) ? act_workspace_bytes(type, nb1 * T, K) + 256 : 0;
}

// The routed GEMV over all (token, slot) rows, in token chunks: gridDim.y = chunk * n_used <= 65535.  As b200_mul_mat_id below and
// the backend's run_mul_mat_id do it.
static cudaError_t mul_mat_id_gemv(int type, const void * w, int64_t row_stride, int64_t expert_stride, int64_t n_expert, int64_t M, int64_t K,
                                   const float * b, int64_t nb1, const int32_t * ids, int64_t ids_stride, int64_t n_used, int64_t T,
                                   float * dst, void * ws, cudaStream_t st) {
    const ActQ8 act = act_carve(type, ws, nb1 * T, K);
    cudaError_t e = launch_quantize_act(type, b, K, nb1 * T, K, act, st);
    if (e != cudaSuccess) return e;
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
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

size_t b200_mul_mat_id_path_workspace_bytes(int type, int64_t M, int64_t K, int64_t n_expert, int64_t n_used, int64_t T, int64_t nb1) {
    if (!type_ok(type)) return 0;
    const size_t a = act_workspace_bytes(type, nb1 * T, K);
    const size_t g = gemm_grouped_workspace_bytes(type, M, n_used * T, n_expert, K);
    return (a > g ? a : g) + 256;
}

int b200_mul_mat_id_path(int type, const void * w, int64_t row_stride, int64_t expert_stride, int64_t n_expert, int64_t M, int64_t K,
                         const float * b, int64_t nb1, const int32_t * ids, int64_t ids_stride, int64_t n_used, int64_t T,
                         float * dst, void * ws, size_t ws_bytes, int path, int * taken, void * stream) {
    if (taken) *taken = 0;
    if (path < 0 || path > 2) return fail(B200_E_INVALID, "b200_mul_mat_id_path: path must be 0, 1 or 2");
    if (!type_ok(type) || M < 0 || T < 0 || n_used <= 0 || n_expert <= 0 || K <= 0 || K % block_elems(type) || (nb1 != 1 && nb1 != n_used))
        return fail(B200_E_INVALID, "b200_mul_mat_id_path: bad type/shape (n_used > 0, nb1 in {1, n_used})");
    if (M > INT32_MAX || K > INT32_MAX || T * n_used > INT32_MAX || n_expert > INT32_MAX) return fail(B200_E_INVALID, "b200_mul_mat_id_path: dimension too large");
    if (M == 0 || T == 0) return B200_OK;
    if (ws_bytes < b200_mul_mat_id_path_workspace_bytes(type, M, K, n_expert, n_used, T, nb1))
        return fail(B200_E_WORKSPACE, "b200_mul_mat_id_path: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    // path 0 restates the rule of run_mul_mat_id (backend/ggml_b200.cpp), which the plugin's prebuilt objects compile in: keep the two
    // in step.  Many (token, slot) rows and a grouped workspace (K-quant, n_expert <= 256) take the grouped GEMM; operands it cannot
    // take fall back to the GEMV.
    const int64_t jobs = T * n_used;
    if (path == 2 || (path == 0 && jobs >= 32 && gemm_grouped_workspace_bytes(type, M, jobs, n_expert, K) != 0)) {
        GemmGroupedArgs ga{};
        ga.w = (const uint8_t *)w; ga.row_stride = row_stride; ga.expert_stride = expert_stride; ga.M = (int)M; ga.K = (int)K; ga.n_expert = (int)n_expert;
        ga.x = b; ga.ldx = K; ga.nb1 = (int)nb1;
        ga.ids = ids; ga.ids_stride = ids_stride; ga.T = (int)T; ga.n_used = (int)n_used;
        ga.dst = dst; ga.ldd = M; ga.workspace = ws; ga.workspace_bytes = ws_bytes;
        const cudaError_t ge = launch_gemm_grouped(type, ga, st);
        if (ge == cudaErrorNotSupported || ge == cudaErrorMisalignedAddress) {
            cudaGetLastError();
            if (path == 2) return fail(B200_E_UNSUPPORTED, "b200_mul_mat_id_path: the grouped GEMM takes K-quant experts, n_expert <= 256 and aligned operands");
        } else {
            if (ge == cudaSuccess && taken) *taken = 2;
            return from_cuda(ge, "b200_mul_mat_id_path(grouped gemm)");
        }
    }
    const cudaError_t e = mul_mat_id_gemv(type, w, row_stride, expert_stride, n_expert, M, K, b, nb1, ids, ids_stride, n_used, T, dst, ws, st);
    if (e == cudaSuccess && taken) *taken = 1;
    return from_cuda(e, "b200_mul_mat_id_path(gemv)");
}

int64_t b200_moe_route_max_tiles(int64_t n_expert, int64_t n_used, int64_t T) {
    if (n_expert <= 0 || n_used <= 0 || T < 0) return 0;
    return moe_max_tiles(T * n_used, n_expert);
}

int64_t b200_moe_route(const int32_t * ids, int64_t ids_stride, int64_t n_expert, int64_t n_used, int64_t T, int64_t nb1,
                       int32_t * tile_expert, int32_t * col_src, int32_t * col_dst, void * stream) {
    if (n_used <= 0 || T <= 0 || n_expert <= 0 || (nb1 != 1 && nb1 != n_used) || !ids || !tile_expert || !col_src || !col_dst)
        return fail(B200_E_INVALID, "b200_moe_route: bad arguments (n_used > 0, T > 0, nb1 in {1, n_used})");
    if (n_expert > 256) return fail(B200_E_UNSUPPORTED, "b200_moe_route: n_expert must be <= 256");
    const int64_t max_tiles = moe_max_tiles(T * n_used, n_expert);
    if (T * n_used > INT32_MAX || max_tiles * MOE_TILE_COLS > INT32_MAX) return fail(B200_E_INVALID, "b200_moe_route: too many jobs");
    note_launch();
    const cudaError_t e = launch_moe_route(ids, ids_stride, (int)T, (int)n_used, (int)nb1, (int)n_expert, (int)max_tiles, tile_expert, col_src, col_dst,
                                           (cudaStream_t)stream);
    if (e != cudaSuccess) return from_cuda(e, "b200_moe_route");
    return max_tiles;
}

int b200_mul_mat_id(int type, const void * w, int64_t row_stride, int64_t expert_stride, int64_t n_expert, int64_t M, int64_t K,
                    const float * b, int64_t nb1, const int32_t * ids, int64_t ids_stride, int64_t n_used, int64_t T,
                    float * dst, void * ws, size_t ws_bytes, void * stream) {
    if (!type_ok(type) || M < 0 || T < 0 || n_used <= 0 || n_expert <= 0 || K <= 0 || K % block_elems(type) || (nb1 != 1 && nb1 != n_used))
        return fail(B200_E_INVALID, "b200_mul_mat_id: bad type/shape");
    if (M == 0 || T == 0) return B200_OK;
    if (ws_bytes < b200_mul_mat_id_workspace_bytes(type, M, K, n_used, T, nb1)) return fail(B200_E_WORKSPACE, "b200_mul_mat_id: workspace too small");
    return from_cuda(mul_mat_id_gemv(type, w, row_stride, expert_stride, n_expert, M, K, b, nb1, ids, ids_stride, n_used, T, dst, ws, (cudaStream_t)stream),
                     "b200_mul_mat_id");
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
