// ops.cu -- supporting (non mat-mul) ops of the Llama / Mixtral graphs.  See qmm_ops.cuh.
// Semantics restated from the CPU backend (ggml/src/ggml-cpu/ops.cpp): RMS_NORM :3731-3790 (double-precision sum of
// float squares, scale = 1/sqrtf(mean+eps)); ROPE :5818-6100 (theta iterated multiplicatively per pair, YaRN ramp);
// SET_ROWS / GET_ROWS (row scatter / gather with index broadcast); GLU SWIGLU (vec.cpp:417, silu(x) = x/(1+expf(-x)));
// FLASH_ATTN_EXT :8475-8700 (online softmax; we accumulate V in fp32 where the CPU uses fp16).
#include <cuda_fp16.h>

#include "qmm_formats.cuh"
#include "qmm_kernels.cuh"
#include "qmm_ops.cuh"
#include "qmm_attn.cuh"

namespace qmm {
namespace ops {

enum { TY_F32 = 0, TY_F16 = 1, TY_I32 = 26, TY_I64 = 27 };

static inline unsigned cdiv(int64_t a, int64_t b) { return (unsigned)((a + b - 1) / b); }

__device__ __forceinline__ float load_as_f32(const void * p, int type) {
    return type == TY_F16 ? __half2float(*reinterpret_cast<const __half *>(p)) : *reinterpret_cast<const float *>(p);
}
__device__ __forceinline__ void store_from_f32(void * p, int type, float v) {
    if (type == TY_F16) *reinterpret_cast<__half *>(p) = __float2half_rn(v);
    else *reinterpret_cast<float *>(p) = v;
}

// ------------------------------------------------------------------------------------------------ RMS_NORM (+MUL)
// One CTA of 1024 threads per row.  The row is read ONCE into registers with float4 loads issued back to back (the first
// version looped load -> use and was latency-bound: 17 us for 4096 floats), reduced in double like the CPU, and written.
constexpr int RMS_THREADS = 1024;
constexpr int RMS_MAX_V4 = 4;                               // float4 per thread -> rows up to 16384 floats stay in registers
__global__ void __launch_bounds__(RMS_THREADS) rms_norm_kernel(const TensorView x, const TensorView w, bool has_w, const TensorView y, float eps) {
    pdl_prologue();
    const int64_t row = blockIdx.x;
    const int64_t i1 = row % x.ne[1], i2 = (row / x.ne[1]) % x.ne[2], i3 = row / (x.ne[1] * x.ne[2]);
    const float * xr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    float * yr = reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]);
    const float * wr = has_w ? reinterpret_cast<const float *>(reinterpret_cast<const char *>(w.data) + (i1 % w.ne[1]) * w.nb[1] + (i2 % w.ne[2]) * w.nb[2] + (i3 % w.ne[3]) * w.nb[3]) : nullptr;
    const int n = (int)x.ne[0];
    const bool vec = (n % 4 == 0) && n <= RMS_THREADS * 4 * RMS_MAX_V4 && ((reinterpret_cast<uintptr_t>(xr) | reinterpret_cast<uintptr_t>(yr)) & 15) == 0 &&
                     (!wr || (reinterpret_cast<uintptr_t>(wr) & 15) == 0);
    float4 v[RMS_MAX_V4];
    double acc = 0.0;
    if (vec) {
#pragma unroll
        for (int j = 0; j < RMS_MAX_V4; j++) {
            const int i = threadIdx.x + j * RMS_THREADS;
            v[j] = i * 4 < n ? __ldcg(reinterpret_cast<const float4 *>(xr) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < RMS_MAX_V4; j++)
            acc += (double)__fmul_rn(v[j].x, v[j].x) + (double)__fmul_rn(v[j].y, v[j].y) + (double)__fmul_rn(v[j].z, v[j].z) + (double)__fmul_rn(v[j].w, v[j].w);
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) { const float t = __ldcg(xr + i); acc += (double)__fmul_rn(t, t); }
    }
    __shared__ double red[RMS_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    double tot = 0.0;
#pragma unroll
    for (int i = 0; i < RMS_THREADS / 32; i++) tot += red[i];
    const float mean = (float)(tot / (double)n);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, eps)));
    if (vec) {
#pragma unroll
        for (int j = 0; j < RMS_MAX_V4; j++) {
            const int i = threadIdx.x + j * RMS_THREADS;
            if (i * 4 < n) {
                float4 o = make_float4(__fmul_rn(v[j].x, scale), __fmul_rn(v[j].y, scale), __fmul_rn(v[j].z, scale), __fmul_rn(v[j].w, scale));
                if (wr) { const float4 ww = reinterpret_cast<const float4 *>(wr)[i]; o.x = __fmul_rn(o.x, ww.x); o.y = __fmul_rn(o.y, ww.y); o.z = __fmul_rn(o.z, ww.z); o.w = __fmul_rn(o.w, ww.w); }
                reinterpret_cast<float4 *>(yr)[i] = o;
            }
        }
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            float t = __fmul_rn(__ldcg(xr + i), scale);
            if (wr) t = __fmul_rn(t, wr[i]);
            yr[i] = t;
        }
    }
}

cudaError_t rms_norm(const TensorView & x, const TensorView * w, const TensorView & y, float eps, cudaStream_t st) {
    const int64_t rows = x.ne[1] * x.ne[2] * x.ne[3];
    if (rows == 0 || x.ne[0] == 0) return cudaSuccess;
    note_launch();
    return launch_pdl(rms_norm_kernel, dim3((unsigned)rows), dim3(RMS_THREADS), 0, st, x, w ? *w : x, w != nullptr, y, eps);
}

// ------------------------------------------------------------------------------------------------ ADD / MUL with broadcast
__global__ void __launch_bounds__(256) binary_kernel(int op, const TensorView a, const TensorView b, const TensorView y, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t i0 = i % y.ne[0], i1 = (i / y.ne[0]) % y.ne[1], i2 = (i / (y.ne[0] * y.ne[1])) % y.ne[2], i3 = i / (y.ne[0] * y.ne[1] * y.ne[2]);
    const float av = *reinterpret_cast<const float *>(reinterpret_cast<const char *>(a.data) + i0 * a.nb[0] + i1 * a.nb[1] + i2 * a.nb[2] + i3 * a.nb[3]);
    const float bv = *reinterpret_cast<const float *>(reinterpret_cast<const char *>(b.data) + (i0 % b.ne[0]) * b.nb[0] + (i1 % b.ne[1]) * b.nb[1] +
                                                      (i2 % b.ne[2]) * b.nb[2] + (i3 % b.ne[3]) * b.nb[3]);
    *reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i0 * y.nb[0] + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]) =
        op == 0 ? __fadd_rn(av, bv) : (op == 1 ? __fmul_rn(av, bv) : __fdiv_rn(av, bv));
}

// same-shape contiguous operands (the residual adds of a prompt batch): float4 grid-stride, no index arithmetic
__global__ void __launch_bounds__(256) binary_flat4_kernel(int op, const float4 * __restrict__ a, const float4 * __restrict__ b, float4 * __restrict__ y, int64_t n4) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 u = a[i], v = b[i];
        float4 r;
        if (op == 0) { r.x = __fadd_rn(u.x, v.x); r.y = __fadd_rn(u.y, v.y); r.z = __fadd_rn(u.z, v.z); r.w = __fadd_rn(u.w, v.w); }
        else { r.x = __fmul_rn(u.x, v.x); r.y = __fmul_rn(u.y, v.y); r.z = __fmul_rn(u.z, v.z); r.w = __fmul_rn(u.w, v.w); }
        y[i] = r;
    }
}
static bool flat_f32(const TensorView & t) {
    return t.nb[0] == 4 && t.nb[1] == t.ne[0] * 4 && t.nb[2] == t.nb[1] * t.ne[1] && t.nb[3] == t.nb[2] * t.ne[2] && (reinterpret_cast<uintptr_t>(t.data) & 15) == 0;
}

cudaError_t binary(int op, const TensorView & a, const TensorView & b, const TensorView & y, cudaStream_t st) {
    const int64_t n = y.ne[0] * y.ne[1] * y.ne[2] * y.ne[3];
    if (n == 0) return cudaSuccess;
    note_launch();
    if (op < 2 && n % 4 == 0 && n >= 4096 && flat_f32(a) && flat_f32(b) && flat_f32(y) && a.ne[0] == b.ne[0] && a.ne[1] == b.ne[1] && a.ne[2] == b.ne[2] && a.ne[3] == b.ne[3] &&
        a.ne[0] == y.ne[0] && a.ne[1] == y.ne[1] && a.ne[2] == y.ne[2] && a.ne[3] == y.ne[3]) {
        const int64_t n4 = n / 4;
        const unsigned grid = (unsigned)(cdiv(n4, 256) < 132 * 16 ? cdiv(n4, 256) : 132 * 16);
        binary_flat4_kernel<<<grid, 256, 0, st>>>(op, (const float4 *)a.data, (const float4 *)b.data, (float4 *)y.data, n4);
        return cudaGetLastError();
    }
    binary_kernel<<<cdiv(n, 256), 256, 0, st>>>(op, a, b, y, n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ SCALE
__global__ void __launch_bounds__(256) scale_kernel(const TensorView x, const TensorView y, float s, float b, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t i0 = i % y.ne[0], i1 = (i / y.ne[0]) % y.ne[1], i2 = (i / (y.ne[0] * y.ne[1])) % y.ne[2], i3 = i / (y.ne[0] * y.ne[1] * y.ne[2]);
    const float v = *reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i0 * x.nb[0] + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    *reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i0 * y.nb[0] + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]) = __fadd_rn(__fmul_rn(v, s), b);
}
cudaError_t scale(const TensorView & x, const TensorView & y, float s, float b, cudaStream_t st) {
    const int64_t n = y.ne[0] * y.ne[1] * y.ne[2] * y.ne[3];
    if (n == 0) return cudaSuccess;
    note_launch();
    scale_kernel<<<cdiv(n, 256), 256, 0, st>>>(x, y, s, b, n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ ROPE (normal / neox)
struct RopeP { int n_dims, mode; float freq_scale, ext_factor, attn_factor, theta_scale, corr0, corr1; };

__global__ void __launch_bounds__(128) rope_kernel(const TensorView x, const int32_t * __restrict__ pos, const float * __restrict__ ff,
                                                   const TensorView y, RopeP p) {
    // one CTA per (head i1, token i2, batch i3); cache[i] = (cos, sin) of pair i, theta iterated like the CPU cache init
    extern __shared__ float cache[];                       // n_dims floats
    const int i1 = blockIdx.x, i2 = blockIdx.y, i3 = blockIdx.z;
    const int half = p.n_dims / 2;
    if (threadIdx.x == 0) {
        float theta = (float)pos[i2];
        for (int i = 0; i < half; i++) { cache[i] = theta; theta = __fmul_rn(theta, p.theta_scale); }
    }
    __syncthreads();
    const float * xr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    float * yr = reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]);
    for (int i = threadIdx.x; i < half; i += blockDim.x) {
        const float theta_extrap = ff ? __fdiv_rn(cache[i], ff[i]) : cache[i];
        const float theta_interp = __fmul_rn(p.freq_scale, theta_extrap);
        float theta = theta_interp, mscale = p.attn_factor;
        if (p.ext_factor != 0.0f) {
            const float yv = ((float)i - p.corr0) / fmaxf(0.001f, p.corr1 - p.corr0);
            const float ramp_mix = (1.0f - fminf(1.0f, fmaxf(0.0f, yv))) * p.ext_factor;
            theta = theta_interp * (1.0f - ramp_mix) + theta_extrap * ramp_mix;
            mscale *= 1.0f + 0.1f * logf(1.0f / p.freq_scale);
        }
        const float c = cosf(theta) * mscale, s = sinf(theta) * mscale;
        const int ia = p.mode == 0 ? 2 * i : i, ib = p.mode == 0 ? 2 * i + 1 : i + half;
        const float x0 = xr[ia], x1 = xr[ib];
        yr[ia] = __fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, s));
        yr[ib] = __fadd_rn(__fmul_rn(x0, s), __fmul_rn(x1, c));
    }
    for (int i = p.n_dims + threadIdx.x; i < (int)x.ne[0]; i += blockDim.x) yr[i] = xr[i];   // pass-through channels
}

cudaError_t rope(const TensorView & x, const int32_t * pos, const float * ff, const TensorView & y, int n_dims, int mode, int n_ctx_orig,
                 float freq_base, float freq_scale, float ext_factor, float attn_factor, float beta_fast, float beta_slow, cudaStream_t st) {
    if (x.ne[0] * x.ne[1] * x.ne[2] * x.ne[3] == 0) return cudaSuccess;
    if (mode != 0 && mode != 2) return cudaErrorNotSupported;
    RopeP p;
    p.n_dims = n_dims; p.mode = mode; p.freq_scale = freq_scale; p.ext_factor = ext_factor; p.attn_factor = attn_factor;
    p.theta_scale = powf(freq_base, -2.0f / n_dims);
    // ggml_rope_yarn_corr_dims (ggml/src/ggml.c:4370-4383)
    auto corr_dim = [&](float n_rot) { return n_dims * logf(n_ctx_orig / (n_rot * 2 * 3.14159265358979323846f)) / (2 * logf(freq_base)); };
    const float start = floorf(corr_dim(beta_fast)), end = ceilf(corr_dim(beta_slow));
    p.corr0 = start > 0 ? start : 0;
    p.corr1 = end < n_dims - 1 ? end : (float)(n_dims - 1);
    note_launch();
    rope_kernel<<<dim3((unsigned)x.ne[1], (unsigned)x.ne[2], (unsigned)x.ne[3]), 128, sizeof(float) * (size_t)(n_dims / 2 + 1), st>>>(x, pos, ff, y, p);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ fused ROPE + KV store (decode)
__global__ void __launch_bounds__(128) rope_kv_kernel(const RopeKVArgs a, RopeP p, int b0) {
    extern __shared__ float cache[];
    pdl_prologue();
    const int b = blockIdx.x + b0;                               // [0, n_head): Q heads; [n_head, n_head + n_head_kv): K heads; then V chunks
    const int hd = a.head_dim;
    if (b >= a.n_head + a.n_head_kv) {                      // V: f32 -> f16 cache row
        const int h = b - a.n_head - a.n_head_kv;
        __half * dst = reinterpret_cast<__half *>(reinterpret_cast<char *>(a.v_cache) + __ldcg(a.v_idx) * a.v_row_bytes) + (int64_t)h * hd;
        const float * src = a.v_src + (int64_t)h * hd;
        for (int i = threadIdx.x; i < hd; i += blockDim.x) dst[i] = __float2half_rn(__ldcg(src + i));
        return;
    }
    const bool is_k = b >= a.n_head;
    const int h = is_k ? b - a.n_head : b;
    const float * xr = (is_k ? a.k_src : a.q_src) + (int64_t)h * hd;
    float * yr = (is_k ? a.k_dst : a.q_dst) + (int64_t)h * hd;
    __half * cr = is_k ? reinterpret_cast<__half *>(reinterpret_cast<char *>(a.k_cache) + __ldcg(a.k_idx) * a.k_row_bytes) + (int64_t)h * hd : nullptr;
    const int half = p.n_dims / 2;
    if (threadIdx.x == 0) {
        float theta = (float)__ldcg(a.pos);
        for (int i = 0; i < half; i++) { cache[i] = theta; theta = __fmul_rn(theta, p.theta_scale); }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < half; i += blockDim.x) {
        const float theta_extrap = a.freq_factors ? __fdiv_rn(cache[i], a.freq_factors[i]) : cache[i];
        const float theta_interp = __fmul_rn(p.freq_scale, theta_extrap);
        float theta = theta_interp, mscale = p.attn_factor;
        if (p.ext_factor != 0.0f) {
            const float yv = ((float)i - p.corr0) / fmaxf(0.001f, p.corr1 - p.corr0);
            const float ramp_mix = (1.0f - fminf(1.0f, fmaxf(0.0f, yv))) * p.ext_factor;
            theta = theta_interp * (1.0f - ramp_mix) + theta_extrap * ramp_mix;
            mscale *= 1.0f + 0.1f * logf(1.0f / p.freq_scale);
        }
        const float c = cosf(theta) * mscale, s = sinf(theta) * mscale;
        const int ia = p.mode == 0 ? 2 * i : i, ib = p.mode == 0 ? 2 * i + 1 : i + half;
        const float x0 = __ldcg(xr + ia), x1 = __ldcg(xr + ib);
        const float y0 = __fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, s)), y1 = __fadd_rn(__fmul_rn(x0, s), __fmul_rn(x1, c));
        yr[ia] = y0; yr[ib] = y1;
        if (cr) { cr[ia] = __float2half_rn(y0); cr[ib] = __float2half_rn(y1); }
    }
    for (int i = p.n_dims + threadIdx.x; i < hd; i += blockDim.x) { const float v = __ldcg(xr + i); yr[i] = v; if (cr) cr[i] = __float2half_rn(v); }
}

void rope_derived(const RopeKVArgs & a, float & theta_scale, float & corr0, float & corr1) {
    theta_scale = powf(a.freq_base, -2.0f / a.n_dims);
    auto corr_dim = [&](float n_rot) { return a.n_dims * logf(a.n_ctx_orig / (n_rot * 2 * 3.14159265358979323846f)) / (2 * logf(a.freq_base)); };
    const float start = floorf(corr_dim(a.beta_fast)), end = ceilf(corr_dim(a.beta_slow));
    corr0 = start > 0 ? start : 0;
    corr1 = end < a.n_dims - 1 ? end : (float)(a.n_dims - 1);
}

cudaError_t rope_kv_store(const RopeKVArgs & a, cudaStream_t st) {
    if (a.mode != 0 && a.mode != 2) return cudaErrorNotSupported;
    RopeP p;
    p.n_dims = a.n_dims; p.mode = a.mode; p.freq_scale = a.freq_scale; p.ext_factor = a.ext_factor; p.attn_factor = a.attn_factor;
    rope_derived(a, p.theta_scale, p.corr0, p.corr1);
    note_launch();
    static const bool split = getenv("GGML_B200_ROPE_SPLIT") != nullptr;          // (bisection: Q, K and V heads as three launches)
    if (split) {
        cudaError_t e = launch_pdl(rope_kv_kernel, dim3((unsigned)a.n_head), dim3(128), sizeof(float) * (size_t)(a.n_dims / 2 + 1), st, a, p, 0);
        if (e == cudaSuccess) e = launch_pdl(rope_kv_kernel, dim3((unsigned)a.n_head_kv), dim3(128), sizeof(float) * (size_t)(a.n_dims / 2 + 1), st, a, p, a.n_head);
        if (e == cudaSuccess) e = launch_pdl(rope_kv_kernel, dim3((unsigned)a.n_head_kv), dim3(128), sizeof(float) * (size_t)(a.n_dims / 2 + 1), st, a, p, a.n_head + a.n_head_kv);
        return e;
    }
    return launch_pdl(rope_kv_kernel, dim3((unsigned)(a.n_head + 2 * a.n_head_kv)), dim3(128), sizeof(float) * (size_t)(a.n_dims / 2 + 1), st, a, p, 0);
}

// ------------------------------------------------------------------------------------------------ SET_ROWS / GET_ROWS
__global__ void __launch_bounds__(256) set_rows_kernel(const TensorView src, const TensorView idx, const TensorView dst) {
    const int64_t r = blockIdx.x;                           // row over (i01, i02, i03)
    const int64_t i01 = r % src.ne[1], i02 = (r / src.ne[1]) % src.ne[2], i03 = r / (src.ne[1] * src.ne[2]);
    const int64_t i11 = i02 % idx.ne[1], i12 = i03 % idx.ne[2];
    const int64_t row = *reinterpret_cast<const int64_t *>(reinterpret_cast<const char *>(idx.data) + i01 * idx.nb[0] + i11 * idx.nb[1] + i12 * idx.nb[2]);
    const float * s = reinterpret_cast<const float *>(reinterpret_cast<const char *>(src.data) + i01 * src.nb[1] + i02 * src.nb[2] + i03 * src.nb[3]);
    char * d = reinterpret_cast<char *>(dst.data) + row * dst.nb[1] + i02 * dst.nb[2] + i03 * dst.nb[3];
    for (int i = threadIdx.x; i < (int)src.ne[0]; i += blockDim.x) store_from_f32(d + (int64_t)i * dst.nb[0], dst.type, s[i]);
}

cudaError_t set_rows(const TensorView & src, const TensorView & idx, const TensorView & dst, cudaStream_t st) {
    const int64_t rows = src.ne[1] * src.ne[2] * src.ne[3];
    if (rows == 0 || src.ne[0] == 0) return cudaSuccess;
    if (dst.type != TY_F32 && dst.type != TY_F16) return cudaErrorNotSupported;
    note_launch();
    set_rows_kernel<<<(unsigned)rows, 256, 0, st>>>(src, idx, dst);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) get_rows_kernel(const TensorView src, const TensorView idx, const TensorView dst, int be, int bb) {
    const int64_t r = blockIdx.x;                           // (i10, i11, i12)
    const int64_t i10 = r % idx.ne[0], i11 = (r / idx.ne[0]) % idx.ne[1], i12 = r / (idx.ne[0] * idx.ne[1]);
    const int32_t row = *reinterpret_cast<const int32_t *>(reinterpret_cast<const char *>(idx.data) + i10 * idx.nb[0] + i11 * idx.nb[1] + i12 * idx.nb[2]);
    const uint8_t * s = reinterpret_cast<const uint8_t *>(src.data) + (int64_t)row * src.nb[1] + i11 * src.nb[2] + i12 * src.nb[3];
    float * d = reinterpret_cast<float *>(reinterpret_cast<char *>(dst.data) + i10 * dst.nb[1] + i11 * dst.nb[2] + i12 * dst.nb[3]);
    for (int i = threadIdx.x; i < (int)src.ne[0]; i += blockDim.x) {
        float v;
        if (src.type == TY_F32) v = reinterpret_cast<const float *>(s)[i];
        else if (src.type == TY_F16) v = __half2float(reinterpret_cast<const __half *>(s)[i]);
        else v = dequant_elem(src.type, s + (int64_t)(i / be) * bb, i % be);
        d[i] = v;
    }
}

cudaError_t get_rows(const TensorView & src, const TensorView & idx, const TensorView & dst, cudaStream_t st) {
    const int64_t rows = idx.ne[0] * idx.ne[1] * idx.ne[2];
    if (rows == 0 || src.ne[0] == 0) return cudaSuccess;
    int be = 1, bb = 4;
    if (src.type != TY_F32 && src.type != TY_F16) { be = block_elems(src.type); bb = block_bytes(src.type); if (!bb) return cudaErrorNotSupported; }
    note_launch();
    get_rows_kernel<<<(unsigned)rows, 256, 0, st>>>(src, idx, dst, be, bb);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ GLU: SWIGLU
__global__ void __launch_bounds__(256) swiglu_kernel(const TensorView a, const TensorView b, bool split, bool swapped, const TensorView y, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t nc = y.ne[0];
    const int64_t i0 = i % nc, r = i / nc;
    const int64_t i1 = r % y.ne[1], i2 = (r / y.ne[1]) % y.ne[2], i3 = r / (y.ne[1] * y.ne[2]);
    const char * ar = reinterpret_cast<const char *>(a.data) + i1 * a.nb[1] + i2 * a.nb[2] + i3 * a.nb[3];
    const char * br = split ? ar : reinterpret_cast<const char *>(b.data) + i1 * b.nb[1] + i2 * b.nb[2] + i3 * b.nb[3];
    float x, g;
    if (split) {
        x = reinterpret_cast<const float *>(ar)[swapped ? i0 + nc : i0];
        g = reinterpret_cast<const float *>(ar)[swapped ? i0 : i0 + nc];
    } else {
        x = reinterpret_cast<const float *>(ar)[i0];
        g = reinterpret_cast<const float *>(br)[i0];
    }
    const float silu = __fdiv_rn(x, __fadd_rn(1.0f, expf(-x)));
    reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3])[i0] = __fmul_rn(silu, g);
}

__global__ void __launch_bounds__(256) swiglu_flat4_kernel(const float4 * __restrict__ a, const float4 * __restrict__ b, float4 * __restrict__ y, int64_t n4) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 x = a[i], g = b[i];
        float4 r;
        r.x = __fmul_rn(__fdiv_rn(x.x, __fadd_rn(1.0f, expf(-x.x))), g.x);
        r.y = __fmul_rn(__fdiv_rn(x.y, __fadd_rn(1.0f, expf(-x.y))), g.y);
        r.z = __fmul_rn(__fdiv_rn(x.z, __fadd_rn(1.0f, expf(-x.z))), g.z);
        r.w = __fmul_rn(__fdiv_rn(x.w, __fadd_rn(1.0f, expf(-x.w))), g.w);
        y[i] = r;
    }
}

cudaError_t swiglu(const TensorView & a, const TensorView * b, const TensorView & y, bool swapped, cudaStream_t st) {
    const int64_t n = y.ne[0] * y.ne[1] * y.ne[2] * y.ne[3];
    if (n == 0) return cudaSuccess;
    note_launch();
    if (b != nullptr && !swapped && n % 4 == 0 && n >= 4096 && flat_f32(a) && flat_f32(*b) && flat_f32(y) && a.ne[0] == y.ne[0] && b->ne[0] == y.ne[0] &&
        a.ne[1] * a.ne[2] * a.ne[3] == y.ne[1] * y.ne[2] * y.ne[3] && b->ne[1] * b->ne[2] * b->ne[3] == y.ne[1] * y.ne[2] * y.ne[3]) {
        const int64_t n4 = n / 4;
        const unsigned grid = (unsigned)(cdiv(n4, 256) < 132 * 16 ? cdiv(n4, 256) : 132 * 16);
        swiglu_flat4_kernel<<<grid, 256, 0, st>>>((const float4 *)a.data, (const float4 *)b->data, (float4 *)y.data, n4);
        return cudaGetLastError();
    }
    swiglu_kernel<<<cdiv(n, 256), 256, 0, st>>>(a, b ? *b : a, b == nullptr, swapped, y, n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ CPY / CONT / DUP
__global__ void __launch_bounds__(256) copy_kernel(const TensorView s, const TensorView d, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t s0 = i % s.ne[0], s1 = (i / s.ne[0]) % s.ne[1], s2 = (i / (s.ne[0] * s.ne[1])) % s.ne[2], s3 = i / (s.ne[0] * s.ne[1] * s.ne[2]);
    const int64_t d0 = i % d.ne[0], d1 = (i / d.ne[0]) % d.ne[1], d2 = (i / (d.ne[0] * d.ne[1])) % d.ne[2], d3 = i / (d.ne[0] * d.ne[1] * d.ne[2]);
    const float v = load_as_f32(reinterpret_cast<const char *>(s.data) + s0 * s.nb[0] + s1 * s.nb[1] + s2 * s.nb[2] + s3 * s.nb[3], s.type);
    store_from_f32(reinterpret_cast<char *>(d.data) + d0 * d.nb[0] + d1 * d.nb[1] + d2 * d.nb[2] + d3 * d.nb[3], d.type, v);
}

cudaError_t copy(const TensorView & src, const TensorView & dst, cudaStream_t st) {
    const int64_t n = src.ne[0] * src.ne[1] * src.ne[2] * src.ne[3];
    if (n == 0) return cudaSuccess;
    if ((src.type != TY_F32 && src.type != TY_F16) || (dst.type != TY_F32 && dst.type != TY_F16)) return cudaErrorNotSupported;
    note_launch();
    copy_kernel<<<cdiv(n, 256), 256, 0, st>>>(src, dst, n);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ multi-region copy
__global__ void __launch_bounds__(256) multi_copy_kernel(const MultiCopyArgs a) {
    const int r = blockIdx.x;
    if (r >= a.n) return;
    const unsigned char * s = reinterpret_cast<const unsigned char *>(a.src[r]);
    unsigned char * d = reinterpret_cast<unsigned char *>(a.dst[r]);
    for (unsigned i = threadIdx.x; i < a.bytes[r]; i += blockDim.x) d[i] = s[i];
}
cudaError_t multi_copy(const MultiCopyArgs & a, cudaStream_t st) {
    if (a.n <= 0) return cudaSuccess;
    multi_copy_kernel<<<a.n, 256, 0, st>>>(a);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ FLASH_ATTN_EXT
// q [DK, N, H, B] f32 (strided), k [DK, KV, Hkv, B] f16, v [DV, KV, Hkv, B] f16, mask [KV, >=N, 1|H, 1|B] f16 or none,
// dst [DV, H, N, B] f32.  One CTA (4 warps) per (query, head): each warp walks kv positions w, w+4, ... with an online
// softmax; lanes split the head dimension (D/32 elements each, D <= 256); the 4 partial (M, S, acc) are merged in smem.
template <int DPL>   // head-dim elements per lane
__global__ void __launch_bounds__(128) flash_attn_kernel(const TensorView q, const TensorView k, const TensorView v, const TensorView mask, bool has_mask,
                                                         const TensorView dst, float scale, float softcap) {
    pdl_prologue();
    const int iq1 = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int hk = h / (int)(q.ne[2] / k.ne[2]), hv = h / (int)(q.ne[2] / v.ne[2]);
    const int bk = b / (int)(q.ne[3] / k.ne[3]), bv = b / (int)(q.ne[3] / v.ne[3]);
    const float * qr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(q.data) + iq1 * q.nb[1] + h * q.nb[2] + b * q.nb[3]);
    float qv[DPL];
#pragma unroll
    for (int i = 0; i < DPL; i++) qv[i] = __half2float(__float2half_rn(__ldcg(qr + lane * DPL + i)));   // PDL: producer data is read past L1   // the CPU converts q to f16 first (K is f16)
    const char * kb = reinterpret_cast<const char *>(k.data) + hk * k.nb[2] + bk * k.nb[3];
    const char * vb = reinterpret_cast<const char *>(v.data) + hv * v.nb[2] + bv * v.nb[3];
    const __half * mp = has_mask ? reinterpret_cast<const __half *>(reinterpret_cast<const char *>(mask.data) + iq1 * mask.nb[1] +
                                                                     (h % mask.ne[2]) * mask.nb[2] + (b % mask.ne[3]) * mask.nb[3]) : nullptr;
    const int n_kv = (int)k.ne[1];
    float M = -INFINITY, S = 0.0f, acc[DPL];
#pragma unroll
    for (int i = 0; i < DPL; i++) acc[i] = 0.0f;
    for (int ic = warp; ic < n_kv; ic += 4) {
        const float mv = mp ? __half2float(mp[ic]) : 0.0f;
        if (mv == -INFINITY) continue;                      // warp-uniform: same ic for all lanes
        const __half * kr = reinterpret_cast<const __half *>(kb + (int64_t)ic * k.nb[1]) + lane * DPL;
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < DPL; i++) s += qv[i] * __half2float(kr[i]);   // K/V/mask lines cannot be stale: nothing on this SM reads them between our launch and here
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        s *= scale;
        if (softcap != 0.0f) s = softcap * tanhf(s);
        s += mv;
        const float Mnew = fmaxf(M, s);
        const float ms = expf(M - Mnew), vs = expf(s - Mnew);
        const __half * vr = reinterpret_cast<const __half *>(vb + (int64_t)ic * v.nb[1]) + lane * DPL;
#pragma unroll
        for (int i = 0; i < DPL; i++) acc[i] = acc[i] * ms + vs * __half2float(vr[i]);
        S = S * ms + vs;
        M = Mnew;
    }
    __shared__ float sM[4], sS[4], sacc[4][32 * DPL];
    if (lane == 0) { sM[warp] = M; sS[warp] = S; }
#pragma unroll
    for (int i = 0; i < DPL; i++) sacc[warp][lane * DPL + i] = acc[i];
    __syncthreads();
    if (warp == 0) {
        float Mt = fmaxf(fmaxf(sM[0], sM[1]), fmaxf(sM[2], sM[3]));
        float St = 0.0f, out[DPL];
#pragma unroll
        for (int i = 0; i < DPL; i++) out[i] = 0.0f;
#pragma unroll
        for (int w = 0; w < 4; w++) {
            const float f = sM[w] == -INFINITY ? 0.0f : expf(sM[w] - Mt);
            St += sS[w] * f;
#pragma unroll
            for (int i = 0; i < DPL; i++) out[i] += sacc[w][lane * DPL + i] * f;
        }
        const float inv = St == 0.0f ? 0.0f : 1.0f / St;
        float * dr = reinterpret_cast<float *>(reinterpret_cast<char *>(dst.data) + h * dst.nb[1] + iq1 * dst.nb[2] + b * dst.nb[3]);
#pragma unroll
        for (int i = 0; i < DPL; i++) dr[lane * DPL + i] = out[i] * inv;
    }
}

static bool fa_mma_enabled() {
    static const bool on = [] { const char * e = getenv("GGML_B200_FA_MMA"); return !(e && e[0] == '0'); }();
    return on;
}

cudaError_t flash_attn(const TensorView & q, const TensorView & k, const TensorView & v, const TensorView * mask, const TensorView & dst,
                       float scale, float softcap, cudaStream_t st, void * ws, size_t ws_bytes) {
    if (q.ne[1] >= FA_MIN_ROWS_MMA && fa_mma_enabled()) {
        const cudaError_t pe = flash_attn_prefill(q, k, v, mask, dst, scale, softcap, ws, ws_bytes, st);
        if (pe != cudaErrorNotSupported) return pe;
    }
    return flash_attn_scalar(q, k, v, mask, dst, scale, softcap, st);
}

cudaError_t flash_attn_scalar(const TensorView & q, const TensorView & k, const TensorView & v, const TensorView * mask, const TensorView & dst,
                              float scale, float softcap, cudaStream_t st) {
    const int D = (int)q.ne[0];
    if (D != (int)v.ne[0] || D % 32 || D > 256 || k.type != TY_F16 || v.type != TY_F16 || q.type != TY_F32) return cudaErrorNotSupported;
    if (q.ne[1] * q.ne[2] * q.ne[3] == 0) return cudaSuccess;
    if (softcap != 0.0f) scale /= softcap;
    const dim3 grid((unsigned)q.ne[1], (unsigned)q.ne[2], (unsigned)q.ne[3]);
    note_launch();
    cudaError_t le = cudaSuccess;
#define QMM_FA(DPL) le = launch_pdl(flash_attn_kernel<DPL>, grid, dim3(128), 0, st, q, k, v, mask ? *mask : q, mask != nullptr, dst, scale, softcap)
    switch (D / 32) {
        case 1: QMM_FA(1); break; case 2: QMM_FA(2); break; case 3: QMM_FA(3); break; case 4: QMM_FA(4); break;
        case 5: QMM_FA(5); break; case 6: QMM_FA(6); break; case 7: QMM_FA(7); break; case 8: QMM_FA(8); break;
        default: return cudaErrorNotSupported;
    }
#undef QMM_FA
    return le;
}

// ------------------------------------------------------------------------------------------------ the MoE router's small ops
// (build_moe_ffn, src/llama-graph.cpp:1941-2200: logits = gate_inp x cur; probs = soft_max; top-k via ARGSORT + view; weights =
//  get_rows(probs); weights /= sum_rows(weights)).  All tiny ([n_expert, n_tokens]); they exist so that a MoE graph has no node left
//  for the CPU backend (every CPU node costs two graph splits and a device round trip per layer).

// MUL_MAT with f32 / f16 weights: y[m, n] = sum_k w[k, m] * x[k, n].  One warp per output element, fp32 accumulation (the CPU's
// ggml_vec_dot_f32 / _f16 also accumulate in fp32, in SIMD-lane order; f16 weights: the CPU converts x to f16 first, so do we).
__global__ void __launch_bounds__(128) mul_mat_f_kernel(const TensorView w, const TensorView x, const TensorView y) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t m = (int64_t)blockIdx.x * 4 + warp, n = blockIdx.y;
    if (m >= w.ne[1]) return;
    const char * wr = reinterpret_cast<const char *>(w.data) + m * w.nb[1];
    const float * xr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + n * x.nb[1]);
    float acc = 0.0f;
    if (w.type == TY_F32) {
        for (int64_t k = lane; k < w.ne[0]; k += 32) acc = fmaf(reinterpret_cast<const float *>(wr)[k], xr[k], acc);
    } else {
        for (int64_t k = lane; k < w.ne[0]; k += 32) acc = fmaf(__half2float(reinterpret_cast<const __half *>(wr)[k]), __half2float(__float2half_rn(xr[k])), acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) *reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + m * y.nb[0] + n * y.nb[1]) = acc;
}
cudaError_t mul_mat_f(const TensorView & w, const TensorView & x, const TensorView & y, cudaStream_t st) {
    if ((w.type != TY_F32 && w.type != TY_F16) || x.type != TY_F32 || y.type != TY_F32) return cudaErrorNotSupported;
    if (w.ne[1] * x.ne[1] == 0) return cudaSuccess;
    note_launch();
    mul_mat_f_kernel<<<dim3(cdiv(w.ne[1], 4), (unsigned)x.ne[1]), 128, 0, st>>>(w, x, y);
    return cudaGetLastError();
}

// SOFT_MAX (ggml_compute_forward_soft_max_f32, ops.cpp:5451-5565; max_bias == 0, no sinks): y = softmax(x * scale + mask) per row;
// the sum of the exponentials is accumulated in double and the row scaled by (float)(1 / sum), as the CPU does.
__global__ void __launch_bounds__(256) soft_max_kernel(const TensorView x, const TensorView mask, bool has_mask, const TensorView y, float scale) {
    __shared__ float smax[8];
    __shared__ double ssum[8];
    const int64_t row = blockIdx.x;
    const int64_t i1 = row % x.ne[1], i2 = (row / x.ne[1]) % x.ne[2], i3 = row / (x.ne[1] * x.ne[2]);
    const float * xr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    float * yr = reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]);
    const char * mr = has_mask ? reinterpret_cast<const char *>(mask.data) + i1 * mask.nb[1] + (i2 % mask.ne[2]) * mask.nb[2] + (i3 % mask.ne[3]) * mask.nb[3] : nullptr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto val = [&](int64_t i) {
        float v = __fmul_rn(xr[i], scale);
        if (mr) v = __fadd_rn(v, mask.type == TY_F16 ? __half2float(reinterpret_cast<const __half *>(mr)[i]) : reinterpret_cast<const float *>(mr)[i]);
        return v;
    };
    float mx = -INFINITY;
    for (int64_t i = threadIdx.x; i < x.ne[0]; i += blockDim.x) mx = fmaxf(mx, val(i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) smax[warp] = mx;
    __syncthreads();
    mx = smax[0];
#pragma unroll
    for (int i = 1; i < 8; i++) mx = fmaxf(mx, smax[i]);
    double sum = 0.0;
    for (int64_t i = threadIdx.x; i < x.ne[0]; i += blockDim.x) {
        const float e = expf(val(i) - mx);
        yr[i] = e;
        sum += (double)e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) ssum[warp] = sum;
    __syncthreads();
    sum = 0.0;
#pragma unroll
    for (int i = 0; i < 8; i++) sum += ssum[i];
    const float inv = (float)(1.0 / sum);
    for (int64_t i = threadIdx.x; i < x.ne[0]; i += blockDim.x) yr[i] = __fmul_rn(yr[i], inv);
}
cudaError_t soft_max(const TensorView & x, const TensorView * mask, const TensorView & y, float scale, cudaStream_t st) {
    const int64_t rows = x.ne[1] * x.ne[2] * x.ne[3];
    if (rows == 0 || x.ne[0] == 0) return cudaSuccess;
    note_launch();
    soft_max_kernel<<<(unsigned)rows, 256, 0, st>>>(x, mask ? *mask : x, mask != nullptr, y, scale);
    return cudaGetLastError();
}

// ARGSORT (ops.cpp:8350-8389): indices of a row's values in ascending / descending order; bitonic sort of (value, index) pairs in
// shared memory, rows of up to 1024 elements (expert counts).  Ties: lower index first (std::sort leaves them unspecified).
__global__ void __launch_bounds__(512) argsort_kernel(const TensorView x, const TensorView y, int npad, bool desc) {
    extern __shared__ float sv[];                 // npad values, then npad indices
    int * si = reinterpret_cast<int *>(sv + npad);
    const int64_t row = blockIdx.x;
    const int64_t i1 = row % x.ne[1], i2 = (row / x.ne[1]) % x.ne[2], i3 = row / (x.ne[1] * x.ne[2]);
    const float * xr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    int32_t * yr = reinterpret_cast<int32_t *>(reinterpret_cast<char *>(y.data) + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]);
    const int n = (int)x.ne[0];
    for (int i = threadIdx.x; i < npad; i += blockDim.x) { sv[i] = i < n ? xr[i] : 0.0f; si[i] = i < n ? i : -1; }
    __syncthreads();
    // "a before b": padding last; then by value in the requested order; then by index
    auto before = [&](int a, int b) {
        const int ia = si[a], ib = si[b];
        if (ia < 0 || ib < 0) return ib < 0 && ia >= 0;
        const float va = sv[a], vb = sv[b];
        if (va != vb) return desc ? va > vb : va < vb;
        return ia < ib;
    };
    for (int k = 2; k <= npad; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < npad; i += blockDim.x) {
                const int p = i ^ j;
                if (p > i) {
                    const bool up = (i & k) == 0;
                    const bool swap = up ? before(p, i) : before(i, p);
                    if (swap) { const float tv = sv[i]; sv[i] = sv[p]; sv[p] = tv; const int ti = si[i]; si[i] = si[p]; si[p] = ti; }
                }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) yr[i] = si[i];
}
cudaError_t argsort(const TensorView & x, const TensorView & y, bool desc, cudaStream_t st) {
    const int64_t rows = x.ne[1] * x.ne[2] * x.ne[3];
    if (x.ne[0] > 1024) return cudaErrorNotSupported;
    if (rows == 0 || x.ne[0] == 0) return cudaSuccess;
    int npad = 1;
    while (npad < x.ne[0]) npad <<= 1;
    note_launch();
    argsort_kernel<<<(unsigned)rows, npad < 32 ? 32 : (npad > 512 ? 512 : npad), (size_t)npad * 8, st>>>(x, y, npad, desc);
    return cudaGetLastError();
}

// SUM_ROWS (ops.cpp:1456-1492; ggml_vec_sum_f32 accumulates in ggml_float = double): one warp per row
__global__ void __launch_bounds__(128) sum_rows_kernel(const TensorView x, const TensorView y, int64_t rows) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int64_t i1 = row % x.ne[1], i2 = (row / x.ne[1]) % x.ne[2], i3 = row / (x.ne[1] * x.ne[2]);
    const float * xr = reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    double acc = 0.0;
    for (int64_t i = lane; i < x.ne[0]; i += 32) acc += (double)xr[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) *reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]) = (float)acc;
}
cudaError_t sum_rows(const TensorView & x, const TensorView & y, cudaStream_t st) {
    const int64_t rows = x.ne[1] * x.ne[2] * x.ne[3];
    if (rows == 0) return cudaSuccess;
    note_launch();
    sum_rows_kernel<<<cdiv(rows, 4), 128, 0, st>>>(x, y, rows);
    return cudaGetLastError();
}

// CLAMP (ops.cpp:5680-5725): y = max(min(x, hi), lo)
__global__ void __launch_bounds__(256) clamp_kernel(const TensorView x, const TensorView y, float lo, float hi, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t i0 = i % y.ne[0], i1 = (i / y.ne[0]) % y.ne[1], i2 = (i / (y.ne[0] * y.ne[1])) % y.ne[2], i3 = i / (y.ne[0] * y.ne[1] * y.ne[2]);
    const float v = *reinterpret_cast<const float *>(reinterpret_cast<const char *>(x.data) + i0 * x.nb[0] + i1 * x.nb[1] + i2 * x.nb[2] + i3 * x.nb[3]);
    *reinterpret_cast<float *>(reinterpret_cast<char *>(y.data) + i0 * y.nb[0] + i1 * y.nb[1] + i2 * y.nb[2] + i3 * y.nb[3]) = fmaxf(fminf(v, hi), lo);
}
cudaError_t clamp(const TensorView & x, const TensorView & y, float lo, float hi, cudaStream_t st) {
    const int64_t n = y.ne[0] * y.ne[1] * y.ne[2] * y.ne[3];
    if (n == 0) return cudaSuccess;
    note_launch();
    clamp_kernel<<<cdiv(n, 256), 256, 0, st>>>(x, y, lo, hi, n);
    return cudaGetLastError();
}

}  // namespace ops
}  // namespace qmm
