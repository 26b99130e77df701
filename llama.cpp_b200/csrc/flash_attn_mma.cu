// flash_attn_mma.cu -- FLASH_ATTN_EXT for prompt processing (many query rows): tiled online-softmax attention on the
// tensor cores.  Semantics follow ggml_compute_forward_flash_attn_ext_f16 (ggml/src/ggml-cpu/ops.cpp): q is rounded to
// f16 (K is f16), scores = scale * q.k (+ softcap) + mask, softmax over kv, dst = P.V; dst layout [DV, H, N, B].
//
// This is a supporting op of the mat-mul path (SURVEY.md section 8f rank 1), not the headline kernel: at pp2048 its
// FLOPs are 4 % of the weight GEMMs'.  It uses warp-level mma.sync.m16n8k16 (f16 x f16 -> f32), which is enough to take
// attention from 60 % of the prefill step (scalar kernel in ops.cu) to a few per cent; the wgmma budget goes to the
// quantised GEMM (gemm_tcgen05.cu).
//
// Shape: one CTA = 4 warps = 64 query rows of one head; KV tiles of 64 keys double-buffered with cp.async (L2 only: .cg).
// A pre-pass marks (query tile, kv tile) pairs whose mask is entirely -inf; the main kernel visits active tiles only, so a
// causal prompt costs half the tiles without the op knowing the mask is causal.
#include <cuda_fp16.h>

#include "qmm_kernels.cuh"
#include "qmm_ops.cuh"

namespace qmm {
namespace ops {

namespace {

constexpr int FA_BM = 64, FA_BN = 64, FA_THREADS = 128;
constexpr int FA_MAX_TILES = 2048;                       // kv tiles per row block (n_kv <= 131072)
constexpr int TY_F32_ = 0, TY_F16_ = 1;

__device__ __forceinline__ uint32_t sa(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp16(void * dst, const void * src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], const void * p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(sa(p)));
}
__device__ __forceinline__ void ldsm4t(uint32_t (&r)[4], const void * p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];\n" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(sa(p)));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}

// flags[(mz * n_qt + qt) * n_kt + kt] = 1 iff some mask entry of the 64 x 64 tile is not -inf.  64 threads: one per query row.
__global__ void __launch_bounds__(64) fa_tile_flags_kernel(const TensorView mask, int N, int n_kv, int n_kt, int n_qt, uint8_t * __restrict__ flags) {
    pdl_prologue();
    const int kt = blockIdx.x, qt = blockIdx.y, mz = blockIdx.z;
    const int m2 = mz % (int)mask.ne[2], m3 = mz / (int)mask.ne[2];
    const int iq = qt * FA_BM + (int)threadIdx.x;
    int any = 0;
    if (iq < N) {
        const __half * mp = reinterpret_cast<const __half *>(reinterpret_cast<const char *>(mask.data) + iq * mask.nb[1] + m2 * mask.nb[2] + m3 * mask.nb[3]);
        const int k0 = kt * FA_BN, k1 = min(n_kv, k0 + FA_BN);
        for (int ic = k0; ic < k1; ic++) any |= (int)(__ldcg(reinterpret_cast<const unsigned short *>(mp) + ic) != 0xFC00u);
    }
    any = __syncthreads_or(any);
    if (threadIdx.x == 0) flags[((int64_t)mz * n_qt + qt) * n_kt + kt] = (uint8_t)(any != 0);
}

template <int D>
struct FaSmem {
    static constexpr int LD = D + 8;                     // halves per K/V/Q row (16-byte pad: conflict-free ldmatrix)
    static constexpr int LDM = FA_BN + 8;                // halves per mask row
    static constexpr size_t q_bytes = (size_t)FA_BM * LD * 2;
    static constexpr size_t kv_bytes = (size_t)FA_BN * LD * 2;
    static constexpr size_t m_bytes = (size_t)FA_BM * LDM * 2;
    static constexpr size_t total = q_bytes + 4 * kv_bytes + 2 * m_bytes;
};

template <int D>
__global__ void __launch_bounds__(FA_THREADS) fa_mma_kernel(const TensorView q, const TensorView k, const TensorView v, const TensorView mask, bool has_mask,
                                                            const TensorView dst, float scale, float softcap, const uint8_t * __restrict__ flags, int n_kt,
                                                            int n_qt, bool mask_al16) {
    using S = FaSmem<D>;
    constexpr int LD = S::LD, LDM = S::LDM, KS = D / 16, NT = D / 8;
    extern __shared__ __align__(16) uint8_t fa_smem[];
    __half * sQ = reinterpret_cast<__half *>(fa_smem);
    __half * sK = reinterpret_cast<__half *>(fa_smem + S::q_bytes);                       // [2][FA_BN][LD]
    __half * sV = reinterpret_cast<__half *>(fa_smem + S::q_bytes + 2 * S::kv_bytes);      // [2][FA_BN][LD]
    __half * sM = reinterpret_cast<__half *>(fa_smem + S::q_bytes + 4 * S::kv_bytes);      // [2][FA_BM][LDM]
    __shared__ unsigned short s_list[FA_MAX_TILES];
    __shared__ int s_cnt;

    pdl_prologue();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int N = (int)q.ne[1], n_kv = (int)k.ne[1];
    const int q0 = qt * FA_BM;
    const int hk = h / (int)(q.ne[2] / k.ne[2]), hv = h / (int)(q.ne[2] / v.ne[2]);
    const int bk = b / (int)(q.ne[3] / k.ne[3]), bv = b / (int)(q.ne[3] / v.ne[3]);
    const char * kbase = reinterpret_cast<const char *>(k.data) + hk * k.nb[2] + bk * k.nb[3];
    const char * vbase = reinterpret_cast<const char *>(v.data) + hv * v.nb[2] + bv * v.nb[3];
    const int m2 = has_mask ? h % (int)mask.ne[2] : 0, m3 = has_mask ? b % (int)mask.ne[3] : 0;
    const char * mbase = has_mask ? reinterpret_cast<const char *>(mask.data) + m2 * mask.nb[2] + m3 * mask.nb[3] : nullptr;

    // ---- active kv tiles of this row block (order preserved)
    if (warp == 0) {
        const uint8_t * fl = (has_mask && flags) ? flags + ((int64_t)(m3 * (int)mask.ne[2] + m2) * n_qt + qt) * n_kt : nullptr;
        int cnt = 0;
        for (int base = 0; base < n_kt; base += 32) {
            const int t = base + lane;
            const bool act = t < n_kt && (fl == nullptr || __ldcg(fl + t) != 0);
            const unsigned bal = __ballot_sync(0xffffffffu, act);
            if (act) s_list[cnt + __popc(bal & ((1u << lane) - 1u))] = (unsigned short)t;
            cnt += __popc(bal);
        }
        if (lane == 0) s_cnt = cnt;
    }
    // ---- Q tile: f32 -> f16 (the CPU converts q to the K type before the dot products)
    for (int c = tid; c < FA_BM * (D / 4); c += FA_THREADS) {
        const int r = c / (D / 4), c4 = c % (D / 4);
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q0 + r < N) x = __ldcg(reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(q.data) + (int64_t)(q0 + r) * q.nb[1] + h * q.nb[2] + b * q.nb[3]) + c4);
        uint2 pk;
        pk.x = pack_h2(x.x, x.y);
        pk.y = pack_h2(x.z, x.w);
        *reinterpret_cast<uint2 *>(sQ + r * LD + 4 * c4) = pk;
    }
    __syncthreads();
    const int cnt = s_cnt;

    uint32_t qa[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ks++) ldsm4(qa[ks], sQ + (warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LD + ks * 16 + 8 * (lane >> 4));

    auto load_tile = [&](int kt, int stage) {
        __half * dK = sK + stage * FA_BN * LD;
        __half * dV = sV + stage * FA_BN * LD;
        const int key0 = kt * FA_BN;
        for (int c = tid; c < FA_BN * (D / 8); c += FA_THREADS) {
            const int r = c / (D / 8), ch = c % (D / 8);
            if (key0 + r < n_kv) {
                cp16(dK + r * LD + 8 * ch, kbase + (int64_t)(key0 + r) * k.nb[1] + 16 * ch);
                cp16(dV + r * LD + 8 * ch, vbase + (int64_t)(key0 + r) * v.nb[1] + 16 * ch);
            } else {
                *reinterpret_cast<uint4 *>(dK + r * LD + 8 * ch) = make_uint4(0, 0, 0, 0);
                *reinterpret_cast<uint4 *>(dV + r * LD + 8 * ch) = make_uint4(0, 0, 0, 0);
            }
        }
        if (has_mask) {
            __half * dM = sM + stage * FA_BM * LDM;
            for (int c = tid; c < FA_BM * (FA_BN / 8); c += FA_THREADS) {
                const int r = c / (FA_BN / 8), ch = c % (FA_BN / 8);
                const int kc = key0 + 8 * ch;
                __half * d = dM + r * LDM + 8 * ch;
                if (q0 + r < N && kc + 8 <= n_kv && mask_al16) {
                    cp16(d, mbase + (int64_t)(q0 + r) * mask.nb[1] + 2 * (int64_t)kc);
                } else if (q0 + r < N && kc < n_kv) {
                    const unsigned short * mp = reinterpret_cast<const unsigned short *>(mbase + (int64_t)(q0 + r) * mask.nb[1]);
#pragma unroll
                    for (int i = 0; i < 8; i++) d[i] = kc + i < n_kv ? __ushort_as_half(__ldcg(mp + kc + i)) : __ushort_as_half(0);
                } else {
                    *reinterpret_cast<uint4 *>(d) = make_uint4(0, 0, 0, 0);
                }
            }
        }
        cp_commit();
    };

    float o[NT][4];
#pragma unroll
    for (int i = 0; i < NT; i++) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.0f; }
    float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.0f, 0.0f};

    if (cnt > 0) load_tile(s_list[0], 0);
    for (int it = 0; it < cnt; it++) {
        const int stage = it & 1;
        const int kt = s_list[it];
        if (it + 1 < cnt) { load_tile(s_list[it + 1], stage ^ 1); cp_wait<1>(); } else { cp_wait<0>(); }
        __syncthreads();
        const __half * tK = sK + stage * FA_BN * LD;
        const __half * tV = sV + stage * FA_BN * LD;
        const __half * tM = sM + stage * FA_BM * LDM;

        // ---- S = Q K^T  (16 x 64 per warp)
        float s[FA_BN / 8][4];
#pragma unroll
        for (int i = 0; i < FA_BN / 8; i++) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.0f; }
#pragma unroll
        for (int ks = 0; ks < KS; ks++) {
#pragma unroll
            for (int np = 0; np < FA_BN / 16; np++) {
                uint32_t bf[4];
                ldsm4(bf, tK + (np * 16 + (lane & 7) + 8 * (lane >> 4)) * LD + ks * 16 + 8 * ((lane >> 3) & 1));
                mma16816(s[2 * np], qa[ks], bf[0], bf[1]);
                mma16816(s[2 * np + 1], qa[ks], bf[2], bf[3]);
            }
        }
        // ---- scale, softcap, mask, running max
        const int g = lane >> 2, t4 = lane & 3;
        const bool tail = kt * FA_BN + FA_BN > n_kv;
        float mnew[2] = {mrow[0], mrow[1]};
#pragma unroll
        for (int nt = 0; nt < FA_BN / 8; nt++) {
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int rr = e >> 1, col = nt * 8 + 2 * t4 + (e & 1);
                float x = s[nt][e] * scale;
                if (softcap != 0.0f) x = softcap * tanhf(x);
                if (has_mask) x += __half2float(tM[(warp * 16 + g + 8 * rr) * LDM + col]);
                if (tail && kt * FA_BN + col >= n_kv) x = -INFINITY;
                s[nt][e] = x;
                mnew[rr] = fmaxf(mnew[rr], x);
            }
        }
        float alpha[2], muse[2];
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
            mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 1));
            mnew[rr] = fmaxf(mnew[rr], __shfl_xor_sync(0xffffffffu, mnew[rr], 2));
            muse[rr] = mnew[rr] == -INFINITY ? 0.0f : mnew[rr];
            alpha[rr] = __expf(mrow[rr] - muse[rr]);
            mrow[rr] = mnew[rr];
        }
        float psum[2] = {0.0f, 0.0f};
        uint32_t pa[FA_BN / 16][4];
#pragma unroll
        for (int nt = 0; nt < FA_BN / 8; nt++) {
            const float p0 = __expf(s[nt][0] - muse[0]), p1 = __expf(s[nt][1] - muse[0]);
            const float p2 = __expf(s[nt][2] - muse[1]), p3 = __expf(s[nt][3] - muse[1]);
            psum[0] += p0 + p1;
            psum[1] += p2 + p3;
            pa[nt >> 1][(nt & 1) * 2 + 0] = pack_h2(p0, p1);
            pa[nt >> 1][(nt & 1) * 2 + 1] = pack_h2(p2, p3);
        }
        lrow[0] = lrow[0] * alpha[0] + psum[0];
        lrow[1] = lrow[1] * alpha[1] + psum[1];
#pragma unroll
        for (int i = 0; i < NT; i++) { o[i][0] *= alpha[0]; o[i][1] *= alpha[0]; o[i][2] *= alpha[1]; o[i][3] *= alpha[1]; }
        // ---- O += P V
#pragma unroll
        for (int kk = 0; kk < FA_BN / 16; kk++) {
#pragma unroll
            for (int dp = 0; dp < D / 16; dp++) {
                uint32_t bf[4];
                ldsm4t(bf, tV + (kk * 16 + (lane & 7) + 8 * ((lane >> 3) & 1)) * LD + dp * 16 + 8 * (lane >> 4));
                mma16816(o[2 * dp], pa[kk], bf[0], bf[1]);
                mma16816(o[2 * dp + 1], pa[kk], bf[2], bf[3]);
            }
        }
        __syncthreads();                                    // the stage may be overwritten by the next iteration's prefetch
    }

    // ---- normalise and store: dst[d, h, iq, b]
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        float l = lrow[rr];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = l > 0.0f ? 1.0f / l : 0.0f;
        const int iq = q0 + warp * 16 + g + 8 * rr;
        if (iq < N) {
            float * dr = reinterpret_cast<float *>(reinterpret_cast<char *>(dst.data) + h * dst.nb[1] + (int64_t)iq * dst.nb[2] + b * dst.nb[3]);
#pragma unroll
            for (int nt = 0; nt < NT; nt++) *reinterpret_cast<float2 *>(dr + nt * 8 + 2 * t4) = make_float2(o[nt][2 * rr] * inv, o[nt][2 * rr + 1] * inv);
        }
    }
}

inline bool al16(const void * p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

// Bytes of scratch flash_attn_prefill wants for the tile-activity flags (0: shape not handled by the tensor-core kernel).
size_t flash_attn_workspace_bytes(const TensorView & q, const TensorView & k, const TensorView * mask) {
    const int D = (int)q.ne[0];
    if (!(D == 64 || D == 128) || q.ne[1] < FA_MIN_ROWS_MMA) return 0;
    const int64_t n_kt = (k.ne[1] + FA_BN - 1) / FA_BN, n_qt = (q.ne[1] + FA_BM - 1) / FA_BM;
    if (n_kt > FA_MAX_TILES) return 0;
    const int64_t mz = mask ? mask->ne[2] * mask->ne[3] : 1;
    return (size_t)(n_kt * n_qt * mz) + 256;
}

// Returns cudaErrorNotSupported when the shape is outside what this kernel handles (caller falls back to the scalar kernel).
cudaError_t flash_attn_prefill(const TensorView & q, const TensorView & k, const TensorView & v, const TensorView * mask, const TensorView & dst,
                               float scale, float softcap, void * ws, size_t ws_bytes, cudaStream_t st) {
    const int D = (int)q.ne[0];
    if (!(D == 64 || D == 128) || D != (int)v.ne[0] || D != (int)k.ne[0] || q.ne[1] < FA_MIN_ROWS_MMA) return cudaErrorNotSupported;
    if (k.type != TY_F16_ || v.type != TY_F16_ || q.type != TY_F32_ || (mask && mask->type != TY_F16_)) return cudaErrorNotSupported;
    if (k.ne[1] != v.ne[1] || k.ne[1] <= 0) return cudaErrorNotSupported;
    // 16-byte alignment of every row the kernel copies in chunks
    if (!al16(q.data) || q.nb[1] % 16 || q.nb[2] % 16 || q.nb[3] % 16) return cudaErrorNotSupported;
    if (!al16(k.data) || k.nb[1] % 16 || k.nb[2] % 16 || k.nb[3] % 16) return cudaErrorNotSupported;
    if (!al16(v.data) || v.nb[1] % 16 || v.nb[2] % 16 || v.nb[3] % 16) return cudaErrorNotSupported;
    if (!((reinterpret_cast<uintptr_t>(dst.data) & 7) == 0) || dst.nb[1] % 8 || dst.nb[2] % 8 || dst.nb[3] % 8) return cudaErrorNotSupported;
    const int N = (int)q.ne[1], n_kv = (int)k.ne[1];
    const int n_kt = (n_kv + FA_BN - 1) / FA_BN, n_qt = (N + FA_BM - 1) / FA_BM;
    if (n_kt > FA_MAX_TILES) return cudaErrorNotSupported;
    if (softcap != 0.0f) scale /= softcap;

    uint8_t * flags = nullptr;
    bool mask_al16 = false;
    if (mask) {
        if (mask->ne[1] < N) return cudaErrorNotSupported;
        const int mz = (int)(mask->ne[2] * mask->ne[3]);
        mask_al16 = al16(mask->data) && mask->nb[1] % 16 == 0 && mask->nb[2] % 16 == 0 && mask->nb[3] % 16 == 0;
        if (ws && ws_bytes >= (size_t)n_kt * n_qt * mz + 256) {
            flags = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
            note_launch();
            cudaError_t e = launch_pdl(fa_tile_flags_kernel, dim3((unsigned)n_kt, (unsigned)n_qt, (unsigned)mz), dim3(64), 0, st, *mask, N, n_kv, n_kt, n_qt, flags);
            if (e != cudaSuccess) return e;
        }
    }
    const dim3 grid((unsigned)n_qt, (unsigned)q.ne[2], (unsigned)q.ne[3]);
    static bool attr_done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(fa_mma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FaSmem<64>::total);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(fa_mma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FaSmem<128>::total);
        if (e != cudaSuccess) return e;
        attr_done[dev] = true;
    }
    note_launch();
    if (D == 64)
        return launch_pdl(fa_mma_kernel<64>, grid, dim3(FA_THREADS), FaSmem<64>::total, st, q, k, v, mask ? *mask : q, mask != nullptr, dst, scale, softcap,
                          (const uint8_t *)flags, n_kt, n_qt, mask_al16);
    return launch_pdl(fa_mma_kernel<128>, grid, dim3(FA_THREADS), FaSmem<128>::total, st, q, k, v, mask ? *mask : q, mask != nullptr, dst, scale, softcap,
                      (const uint8_t *)flags, n_kt, n_qt, mask_al16);
}

}  // namespace ops
}  // namespace qmm
