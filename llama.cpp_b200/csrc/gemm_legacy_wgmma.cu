// gemm_legacy_wgmma.cu -- prefill GEMM for the LEGACY block formats (Q4_0, Q8_0) on the sm_90a warpgroup tensor cores:
//     dst[M, N] = W[M, K] . X[K, N],   N > 8
// (the mmq regime of ggml_compute_forward_mul_mat, ggml-cpu.c:1254-1452, for block_q4_0 / block_q8_0 weights; closest analogue in
// the reference: mul_mat_q with load_tiles_q4_0 / load_tiles_q8_0, ggml-cuda/mmq.cuh:179,463 on mma.sync int8).
//
// What the CPU computes per 32-weight block (ggml_vec_dot_q4_0_q8_0 / ggml_vec_dot_q8_0_q8_0, ggml-cpu/quants.c:225-330):
//     sumf += (fp32(d_w) * fp32(d_a)) * SUM_k (q_w - 8) q_a            (Q8_0: q_w as is)
// with the activations quantised to Q8_0 (quantize_row_q8_0, ggml-quants.c:276-299; d_a stored as fp16).
//
// The K-quant kernel (gemm_tcgen05.cu) keeps integers exact and rescales once per 256 weights; with a scale per 32 weights that
// would mean draining the accumulators eight times as often.  Here the scales are folded INTO the operands instead, without losing bits:
//     a = fp32(d_w) * (q_w - 8)      15 significant bits (Q8_0: 19)          b = fp32(d_a) * q_a       19 significant bits
// are both split exactly into two fp16 numbers (a = a_hi + a_lo, b = b_hi + b_lo: 11 + 11 bits), and
//     a b  ~  a_hi b_hi + a_lo b_hi + a_hi b_lo                               (the dropped a_lo b_lo term is 2^-22 of the product)
// is three wgmma.mma_async instructions accumulating in fp32 registers over the WHOLE K dimension: one write-out per tile.
// The result differs from the CPU's only in fp32 rounding / summation order (tests: <= 1e-3 absolute against the reference's own kernels, measured
// ~1e-6 relative).  Values whose fp16 image would overflow (|a| or |b| >= 65504) are outside this kernel's domain; that is a weight or
// activation of magnitude 65504, which the reference's own fp16 scales cannot represent either.
//
// Structure (one CTA of two warpgroups per 128 x 128 output tile; warpgroup g owns weight rows 64 g .. 64 g + 63):
//   thread (row r, half h) of a warpgroup owns 4 consecutive 32-weight blocks of its row per 256-weight "superstep" (72 bytes of Q4_0 /
//   136 of Q8_0, fetched one superstep ahead with 8-byte loads) and expands ONE block per stage into the hi and lo atoms of a ring of 3
//   stages (canonical K-major SWIZZLE_128B, 64 fp16 per row).  A stage holds, for every row, block j (kk 0..31) and block 4 + j
//   (kk 32..63) of the superstep -- the order of k inside a dot product is free, and this one lets a thread read its weights as one
//   contiguous run.  Thread 0 also starts the bulk copy of the stage's activation atoms (hi | lo, 32 KB, written in exactly this layout
//   by the pre-pass) once both warpgroups have released the stage.  A warpgroup waits for its own rows and the copy, issues its 12
//   m64n128k16 MMAs (4 k-slices x {hi hi, lo hi, hi lo}); while one warpgroup multiplies, the other expands.
// Algorithmic FLOPs per launch: 2 M N K (the tensor pipe executes 3x that).  Roofline: fp16 tensor pipe / 3.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "gemm_layout.cuh"
#include "qmm_formats.cuh"
#include "qmm_kernels.cuh"
#include "tcgen05_ptx.cuh"

namespace qmm {

namespace {

constexpr int LG_MT = 128, LG_NT = 128;
constexpr int LG_THREADS = 256;                          // two warpgroups, 64 weight rows each
constexpr int LG_STAGES = 3;
constexpr int LG_ATOM = 128 * 128;                       // bytes of one atom: 128 rows x 64 fp16
constexpr int LG_STAGE_B = 2 * LG_ATOM;                  // activation atoms of a stage: hi | lo
constexpr int LG_STAGE = 2 * LG_ATOM + LG_STAGE_B;       // A hi | A lo | B hi | B lo
constexpr size_t LG_SMEM = 1024 + (size_t)LG_STAGES * LG_STAGE + 256;

inline int64_t lg_rup(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

template <int T> struct LgFmt;
template <> struct LgFmt<T_Q4_0> { static constexpr int BB = 18, NW = 9; };     // bytes per block; 8-byte words per 4 blocks
template <> struct LgFmt<T_Q8_0> { static constexpr int BB = 34, NW = 17; };

// ------------------------------------------------------------------------------------------------ activation pre-pass
// One warp per (256-element superstep, token); lane l owns elements 8l .. 8l+7 = chunk (l & 3) of Q8_0 block (l >> 2).  Quantises like
// quantize_q8_0_kernel (act_quant.cu: mode 0 = quantize_row_q8_0_ref, mode 1 = the x86 from_float), then writes b = fp32(fp16(d)) * q
// split into hi / lo fp16 as one 16-byte chunk of the stage's hi atom and one of its lo atom.  Tokens >= N are written as zeros.
__global__ void __launch_bounds__(256) quantize_act_legacy_kernel(const float * __restrict__ x, int64_t ldx, int N, int nss, int npad, uint8_t * __restrict__ bimg, int mode) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ss = blockIdx.x, n = blockIdx.y * 8 + warp;
    if (n >= npad) return;
    const int tile = n / LG_NT, nr = n % LG_NT;
    float v[8];
    if (n < N) {
        const float4 a = *reinterpret_cast<const float4 *>(x + n * ldx + 256 * (int64_t)ss + 8 * lane), b = *reinterpret_cast<const float4 *>(x + n * ldx + 256 * (int64_t)ss + 8 * lane + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = 0.0f;
    }
    float amax = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(v[i]));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const float d = __fdiv_rn(amax, 127.0f);
    const float dh = __half2float(__float2half_rn(d));                  // block_q8_0.d is stored as fp16
    const float id = mode == 0 ? (d != 0.0f ? __fdiv_rn(1.0f, d) : 0.0f) : (amax != 0.0f ? __fdiv_rn(127.0f, amax) : 0.0f);
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        float b2[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const float t = __fmul_rn(v[2 * i + e], id);
            const int q = mode == 0 ? (int)roundf(t) : __float2int_rn(t);
            b2[e] = __fmul_rn(dh, (float)q);                            // exact: 11 x 8 bits
        }
        const __half h0 = __float2half_rn(b2[0]), h1 = __float2half_rn(b2[1]);
        const __half l0 = __float2half_rn(__fsub_rn(b2[0], __half2float(h0))), l1 = __float2half_rn(__fsub_rn(b2[1], __half2float(h1)));
        hi[i] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
        lo[i] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    }
    const int bq = lane >> 2, cq = lane & 3;                            // block inside the superstep, 8-element chunk inside the block
    const int stage = bq & 3, chunk = 4 * (bq >> 2) + cq;               // stage j holds blocks j and 4 + j
    uint8_t * img = bimg + (((int64_t)tile * nss + ss) * 4 + stage) * LG_STAGE_B;
    const int off = gl::atom_off(nr, 8 * chunk);
    *reinterpret_cast<uint4 *>(img + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4 *>(img + LG_ATOM + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// ------------------------------------------------------------------------------------------------ weight expansion
// 32-bit word at a compile-time byte offset (a multiple of 2) inside a buffer of 32-bit words held in registers
template <int OFF, int NWORDS>
__device__ __forceinline__ uint32_t word_at(const uint32_t (&w)[NWORDS]) {
    static_assert(OFF % 2 == 0 && OFF / 4 < NWORDS, "word_at");
    if constexpr (OFF % 4 == 0) return w[OFF / 4];
    else {
        static_assert(OFF / 4 + 1 < NWORDS, "word_at");
        return __funnelshift_r(w[OFF / 4], w[OFF / 4 + 1], 16);
    }
}
template <int OFF, int NWORDS>
__device__ __forceinline__ __half2 scale_at(const uint32_t (&w)[NWORDS]) {       // the fp16 block scale at byte OFF, in both halves
    const uint32_t v = OFF % 4 == 0 ? (w[OFF / 4] & 0xFFFFu) : (w[OFF / 4] >> 16);
    const uint32_t vv = v | (v << 16);
    return *reinterpret_cast<const __half2 *>(&vv);
}
__device__ __forceinline__ __half2 u32_as_h2(uint32_t v) { return *reinterpret_cast<const __half2 *>(&v); }
__device__ __forceinline__ uint32_t h2_bits(__half2 v) { return *reinterpret_cast<const uint32_t *>(&v); }

// two values v (small exact integers in fp16) times the block scale -> hi = fp16(v d), lo = v d - hi (exact: one rounding of an exactly
// representable result; below fp16's subnormal grid the tail is dropped -- an absolute error under 2^-25 |activation|)
__device__ __forceinline__ void split2(__half2 v, __half2 d2, uint32_t & hi, uint32_t & lo) {
    const __half2 h = __hmul2(v, d2);
    const __half2 l = __hfma2(v, d2, __hneg2(h));
    hi = h2_bits(h); lo = h2_bits(l);
}
// bytes n0..n3 of `x` (each < 256, here < 64 or biased int8) -> half2 (1024 + n0, 1024 + n1) and (1024 + n2, 1024 + n3): 0x6400 | n
__device__ __forceinline__ __half2 pair01(uint32_t x) { return u32_as_h2(__byte_perm(x, 0x64646464u, 0x5140)); }
__device__ __forceinline__ __half2 pair23(uint32_t x) { return u32_as_h2(__byte_perm(x, 0x64646464u, 0x7362)); }

// Expand 8 consecutive elements given as two 4-byte groups of codes (bias: the fp16 value to subtract, 1024 + 8 or 1024 + 128) and
// store them as chunk `chunk` of row r in the hi and the lo atom.
__device__ __forceinline__ void put_chunk(uint32_t c0, uint32_t c1, __half2 bias, __half2 d2, int r, int chunk, uint8_t * a_hi, uint8_t * a_lo) {
    uint32_t hi[4], lo[4];
    split2(__hsub2(pair01(c0), bias), d2, hi[0], lo[0]);
    split2(__hsub2(pair23(c0), bias), d2, hi[1], lo[1]);
    split2(__hsub2(pair01(c1), bias), d2, hi[2], lo[2]);
    split2(__hsub2(pair23(c1), bias), d2, hi[3], lo[3]);
    const int off = (r >> 3) * 1024 + (r & 7) * 128 + ((chunk ^ (r & 7)) << 4);          // gl::atom_off(r, 8 * chunk)
    *reinterpret_cast<uint4 *>(a_hi + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4 *>(a_lo + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// block J (0..3) of the thread's four: natural element order, kk = 32 h + e
template <int T, int J, int NWORDS>
__device__ __forceinline__ void expand_block(const uint32_t (&w)[NWORDS], int r, int h, uint8_t * a_hi, uint8_t * a_lo) {
    constexpr int BB = LgFmt<T>::BB, O = J * BB;
    const __half2 d2 = scale_at<O, NWORDS>(w);
    if constexpr (T == T_Q4_0) {
        // block_q4_0 (ggml-common.h:194-199): element e < 16 is the low nibble of qs[e], element 16 + e the high nibble; value d (q - 8)
        const uint32_t q0 = word_at<O + 2, NWORDS>(w), q1 = word_at<O + 6, NWORDS>(w), q2 = word_at<O + 10, NWORDS>(w), q3 = word_at<O + 14, NWORDS>(w);
        const __half2 bias = u32_as_h2(0x64086408u);                                    // 1032 = 1024 + 8
        put_chunk(q0 & 0x0F0F0F0Fu, q1 & 0x0F0F0F0Fu, bias, d2, r, 4 * h + 0, a_hi, a_lo);
        put_chunk(q2 & 0x0F0F0F0Fu, q3 & 0x0F0F0F0Fu, bias, d2, r, 4 * h + 1, a_hi, a_lo);
        put_chunk((q0 >> 4) & 0x0F0F0F0Fu, (q1 >> 4) & 0x0F0F0F0Fu, bias, d2, r, 4 * h + 2, a_hi, a_lo);
        put_chunk((q2 >> 4) & 0x0F0F0F0Fu, (q3 >> 4) & 0x0F0F0F0Fu, bias, d2, r, 4 * h + 3, a_hi, a_lo);
    } else {
        // block_q8_0 (ggml-common.h:224-228): 32 int8; code = q + 128 (0..255), value d q
        const __half2 bias = u32_as_h2(0x64806480u);                                    // 1152 = 1024 + 128
#pragma unroll
        for (int c = 0; c < 4; c++) {
            uint32_t a, b;
            if (c == 0) { a = word_at<O + 2, NWORDS>(w); b = word_at<O + 6, NWORDS>(w); }
            else if (c == 1) { a = word_at<O + 10, NWORDS>(w); b = word_at<O + 14, NWORDS>(w); }
            else if (c == 2) { a = word_at<O + 18, NWORDS>(w); b = word_at<O + 22, NWORDS>(w); }
            else { a = word_at<O + 26, NWORDS>(w); b = word_at<O + 30, NWORDS>(w); }
            put_chunk(a ^ 0x80808080u, b ^ 0x80808080u, bias, d2, r, 4 * h + c, a_hi, a_lo);
        }
    }
}

struct LegacyKArgs {
    const uint8_t * w; int64_t row_stride; int M, K, N;
    const uint8_t * bimg;
    float * dst; int64_t ldd;
};

template <int T>
__global__ void __launch_bounds__(LG_THREADS, 1) gemm_legacy_wgmma_kernel(const LegacyKArgs p) {
    using F = LgFmt<T>;
    constexpr int NWORDS = 2 * F::NW + 2;                    // (+ 2: word_at may name the word after the last one it needs)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t * smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem + (size_t)LG_STAGES * LG_STAGE);
    uint64_t * bar_full = bars;                              // [LG_STAGES] the activation copy of the stage landed
    uint64_t * bar_empty = bars + LG_STAGES;                 // [LG_STAGES] both warpgroups' MMAs have read the stage (256 arrivals)

    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;
    const int m0 = blockIdx.x * LG_MT, tile = blockIdx.y;
    const int nss = p.K >> 8;

    if (tid == 0) {
        for (int i = 0; i < LG_STAGES; i++) { g_mbar_init(bar_full + i, 1); g_mbar_init(bar_empty + i, LG_THREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();

    const int r = 64 * wg + (t & 63), h = t >> 6;
    const bool row_ok = m0 + r < p.M;
    const uint8_t * wsrc = p.w + (int64_t)(m0 + r) * p.row_stride + (int64_t)h * (4 * F::BB);
    const uint32_t a_off = (uint32_t)wg * 64 * 128;          // this warpgroup's 64 rows inside an A atom (8 row groups of 1024 B)
    uint32_t cur[NWORDS], nxt[NWORDS];
#pragma unroll
    for (int i = 0; i < NWORDS; i++) { cur[i] = 0u; nxt[i] = 0u; }
    auto fetch = [&](uint32_t (&dst)[NWORDS], int ss) {
        if (row_ok) {
            const uint2 * src = reinterpret_cast<const uint2 *>(wsrc + (int64_t)ss * (8 * F::BB));
#pragma unroll
            for (int i = 0; i < F::NW; i++) { const uint2 w2 = __ldg(src + i); dst[2 * i] = w2.x; dst[2 * i + 1] = w2.y; }
        }
    };
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; i++) acc[i] = 0.0f;
    fetch(nxt, 0);
    for (int ss = 0; ss < nss; ss++) {
#pragma unroll
        for (int i = 0; i < NWORDS; i++) cur[i] = nxt[i];
        if (ss + 1 < nss) fetch(nxt, ss + 1);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t it = (uint32_t)ss * 4u + (uint32_t)j;
            const uint32_t s = it % LG_STAGES, ph = (it / LG_STAGES) & 1u;
            uint8_t * st = smem + (size_t)s * LG_STAGE;
            if (tid == 0) {
                g_mbar_wait(bar_empty + s, ph ^ 1u);
                g_mbar_expect_tx(bar_full + s, (uint32_t)LG_STAGE_B);
                g_bulk_g2s(st + 2 * LG_ATOM, p.bimg + (((int64_t)tile * nss + ss) * 4 + j) * LG_STAGE_B, (uint32_t)LG_STAGE_B, bar_full + s);
            }
            if (j == 0) expand_block<T, 0, NWORDS>(cur, r, h, st, st + LG_ATOM);
            else if (j == 1) expand_block<T, 1, NWORDS>(cur, r, h, st, st + LG_ATOM);
            else if (j == 2) expand_block<T, 2, NWORDS>(cur, r, h, st, st + LG_ATOM);
            else expand_block<T, 3, NWORDS>(cur, r, h, st, st + LG_ATOM);
            fence_proxy_async();                            // generic-proxy smem writes -> visible to the tensor core (async proxy)
            wg_bar_sync(wg);
            g_mbar_wait(bar_full + s, ph);
            const uint32_t a_hi = s32(st) + a_off, a_lo = a_hi + LG_ATOM, b_hi = s32(st) + 2 * LG_ATOM, b_lo = b_hi + LG_ATOM;
            acc_fence(acc);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 4; ks++) {
                const uint64_t dah = make_desc_sw128(a_hi + ks * 32), dal = make_desc_sw128(a_lo + ks * 32);
                const uint64_t dbh = make_desc_sw128(b_hi + ks * 32), dbl = make_desc_sw128(b_lo + ks * 32);
                wgmma_m64n128k16_f16(acc, dah, dbh, (it | (uint32_t)ks) != 0 ? 1u : 0u);
                wgmma_m64n128k16_f16(acc, dal, dbh, 1u);
                wgmma_m64n128k16_f16(acc, dah, dbl, 1u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            acc_fence(acc);
            g_mbar_arrive(bar_empty + s);                   // this thread's reads of the stage are done
        }
    }

    // write out: dst[n*ldd + m]; thread t holds rows er, er + 8 and columns 8 i + 2 (t % 4) (+ 1) of its warpgroup's 64 x 128 tile
    const int c4 = t & 3, er = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);
    const bool ok_lo = m0 + er < p.M, ok_hi = m0 + er + 8 < p.M;
#pragma unroll
    for (int i = 0; i < 16; i++) {
#pragma unroll
        for (int c = 0; c < 2; c++) {
            const int n = tile * LG_NT + 8 * i + 2 * c4 + c;
            if (n >= p.N) continue;
            if (ok_lo) p.dst[(int64_t)n * p.ldd + m0 + er] = acc[4 * i + c];
            if (ok_hi) p.dst[(int64_t)n * p.ldd + m0 + er + 8] = acc[4 * i + 2 + c];
        }
    }
}

}  // namespace

size_t gemm_legacy_workspace_bytes(int type, int64_t M, int64_t N, int64_t K) {
    (void)M;
    if (!(type == T_Q4_0 || type == T_Q8_0) || K % 256 || N <= 0) return 0;
    return (size_t)(lg_rup(N, LG_NT) / LG_NT * (K / 64) * LG_STAGE_B + 1024);
}

cudaError_t launch_gemm_legacy(int type, const GemmArgs & a, cudaStream_t st) {
    if (!(type == T_Q4_0 || type == T_Q8_0) || a.K % 256 || a.N <= 0 || a.M <= 0) return cudaErrorNotSupported;
    // a thread reads its 72 / 136 weight bytes per superstep with 8-byte loads; the pre-pass reads float4
    if ((reinterpret_cast<uintptr_t>(a.w) & 7) || (a.row_stride & 7)) return cudaErrorMisalignedAddress;
    if ((reinterpret_cast<uintptr_t>(a.x) & 15) || (a.ldx & 3)) return cudaErrorMisalignedAddress;
    if (a.workspace_bytes < gemm_legacy_workspace_bytes(type, a.M, a.N, a.K)) return cudaErrorInvalidValue;
    const int npad = (int)lg_rup(a.N, LG_NT), nss = a.K / 256, ntiles = npad / LG_NT;
    uint8_t * bimg = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(a.workspace) + 255) & ~uintptr_t(255));
    if (!a.reuse_operands) {
        note_launch();
        quantize_act_legacy_kernel<<<dim3((unsigned)nss, (unsigned)(npad / 8)), 256, 0, st>>>(a.x, a.ldx, a.N, nss, npad, bimg, get_q8_0_mode());
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    static bool attr_done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(gemm_legacy_wgmma_kernel<T_Q4_0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LG_SMEM);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(gemm_legacy_wgmma_kernel<T_Q8_0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LG_SMEM);
        if (e != cudaSuccess) return e;
        attr_done[dev] = true;
    }
    const LegacyKArgs k{a.w, a.row_stride, a.M, a.K, a.N, bimg, a.dst, a.ldd};
    const dim3 grid((unsigned)((a.M + LG_MT - 1) / LG_MT), (unsigned)ntiles);
    note_launch();
    if (type == T_Q4_0) gemm_legacy_wgmma_kernel<T_Q4_0><<<grid, LG_THREADS, LG_SMEM, st>>>(k);
    else gemm_legacy_wgmma_kernel<T_Q8_0><<<grid, LG_THREADS, LG_SMEM, st>>>(k);
    return cudaGetLastError();
}

}  // namespace qmm
