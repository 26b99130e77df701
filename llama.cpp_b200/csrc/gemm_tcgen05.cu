// gemm_tcgen05.cu -- prefill GEMM for K-quant weights on the sm_90a warpgroup tensor cores (wgmma; the file name is historical):
//     dst[M, N] = W[M, K] . X[K, N],   N > 8      (the mmq regime of ggml_compute_forward_mul_mat, ggml-cpu.c:1254-1452;
//                                                  closest analogue in the reference: mul_mat_q, ggml-cuda/mmq.cuh:946-1231)
//
// Exact-integer formulation (what lets the result match the CPU to fp32 rounding instead of fp16/bf16 rounding):
//   the CPU computes, per 256-weight block kb,   d_w d_a * SUM_j sc_j SUM_k q_w q_a  -  dmin_w d_a * SUM_j m_j bsum_j
//   (ggml-cpu/quants.c:743-767).  Both integer sums are produced on the tensor cores from operands that are small
//   integers, exactly representable in fp16:
//       A  = sc_j * q_w      (<= 63*15 for Q4_K, 63*31 for Q5_K)      B  = q_a (the CPU-identical Q8_K integers)
//       A' = m_j             (6 bit)                                    B' = bsum_j split into (even part, low bit)
//   wgmma.mma_async accumulates them in fp32 registers: exact while a block's partial sums stay below 2^24, which a saturated
//   block exceeds (main sum up to 256*63*15*127 ~ 3.1e7 for Q4_K, 6.3e7 Q5_K, 1.3e8 Q6_K); there the fp32 rounding keeps the
//   result within 6e-6 * sum |w x| (worst 0.21 of that measured on an H100 SXM at 700 W, DESIGN.md 3).  After every K block the block's integer sums are
//   combined in registers with the block's fp16/fp32 scales:
//       acc += (d_w d_a) * main - (dmin_w d_a) * mins
//   i.e. the same per-block fp32 combine the CPU does (the mins term is added first).
//
// Structure: one CTA of two warpgroups per 128 x 128 output tile; warpgroup g owns weight rows 64 g .. 64 g + 63 of the tile.
// Per K block, thread 0 starts one bulk copy of the activation image (written in the canonical 128B-swizzled K-major layout by
// quantize_act_gemm_kernel) while every warpgroup de-quantises ITS rows of the weight block into the same layout; a warpgroup then
// waits only for its own rows and the activation copy, issues its m64n128k16 MMAs and rescales.  The two warpgroups meet only at
// the activation buffer (an mbarrier that counts both out before the next copy), so one de-quantises while the other multiplies.
//
// Algorithmic FLOPs per launch: 2 M N K.  Roofline: fp16 tensor pipe.
#include <cuda_fp16.h>
#include <stdlib.h>

#include "gemm_layout.cuh"
#include "qmm_formats.cuh"
#include "qmm_kernels.cuh"
#include "qmm_moe.cuh"
#include "tcgen05_ptx.cuh"

namespace qmm {

constexpr int GEMM_NT      = 128;                 // token columns per CTA tile
constexpr int GEMM_MT      = 128;                 // weight rows per CTA tile
constexpr int GEMM_THREADS = 256;                 // two warpgroups, 64 weight rows each

static inline int64_t rup(int64_t v, int64_t a) { return (v + a - 1) / a * a; }

// workspace: [B images: ntiles x nkb x bimg_block_bytes] [d_a: nkb x Npad floats]
size_t gemm_workspace_bytes(int type, int64_t M, int64_t N, int64_t K) {
    if (type == T_Q4_0 || type == T_Q8_0) return gemm_legacy_workspace_bytes(type, M, N, K);
    if (!(type == T_Q4_K || type == T_Q5_K || type == T_Q6_K) || K % 256 || N <= 0) return 0;
    const int64_t nkb = K / 256;
    const int64_t npad = rup(N, GEMM_NT);
    return (size_t)(npad / GEMM_NT * nkb * gl::bimg_block_bytes(GEMM_NT) + nkb * npad * 4 + 1024);
}

// ------------------------------------------------------------------------------------------------ activation pre-pass
// One CTA of 256 threads per (K block, token).  Quantises exactly like quantize_q8_K_kernel (act_quant.cu) and writes
// the fp16-integer operand images described in gemm_layout.cuh.  Tokens n >= N (tile padding) are written as zeros.
__device__ __forceinline__ unsigned long long g_warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long t = __shfl_xor_sync(0xffffffffu, v, o); v = t > v ? t : v; }
    return v;
}

// One WARP per (K block, token), 8 tokens per CTA.  Lane l owns elements 8l .. 8l+7 of the block: they are one 16-byte chunk
// of one atom row (chunk l % 8 of atom l / 8; the k permutation stays inside a chunk), so the operand image is written with
// one 16-byte store per lane.
__global__ void __launch_bounds__(256) quantize_act_gemm_kernel(const float * __restrict__ x, int64_t ldx, int N, int nkb, int npad,
                                                                uint8_t * __restrict__ bimg, float * __restrict__ da, int NT, const int * __restrict__ col_src) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int kb = blockIdx.x, n = blockIdx.y * 8 + warp;
    if (n >= npad) return;
    const int sn = col_src ? col_src[n] : (n < N ? n : -1);            // source column of image column n (grouped launches gather)
    const int tile = n / NT, nr = n % NT;
    uint8_t * img = bimg + ((int64_t)tile * nkb + kb) * gl::bimg_block_bytes(NT);
    float v[8];
    if (sn >= 0) {
        const float4 a = *reinterpret_cast<const float4 *>(x + sn * ldx + 256 * (int64_t)kb + 8 * lane), b = *reinterpret_cast<const float4 *>(x + sn * ldx + 256 * (int64_t)kb + 8 * lane + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = 0.0f;
    }
    // quantize_row_q8_K_ref (ggml-quants.c:2768-2805): the FIRST element of largest magnitude decides scale and sign
    unsigned mloc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { const unsigned a = (v[i] == v[i]) ? (__float_as_uint(v[i]) & 0x7fffffffu) : 0u; mloc = a > mloc ? a : mloc; }
    unsigned mall = mloc;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned t = __shfl_xor_sync(0xffffffffu, mall, o); mall = t > mall ? t : mall; }
    const unsigned holders = __ballot_sync(0xffffffffu, mloc == mall);
    const int wl = __ffs((int)holders) - 1;
    float mine = 0.0f;
#pragma unroll
    for (int i = 7; i >= 0; i--) mine = ((__float_as_uint(v[i]) & 0x7fffffffu) == mall && v[i] == v[i]) ? v[i] : mine;
    const float maxv = __shfl_sync(0xffffffffu, mine, wl);
    const float amax = __uint_as_float(mall);
    int q[8];
    float d = 0.0f;
    if (amax > 0.0f) {
        const float iscale = __fdiv_rn(-127.0f, maxv);
#pragma unroll
        for (int i = 0; i < 8; i++) { const int t = __float2int_rn(__fmul_rn(iscale, v[i])); q[i] = t > 127 ? 127 : t; }
        d = __fdiv_rn(1.0f, iscale);
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) q[i] = 0;
    }
    // chunk of 8 fp16 integers: slot kperm(i) holds element i (swap of bits 0 and 1)
    __half2 h01 = __halves2half2(__int2half_rn(q[0]), __int2half_rn(q[2]));   // slots 0,1 <- elements 0,2
    __half2 h23 = __halves2half2(__int2half_rn(q[1]), __int2half_rn(q[3]));   // slots 2,3 <- elements 1,3
    __half2 h45 = __halves2half2(__int2half_rn(q[4]), __int2half_rn(q[6]));
    __half2 h67 = __halves2half2(__int2half_rn(q[5]), __int2half_rn(q[7]));
    uint4 pk;
    pk.x = *reinterpret_cast<uint32_t *>(&h01); pk.y = *reinterpret_cast<uint32_t *>(&h23);
    pk.z = *reinterpret_cast<uint32_t *>(&h45); pk.w = *reinterpret_cast<uint32_t *>(&h67);
    *reinterpret_cast<uint4 *>(img + (lane >> 3) * gl::atom_bytes(NT) + gl::atom_off(nr, 8 * (lane & 7))) = pk;
    // sums of 32 (4 lanes), split into even part and low bit for the mins operand
    int s = q[0] + q[1] + q[2] + q[3] + q[4] + q[5] + q[6] + q[7];
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    const int bs32 = __shfl_sync(0xffffffffu, s, 4 * (lane & 7));
    if (lane < 16) {
        const int val = lane < 8 ? (bs32 & ~1) : (bs32 & 1);
        *reinterpret_cast<__half *>(img + gl::ATOMS_PER_BLOCK * gl::atom_bytes(NT) + gl::atom_off(nr, lane)) = __int2half_rn(val);
    }
    if (lane == 0) da[(int64_t)kb * npad + n] = d;
}

// ------------------------------------------------------------------------------------------------ weight de-quantiser
// Thread (row r, half h) expands groups 2h, 2h+1 (64 weights each) of its row's block into atoms 2h, 2h+1.
__device__ __forceinline__ uint32_t h2_as_u32(__half2 v) { return *reinterpret_cast<uint32_t *>(&v); }
__device__ __forceinline__ uint32_t cvt2(uint32_t nib2, __half2 sc, __half2 bias) {      // nib2: two 4/5-bit codes at bits 0.. and 16..
    const uint32_t m = nib2 | 0x64006400u;                                                // 1024 + q in both halves
    return h2_as_u32(__hfma2(*reinterpret_cast<const __half2 *>(&m), sc, bias));          // (1024+q)*sc - 1024*sc = sc*q, exact
}

template <int T>
__device__ __forceinline__ void dequant_block_to_smem(const uint8_t * __restrict__ blk, bool valid, int r, int h, uint8_t * sA, uint8_t * sAmin) {
    uint4 hdr = make_uint4(0, 0, 0, 0);
    if (valid) hdr = __ldg(reinterpret_cast<const uint4 *>(blk));
    constexpr int QS_OFF = (T == T_Q4_K) ? 16 : 48;
    uint4 qhA = make_uint4(0, 0, 0, 0), qhB = make_uint4(0, 0, 0, 0);
    if (T == T_Q5_K && valid) { qhA = __ldg(reinterpret_cast<const uint4 *>(blk + 16)); qhB = __ldg(reinterpret_cast<const uint4 *>(blk + 32)); }
#pragma unroll
    for (int gg = 0; gg < 2; gg++) {
        const int g = 2 * h + gg;
        int sc0, mn0, sc1, mn1;
        k4_scale_min(2 * g, hdr.y, hdr.z, hdr.w, sc0, mn0);
        k4_scale_min(2 * g + 1, hdr.y, hdr.z, hdr.w, sc1, mn1);
        const __half2 sl = __half2half2(__int2half_rn(sc0)), bl = __half2half2(__int2half_rn(-1024 * sc0));
        const __half2 sh = __half2half2(__int2half_rn(sc1)), bh = __half2half2(__int2half_rn(-1024 * sc1));
        uint4 U[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
        if (valid) { U[0] = __ldg(reinterpret_cast<const uint4 *>(blk + QS_OFF + 32 * g)); U[1] = __ldg(reinterpret_cast<const uint4 *>(blk + QS_OFF + 32 * g + 16)); }
        uint8_t * atom = sA + g * gl::atom_bytes(GEMM_MT) + (r >> 3) * 1024 + (r & 7) * 128;
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const uint32_t w[4] = {U[u].x, U[u].y, U[u].z, U[u].w};
            const uint4 QH = u == 0 ? qhA : qhB;
            const uint32_t hq[4] = {QH.x, QH.y, QH.z, QH.w};
#pragma unroll
            for (int wp = 0; wp < 2; wp++) {
                uint32_t lo[4], hi[4];
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    const uint32_t ww = w[2 * wp + i];
                    uint32_t l0 = ww & 0x000F000Fu, l1 = (ww >> 8) & 0x000F000Fu, h0 = (ww >> 4) & 0x000F000Fu, h1 = (ww >> 12) & 0x000F000Fu;
                    if (T == T_Q5_K) {      // 5th bit: bit 2g of qh[l] for low-nibble elements, bit 2g+1 for high-nibble elements
                        const uint32_t hh = hq[2 * wp + i];
                        l0 |= ((hh >> (2 * g)) & 0x00010001u) << 4;      l1 |= ((hh >> (2 * g + 8)) & 0x00010001u) << 4;
                        h0 |= ((hh >> (2 * g + 1)) & 0x00010001u) << 4;  h1 |= ((hh >> (2 * g + 9)) & 0x00010001u) << 4;
                    }
                    lo[2 * i] = cvt2(l0, sl, bl); lo[2 * i + 1] = cvt2(l1, sl, bl);
                    hi[2 * i] = cvt2(h0, sh, bh); hi[2 * i + 1] = cvt2(h1, sh, bh);
                }
                const int cl = 2 * u + wp, ch = 4 + 2 * u + wp;
                *reinterpret_cast<uint4 *>(atom + ((cl ^ (r & 7)) << 4)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                *reinterpret_cast<uint4 *>(atom + ((ch ^ (r & 7)) << 4)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            }
        }
    }
    if (h == 0) {                                            // mins atom: kk 0..7 = kk 8..15 = m_j
        uint32_t mh[4];
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
            int sa, ma, sb, mb;
            k4_scale_min(2 * jj, hdr.y, hdr.z, hdr.w, sa, ma);
            k4_scale_min(2 * jj + 1, hdr.y, hdr.z, hdr.w, sb, mb);
            mh[jj] = h2_as_u32(__halves2half2(__int2half_rn(ma), __int2half_rn(mb)));
        }
        uint8_t * arow = sAmin + (r >> 3) * 1024 + (r & 7) * 128;
        const uint4 mv = make_uint4(mh[0], mh[1], mh[2], mh[3]);
        *reinterpret_cast<uint4 *>(arow + ((0 ^ (r & 7)) << 4)) = mv;
        *reinterpret_cast<uint4 *>(arow + ((1 ^ (r & 7)) << 4)) = mv;
    }
}

// Q6_K: x = d * sc * (q - 32), sc int8, q 6 bit.  |sc (q-32)| reaches 4096 > 2048, so odd products would not be exact in
// fp16.  Split sc = sc_even + sc_lsb (sc_lsb = sc & 1): A1 = sc_even (q-32) is even and <= 4096 (exact), A2 = sc_lsb (q-32)
// is tiny; both tiles are multiplied with the same B and accumulated into the same registers (32 MMAs per block, no mins).
// Thread (row r, half h) expands weights 128h .. 128h+127 into atoms 2h (quarters 0,1) and 2h+1 (quarters 2,3).
__device__ __forceinline__ uint32_t ldg4_a2(const uint8_t * p) {       // 4 bytes from a 2-byte aligned global address
    const uint32_t * w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(3));
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 2) * 8;
    return __funnelshift_r(__ldg(w), __ldg(w + 1), sh);
}

__device__ __forceinline__ void dequant_q6_block_to_smem(const uint8_t * __restrict__ blk, bool valid, int r, int h, uint8_t * sA1, uint8_t * sA2) {
    uint32_t ql[16], qh[8], scw[2];
#pragma unroll
    for (int i = 0; i < 16; i++) ql[i] = valid ? ldg4_a2(blk + 64 * h + 4 * i) : 0u;
#pragma unroll
    for (int i = 0; i < 8; i++) qh[i] = valid ? ldg4_a2(blk + 128 + 32 * h + 4 * i) : 0u;
#pragma unroll
    for (int i = 0; i < 2; i++) scw[i] = valid ? ldg4_a2(blk + 192 + 8 * h + 4 * i) : 0u;
    const __half2 k1056 = __half2half2(__int2half_rn(1056));
#pragma unroll
    for (int qtr = 0; qtr < 4; qtr++) {
        // scales of this quarter: index 2*qtr (l < 16) and 2*qtr + 1 (l >= 16) within the half
        __half2 se[2], so[2];
#pragma unroll
        for (int hl = 0; hl < 2; hl++) {
            const int si = 2 * qtr + hl;
            const int sc = (int)(int8_t)((scw[si >> 2] >> (8 * (si & 3))) & 0xFFu);
            const int lsb = sc & 1;
            se[hl] = __half2half2(__int2half_rn(sc - lsb));
            so[hl] = __half2half2(__int2half_rn(lsb));
        }
        const int atom = 2 * h + (qtr >> 1);
        const int kk0 = 32 * (qtr & 1);                   // k offset of this quarter inside the atom
        uint8_t * row1 = sA1 + atom * gl::atom_bytes(GEMM_MT) + (r >> 3) * 1024 + (r & 7) * 128;
        uint8_t * row2 = sA2 + atom * gl::atom_bytes(GEMM_MT) + (r >> 3) * 1024 + (r & 7) * 128;
#pragma unroll
        for (int cc = 0; cc < 4; cc++) {                  // chunk of 8 weights: l = 8cc .. 8cc+7  (two ql words)
            uint32_t o1[4], o2[4];
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int wi = 2 * cc + i;                // word index: l = 4wi .. 4wi+3
                const uint32_t lw = ql[(qtr & 1) * 8 + wi];
                const uint32_t hw = qh[wi];
                const uint32_t n02 = ((qtr < 2 ? lw : (lw >> 4)) & 0x000F000Fu) | (((hw >> (2 * qtr)) & 0x00030003u) << 4);
                const uint32_t n13 = ((qtr < 2 ? (lw >> 8) : (lw >> 12)) & 0x000F000Fu) | (((hw >> (2 * qtr + 8)) & 0x00030003u) << 4);
                const uint32_t m02 = n02 | 0x64006400u, m13 = n13 | 0x64006400u;          // 1024 + code
                const __half2 v02 = __hsub2(*reinterpret_cast<const __half2 *>(&m02), k1056);   // code - 32, exact
                const __half2 v13 = __hsub2(*reinterpret_cast<const __half2 *>(&m13), k1056);
                const int hl = wi >> 2;                   // l >= 16 ?
                o1[2 * i] = h2_as_u32(__hmul2(v02, se[hl])); o1[2 * i + 1] = h2_as_u32(__hmul2(v13, se[hl]));
                o2[2 * i] = h2_as_u32(__hmul2(v02, so[hl])); o2[2 * i + 1] = h2_as_u32(__hmul2(v13, so[hl]));
            }
            const int chunk = (kk0 >> 3) + cc;
            *reinterpret_cast<uint4 *>(row1 + ((chunk ^ (r & 7)) << 4)) = make_uint4(o1[0], o1[1], o1[2], o1[3]);
            *reinterpret_cast<uint4 *>(row2 + ((chunk ^ (r & 7)) << 4)) = make_uint4(o2[0], o2[1], o2[2], o2[3]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ main kernel
struct GemmKArgs {
    const uint8_t * w; int64_t row_stride; int M, K, N, npad;
    const uint8_t * bimg; const float * da;
    float * dst; int64_t ldd;
    // grouped (MUL_MAT_ID) launches: column tile t multiplies expert tile_expert[t] (< 0: the tile does not exist) and image column n
    // is written to dst column col_dst[n] (< 0: padding).  nullptr: a plain GEMM.
    const int * tile_expert; const int * col_dst; int64_t expert_stride;
};
template <bool GROUPED> __device__ __forceinline__ int gemm_dst_col_t(const GemmKArgs & p, int n) { if constexpr (GROUPED) return p.col_dst[n]; else return n < p.N ? n : -1; }

template <int T> struct KqCfg {
    static constexpr bool IS_Q6 = (T == T_Q6_K);
    static constexpr int ATOM_A = GEMM_MT * 128, ATOM_B = GEMM_NT * 128;
    static constexpr int A_BYTES = (IS_Q6 ? 8 : 5) * ATOM_A;      // 4 atoms + (Q6_K: 4 atoms of the odd-scale part; else 1 of mins)
    static constexpr int B_BYTES = 5 * ATOM_B;                     // exactly one B image block (gemm_layout.cuh)
    static constexpr size_t SMEM = 1024 + (size_t)A_BYTES + B_BYTES + 64;
};

// acc += scale(row) * d_a(col) * v over the thread's fragment (see wgmma_m64n128k16_f16 for which element each register holds)
__device__ __forceinline__ void kq_combine(float (&acc)[64], const float (&v)[64], float s_lo, float s_hi, const float * __restrict__ dap, int c4) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const float2 da = __ldg(reinterpret_cast<const float2 *>(dap + 8 * i + 2 * c4));
        acc[4 * i + 0] += (s_lo * da.x) * v[4 * i + 0];
        acc[4 * i + 1] += (s_lo * da.y) * v[4 * i + 1];
        acc[4 * i + 2] += (s_hi * da.x) * v[4 * i + 2];
        acc[4 * i + 3] += (s_hi * da.y) * v[4 * i + 3];
    }
}

template <int T, bool GROUPED>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_q_wgmma_kernel(const GemmKArgs p) {
    // The grouped (MUL_MAT_ID) form is its own instantiation, so that the plain GEMM carries no expert lookup.
    const uint8_t * wbase = p.w;
    if constexpr (GROUPED) {                               // this column tile's expert (uniform per CTA)
        const int e = p.tile_expert[blockIdx.y];
        if (e < 0) return;
        wbase += (int64_t)e * p.expert_stride;
    }
    using C = KqCfg<T>;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t * smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t * sA = smem;                                   // 4 atoms
    uint8_t * sAx = sA + 4 * C::ATOM_A;                    // Q4_K/Q5_K: 1 atom of mins; Q6_K: 4 atoms of the odd-scale part
    uint8_t * sB = sA + C::A_BYTES;
    uint64_t * bar_full = reinterpret_cast<uint64_t *>(sB + C::B_BYTES);    // bulk copy of the B block landed
    uint64_t * bar_empty = bar_full + 1;                   // both warpgroups' MMAs have read it (256 arrivals)

    const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127;
    const int m0 = blockIdx.x * GEMM_MT, tile = blockIdx.y;
    const int nkb = p.K >> 8;
    constexpr int BB = Fmt<T>::BB;

    if (tid == 0) { g_mbar_init(bar_full, 1); g_mbar_init(bar_empty, GEMM_THREADS); asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
    __syncthreads();

    // de-quantiser ownership: thread (row r, half h) expands weights 128 h .. 128 h + 127 of row r (only rows of its own warpgroup)
    const int r = 64 * wg + (t & 63), h = t >> 6;
    const bool row_ok = m0 + r < p.M;
    const uint8_t * wrow = wbase + (int64_t)(m0 + r) * p.row_stride;
    // accumulator ownership: rows er, er + 8 of the tile, columns 8 i + 2 c4 (+ 1)
    const int c4 = t & 3, er = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);
    const bool ok_lo = m0 + er < p.M, ok_hi = m0 + er + 8 < p.M;
    const uint8_t * ew_lo = wbase + (int64_t)(m0 + er) * p.row_stride, * ew_hi = ew_lo + 8 * p.row_stride;
    const uint32_t a_off = (uint32_t)wg * 64 * 128;        // this warpgroup's 64 rows inside an A atom (8 row groups of 1024 B)

    float acc[64], v[64];
#pragma unroll
    for (int i = 0; i < 64; i++) { acc[i] = 0.0f; v[i] = 0.0f; }
    const int64_t bblk = gl::bimg_block_bytes(GEMM_NT);

    for (int kb = 0; kb < nkb; kb++) {
        const uint32_t par = (uint32_t)(kb & 1);
        // (1) B image of this block: one bulk copy, once both warpgroups are done with the previous one
        if (tid == 0) {
            g_mbar_wait(bar_empty, par ^ 1u);
            g_mbar_expect_tx(bar_full, (uint32_t)bblk);
            g_bulk_g2s(sB, p.bimg + ((int64_t)tile * nkb + kb) * bblk, (uint32_t)bblk, bar_full);
        }
        // (2) this warpgroup's weight rows -> fp16 integers in the swizzled K-major layout
        if constexpr (C::IS_Q6) dequant_q6_block_to_smem(wrow + (int64_t)kb * BB, row_ok, r, h, sA, sAx);
        else dequant_block_to_smem<T>(wrow + (int64_t)kb * BB, row_ok, r, h, sA, sAx);
        fence_proxy_async();                                // generic-proxy smem writes -> visible to the tensor core (async proxy)
        wg_bar_sync(wg);
        float dw_lo = 0.0f, dw_hi = 0.0f, dm_lo = 0.0f, dm_hi = 0.0f;
        if constexpr (C::IS_Q6) {
            if (ok_lo) dw_lo = __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short *>(ew_lo + (int64_t)kb * BB + 208))));
            if (ok_hi) dw_hi = __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short *>(ew_hi + (int64_t)kb * BB + 208))));
        } else {
            if (ok_lo) {
                const uint32_t dd = __ldg(reinterpret_cast<const uint32_t *>(ew_lo + (int64_t)kb * BB));
                dw_lo = __half2float(__ushort_as_half((unsigned short)(dd & 0xFFFFu)));
                dm_lo = __half2float(__ushort_as_half((unsigned short)(dd >> 16)));
            }
            if (ok_hi) {
                const uint32_t dd = __ldg(reinterpret_cast<const uint32_t *>(ew_hi + (int64_t)kb * BB));
                dw_hi = __half2float(__ushort_as_half((unsigned short)(dd & 0xFFFFu)));
                dm_hi = __half2float(__ushort_as_half((unsigned short)(dd >> 16)));
            }
        }
        const float * dap = p.da + (int64_t)kb * p.npad + tile * GEMM_NT;
        g_mbar_wait(bar_full, par);
        // (3) mins term: one K = 16 MMA; acc += d_a * (-dmin_w * mins)
        if constexpr (!C::IS_Q6) {
            acc_fence(v);
            wgmma_fence();
            wgmma_m64n128k16_f16(v, make_desc_sw128(s32(sAx) + a_off), make_desc_sw128(s32(sB + 4 * C::ATOM_B)), 0u);
            wgmma_commit();
            wgmma_wait<0>();
            acc_fence(v);
            kq_combine(acc, v, -dm_lo, -dm_hi, dap, c4);
        }
        // (4) main term: 16 MMAs (Q6_K: 32, both scale parts into the same accumulator); acc += d_a * (d_w * main)
        acc_fence(v);
        wgmma_fence();
#pragma unroll
        for (int a = 0; a < 4; a++) {
#pragma unroll
            for (int ks = 0; ks < 4; ks++) {
                const uint64_t db_ = make_desc_sw128(s32(sB + a * C::ATOM_B) + ks * 32);
                wgmma_m64n128k16_f16(v, make_desc_sw128(s32(sA + a * C::ATOM_A) + a_off + ks * 32), db_, (a | ks) != 0 ? 1u : 0u);
                if constexpr (C::IS_Q6) wgmma_m64n128k16_f16(v, make_desc_sw128(s32(sAx + a * C::ATOM_A) + a_off + ks * 32), db_, 1u);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(v);
        g_mbar_arrive(bar_empty);                           // this thread's reads of B (and of its warpgroup's A rows) are done
        kq_combine(acc, v, dw_lo, dw_hi, dap, c4);
    }

    // (5) write out: dst[n*ldd + m]
#pragma unroll
    for (int i = 0; i < 16; i++) {
#pragma unroll
        for (int c = 0; c < 2; c++) {
            const int col = gemm_dst_col_t<GROUPED>(p, tile * GEMM_NT + 8 * i + 2 * c4 + c);
            if (col < 0) continue;
            if (ok_lo) p.dst[(int64_t)col * p.ldd + m0 + er] = acc[4 * i + c];
            if (ok_hi) p.dst[(int64_t)col * p.ldd + m0 + er + 8] = acc[4 * i + 2 + c];
        }
    }
}

template <int T>
static cudaError_t launch_kq(const GemmKArgs & k, dim3 grid, cudaStream_t st) {
    static bool attr_done[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr_done[dev]) {
        cudaError_t e = cudaFuncSetAttribute(gemm_q_wgmma_kernel<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KqCfg<T>::SMEM);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(gemm_q_wgmma_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)KqCfg<T>::SMEM);
        if (e != cudaSuccess) return e;
        attr_done[dev] = true;
    }
    if (k.tile_expert != nullptr) gemm_q_wgmma_kernel<T, true><<<grid, GEMM_THREADS, KqCfg<T>::SMEM, st>>>(k);
    else gemm_q_wgmma_kernel<T, false><<<grid, GEMM_THREADS, KqCfg<T>::SMEM, st>>>(k);
    return cudaGetLastError();
}

// which operand images the workspace holds (0 K-quant, 1 legacy): a caller's reuse_operands flag only names the activation
static thread_local int g_last_gemm_family = 0;
static thread_local bool g_kquant_images_stale = false;
static inline void g_last_gemm_family_guard() { if (g_last_gemm_family == 1) { g_kquant_images_stale = true; g_last_gemm_family = 0; } }

cudaError_t launch_gemm(int type, const GemmArgs & a, cudaStream_t st) {
    if (type == T_Q4_0 || type == T_Q8_0) {
        // the legacy formats have their own operand images: "same activation as last time" only holds after another legacy launch
        static thread_local const void * last_ws_l = nullptr;
        GemmArgs b = a;
        b.reuse_operands = a.reuse_operands && last_ws_l == a.workspace && g_last_gemm_family == 1;
        const cudaError_t e = launch_gemm_legacy(type, b, st);
        if (e == cudaSuccess) { last_ws_l = a.workspace; g_last_gemm_family = 1; }
        return e;
    }
    g_last_gemm_family_guard();
    if (!(type == T_Q4_K || type == T_Q5_K || type == T_Q6_K) || a.K % 256 || a.N <= 0 || a.M <= 0) return cudaErrorNotSupported;
    if (type == T_Q6_K ? ((reinterpret_cast<uintptr_t>(a.w) & 1) || (a.row_stride & 1)) : ((reinterpret_cast<uintptr_t>(a.w) & 15) || (a.row_stride & 15))) return cudaErrorMisalignedAddress;
    const int NT = GEMM_NT;
    const int npad = (int)rup(a.N, NT), nkb = a.K / 256, ntiles = npad / NT;
    if (a.workspace_bytes < gemm_workspace_bytes(type, a.M, a.N, a.K)) return cudaErrorInvalidValue;
    if ((reinterpret_cast<uintptr_t>(a.x) & 15) || (a.ldx & 3)) return cudaErrorMisalignedAddress;   // the pre-pass reads float4
    uint8_t * bimg = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(a.workspace) + 255) & ~uintptr_t(255));
    float * da = reinterpret_cast<float *>(bimg + (int64_t)ntiles * nkb * gl::bimg_block_bytes(NT));
    cudaError_t e = cudaSuccess;
    static thread_local const void * last_ws = nullptr;
    const bool reuse = a.reuse_operands && last_ws == a.workspace && !g_kquant_images_stale;
    g_kquant_images_stale = false;
    last_ws = a.workspace;
    if (!reuse) {
        note_launch();
        quantize_act_gemm_kernel<<<dim3((unsigned)nkb, (unsigned)(npad / 8)), 256, 0, st>>>(a.x, a.ldx, a.N, nkb, npad, bimg, da, NT, nullptr);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    GemmKArgs k{a.w, a.row_stride, a.M, a.K, a.N, npad, bimg, da, a.dst, a.ldd, nullptr, nullptr, 0};
    const dim3 grid((unsigned)((a.M + GEMM_MT - 1) / GEMM_MT), (unsigned)ntiles);
    note_launch();
    if (type == T_Q4_K) return launch_kq<T_Q4_K>(k, grid, st);
    if (type == T_Q5_K) return launch_kq<T_Q5_K>(k, grid, st);
    return launch_kq<T_Q6_K>(k, grid, st);
}

// ------------------------------------------------------------------------------------------------ grouped GEMM (MUL_MAT_ID, many tokens)
// ggml_compute_forward_mul_mat_id (ggml-cpu.c:1534-1707) groups the (token, slot) rows by expert on one thread and runs one mat-mul
// per expert.  Here: one small kernel sorts the jobs by expert into column tiles (all on the device, no host round trip: the launch
// covers the worst-case number of tiles and the tiles that do not exist exit at once), the activation pre-pass gathers each tile's
// columns, and the GEMM kernel takes the expert's weights per tile and scatters the output columns.
__global__ void __launch_bounds__(1024) moe_route_kernel(const int32_t * __restrict__ ids, int64_t ids_stride, int T, int n_used, int nb1, int n_expert, int NT, int max_tiles,
                                                         int * __restrict__ tile_expert, int * __restrict__ col_src, int * __restrict__ col_dst) {
    __shared__ int cnt[256], base[256], fill[256];
    const int tid = threadIdx.x, R = T * n_used;
    for (int e = tid; e < n_expert; e += blockDim.x) { cnt[e] = 0; fill[e] = 0; }
    for (int i = tid; i < max_tiles; i += blockDim.x) tile_expert[i] = -1;
    for (int i = tid; i < max_tiles * NT; i += blockDim.x) { col_src[i] = -1; col_dst[i] = -1; }
    __syncthreads();
    for (int j = tid; j < R; j += blockDim.x) {
        const int t = j / n_used, s_ = j % n_used, e = ids[(int64_t)t * ids_stride + s_];
        if (e >= 0 && e < n_expert) atomicAdd(&cnt[e], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int tiles = 0;
        for (int e = 0; e < n_expert; e++) {
            base[e] = tiles * NT;
            const int nt = (cnt[e] + NT - 1) / NT;
            for (int q = 0; q < nt; q++) tile_expert[tiles + q] = e;
            tiles += nt;
        }
    }
    __syncthreads();
    for (int j = tid; j < R; j += blockDim.x) {
        const int t = j / n_used, s_ = j % n_used, e = ids[(int64_t)t * ids_stride + s_];
        if (e < 0 || e >= n_expert) continue;
        const int pos = base[e] + atomicAdd(&fill[e], 1);     // (the order inside an expert's group does not change any result: columns are independent)
        col_src[pos] = t * nb1 + (nb1 == 1 ? 0 : s_);
        col_dst[pos] = j;
    }
}

static_assert(MOE_TILE_COLS == GEMM_NT, "the router's tiles are the GEMM's column tiles");

cudaError_t launch_moe_route(const int32_t * ids, int64_t ids_stride, int T, int n_used, int nb1, int n_expert, int max_tiles,
                             int * tile_expert, int * col_src, int * col_dst, cudaStream_t st) {
    if (n_expert <= 0 || n_expert > 256) return cudaErrorNotSupported;      // the per-expert counters live in shared memory
    moe_route_kernel<<<1, 1024, 0, st>>>(ids, ids_stride, T, n_used, nb1, n_expert, GEMM_NT, max_tiles, tile_expert, col_src, col_dst);
    return cudaGetLastError();
}

size_t gemm_grouped_workspace_bytes(int type, int64_t M, int64_t jobs, int64_t n_expert, int64_t K) {
    (void)M;
    if (!(type == T_Q4_K || type == T_Q5_K || type == T_Q6_K) || K % 256 || jobs <= 0 || n_expert > 256) return 0;
    const int NT = GEMM_NT;
    const int64_t max_tiles = moe_max_tiles(jobs, n_expert), nkb = K / 256;
    return (size_t)(max_tiles * nkb * gl::bimg_block_bytes(NT) + nkb * max_tiles * NT * 4 + (max_tiles + 2 * max_tiles * NT) * 4 + 2048);
}

cudaError_t launch_gemm_grouped(int type, const GemmGroupedArgs & a, cudaStream_t st) {
    if (!(type == T_Q4_K || type == T_Q5_K || type == T_Q6_K) || a.K % 256 || a.M <= 0 || a.T <= 0 || a.n_used <= 0 || a.n_expert <= 0 || a.n_expert > 256) return cudaErrorNotSupported;
    if (type == T_Q6_K ? ((reinterpret_cast<uintptr_t>(a.w) & 1) || (a.row_stride & 1) || (a.expert_stride & 1)) : ((reinterpret_cast<uintptr_t>(a.w) & 15) || (a.row_stride & 15) || (a.expert_stride & 15))) return cudaErrorMisalignedAddress;
    if ((reinterpret_cast<uintptr_t>(a.x) & 15) || (a.ldx & 3)) return cudaErrorMisalignedAddress;
    const int NT = GEMM_NT;
    const int64_t jobs = (int64_t)a.T * a.n_used;
    const int max_tiles = (int)moe_max_tiles(jobs, a.n_expert), nkb = a.K / 256, npad = max_tiles * NT;
    if (a.workspace_bytes < gemm_grouped_workspace_bytes(type, a.M, jobs, a.n_expert, a.K)) return cudaErrorInvalidValue;
    uint8_t * bimg = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(a.workspace) + 255) & ~uintptr_t(255));
    float * da = reinterpret_cast<float *>(bimg + (int64_t)max_tiles * nkb * gl::bimg_block_bytes(NT));
    int * tile_expert = reinterpret_cast<int *>(da + (int64_t)nkb * npad);
    int * col_src = tile_expert + max_tiles, * col_dst = col_src + npad;
    note_launch(2);
    cudaError_t e = launch_moe_route(a.ids, a.ids_stride, a.T, a.n_used, a.nb1, a.n_expert, max_tiles, tile_expert, col_src, col_dst, st);
    if (e != cudaSuccess) return e;
    quantize_act_gemm_kernel<<<dim3((unsigned)nkb, (unsigned)(npad / 8)), 256, 0, st>>>(a.x, a.ldx, 0, nkb, npad, bimg, da, NT, col_src);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    GemmKArgs k{a.w, a.row_stride, a.M, a.K, npad, npad, bimg, da, a.dst, a.ldd, tile_expert, col_dst, a.expert_stride};
    const dim3 grid((unsigned)((a.M + GEMM_MT - 1) / GEMM_MT), (unsigned)max_tiles);
    note_launch();
    if (type == T_Q4_K) return launch_kq<T_Q4_K>(k, grid, st);
    if (type == T_Q5_K) return launch_kq<T_Q5_K>(k, grid, st);
    return launch_kq<T_Q6_K>(k, grid, st);
}

}  // namespace qmm
