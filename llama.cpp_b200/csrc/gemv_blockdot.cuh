// gemv_blockdot.cuh -- pieces shared by the decode GEMV kernels (gemv2.cu, gemv3.cu, decode_flow.cu): tile configuration, the
// mbarrier / cp.async.bulk PTX wrappers and the per-lane 256-weight block dot products.
#pragma once
#include "qmm_formats.cuh"
#include "qmm_kernels.cuh"

namespace qmm {

template <int T> struct G2 {
    static constexpr int BB     = Fmt<T>::BB;
    static constexpr int PIECEB = 8 * BB;                           // bytes of one full row piece (8 blocks)
    static constexpr int PIECE  = (PIECEB + 16 + 15) / 16 * 16;      // smem pitch of a piece: + align-down offset, 16B multiple
    static constexpr int SLOT   = 4 * PIECE + 16;                    // 4 rows + read slack
    static constexpr int WARPS  = (T == T_Q6_K) ? 5 : 6;
    static constexpr int STAGES = 3;
    static constexpr int BSB    = (T == T_Q6_K) ? 48 : 16;           // bytes of bsums per block in smem (Q6_K: 16 x i16 + pad)
    static constexpr int ACTB   = 272;                               // skewed pitch of one block of int8 activations
};

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t * bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t * bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.b32 %0, 1, 0, P1;\n\t}\n"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    int spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1 << 24)) __trap();       // a lost copy must fail the launch, never hang the GPU
    }
}
__device__ __forceinline__ void bulk_g2s(void * smem_dst, const void * gsrc, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// An L2 policy that marks every line it covers evict-first, and bulk_g2s under such a policy: data read once on its way to shared memory
// then leaves L2 before the lines that are read again.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void * smem_dst, const void * gsrc, uint32_t bytes, uint64_t * bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ int dp4a_us(uint32_t a_unsigned, uint32_t b_signed, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;\n" : "=r"(d) : "r"(a_unsigned), "r"(b_signed), "r"(c));
    return d;
}
__device__ __forceinline__ uint4 lds128(const uint8_t * p) { return *reinterpret_cast<const uint4 *>(p); }

// ---------------------------------------------------------------- per-block dot products (one lane, 256 weights)
// act: smem pointer to this block's 256 int8 (skewed plane), bs: its bsums entry, da: its Q8_K scale.
template <int T> struct BlockDot;

template <> struct BlockDot<T_Q4_K> {
    // weights: 9 x 16 B, 16-byte aligned in smem
    __device__ __forceinline__ static float run(const uint8_t * wb, const uint8_t * act, const uint8_t * bs, float da) {
        const uint4 hdr = lds128(wb);
        // 6-bit scales/mins -> 2 x 4 packed bytes each (the reference's utmp shuffle, ggml-cpu/quants.c:726-731)
        const uint32_t sc_lo = hdr.y & 0x3f3f3f3fu, mn_lo = hdr.z & 0x3f3f3f3fu;
        const uint32_t sc_hi = (hdr.w & 0x0f0f0f0fu) | (((hdr.y >> 6) & 0x03030303u) << 4);
        const uint32_t mn_hi = ((hdr.w >> 4) & 0x0f0f0f0fu) | (((hdr.z >> 6) & 0x03030303u) << 4);
        int tot = 0;
#pragma unroll
        for (int g = 0; g < 4; g++) {                       // 64 weights: qs[32g..32g+32) low -> sub-block 2g, high -> 2g+1
            const uint4 q0 = lds128(wb + 16 + 32 * g), q1 = lds128(wb + 32 + 32 * g);
            const uint4 a0 = lds128(act + 64 * g), a1 = lds128(act + 64 * g + 16);
            const uint4 a2 = lds128(act + 64 * g + 32), a3 = lds128(act + 64 * g + 48);
            // four independent dp4a chains (two per nibble plane) instead of two chains of eight: the warp's issue rate was
            // bounded by dependent IDP latency, not by the number of instructions
            int sl = 0, sh = 0, sl2 = 0, sh2 = 0;
            sl  = __dp4a((int)(q0.x & 0x0F0F0F0Fu), (int)a0.x, sl);  sh  = dp4a_us(q0.x & 0xF0F0F0F0u, a2.x, sh);
            sl2 = __dp4a((int)(q0.y & 0x0F0F0F0Fu), (int)a0.y, sl2); sh2 = dp4a_us(q0.y & 0xF0F0F0F0u, a2.y, sh2);
            sl  = __dp4a((int)(q0.z & 0x0F0F0F0Fu), (int)a0.z, sl);  sh  = dp4a_us(q0.z & 0xF0F0F0F0u, a2.z, sh);
            sl2 = __dp4a((int)(q0.w & 0x0F0F0F0Fu), (int)a0.w, sl2); sh2 = dp4a_us(q0.w & 0xF0F0F0F0u, a2.w, sh2);
            sl  = __dp4a((int)(q1.x & 0x0F0F0F0Fu), (int)a1.x, sl);  sh  = dp4a_us(q1.x & 0xF0F0F0F0u, a3.x, sh);
            sl2 = __dp4a((int)(q1.y & 0x0F0F0F0Fu), (int)a1.y, sl2); sh2 = dp4a_us(q1.y & 0xF0F0F0F0u, a3.y, sh2);
            sl  = __dp4a((int)(q1.z & 0x0F0F0F0Fu), (int)a1.z, sl);  sh  = dp4a_us(q1.z & 0xF0F0F0F0u, a3.z, sh);
            sl2 = __dp4a((int)(q1.w & 0x0F0F0F0Fu), (int)a1.w, sl2); sh2 = dp4a_us(q1.w & 0xF0F0F0F0u, a3.w, sh2);
            sl += sl2; sh += sh2;
            const uint32_t scw = g < 2 ? sc_lo : sc_hi;
            const int s0 = (int)((scw >> (16 * (g & 1))) & 0xFFu), s1 = (int)((scw >> (16 * (g & 1) + 8)) & 0xFFu);
            tot += s0 * sl + s1 * (sh >> 4);                // sh is an exact multiple of 16
        }
        const uint4 b = lds128(bs);                         // 8 x int16: sums of the 8 sub-blocks of 32 activations
        int mins = 0;
        mins = __dp2a_lo((int)b.x, (int)mn_lo, mins); mins = __dp2a_hi((int)b.y, (int)mn_lo, mins);
        mins = __dp2a_lo((int)b.z, (int)mn_hi, mins); mins = __dp2a_hi((int)b.w, (int)mn_hi, mins);
        const float dw = __half2float(__ushort_as_half((unsigned short)(hdr.x & 0xFFFFu)));
        const float dm = __half2float(__ushort_as_half((unsigned short)(hdr.x >> 16)));
        return (dw * da) * (float)tot - (dm * da) * (float)mins;
    }
};

template <> struct BlockDot<T_Q5_K> {
    // d,dmin,scales[12] | qh[32] | qs[128] : 11 x 16 B, 16-byte aligned
    __device__ __forceinline__ static float run(const uint8_t * wb, const uint8_t * act, const uint8_t * bs, float da) {
        const uint4 hdr = lds128(wb);
        const uint4 h0 = lds128(wb + 16), h1 = lds128(wb + 32);      // qh[l], l = 0..15 / 16..31
        const uint32_t sc_lo = hdr.y & 0x3f3f3f3fu, mn_lo = hdr.z & 0x3f3f3f3fu;
        const uint32_t sc_hi = (hdr.w & 0x0f0f0f0fu) | (((hdr.y >> 6) & 0x03030303u) << 4);
        const uint32_t mn_hi = ((hdr.w >> 4) & 0x0f0f0f0fu) | (((hdr.z >> 6) & 0x03030303u) << 4);
        int tot = 0;
#pragma unroll
        for (int g = 0; g < 4; g++) {
            const uint4 q0 = lds128(wb + 48 + 32 * g), q1 = lds128(wb + 64 + 32 * g);
            const uint4 a0 = lds128(act + 64 * g), a1 = lds128(act + 64 * g + 16);
            const uint4 a2 = lds128(act + 64 * g + 32), a3 = lds128(act + 64 * g + 48);
            int sl = 0, sh = 0;
            // bit 2g of qh[l] is the 5th bit of low-nibble element l, bit 2g+1 of the high-nibble element
#define QMM_W(Q, H, AL, AH)                                                                                     \
            sl = __dp4a((int)((Q & 0x0F0F0F0Fu) | (((H >> (2 * g)) & 0x01010101u) << 4)), (int)AL, sl);          \
            sh = __dp4a((int)(((Q >> 4) & 0x0F0F0F0Fu) | (((H >> (2 * g + 1)) & 0x01010101u) << 4)), (int)AH, sh);
            QMM_W(q0.x, h0.x, a0.x, a2.x) QMM_W(q0.y, h0.y, a0.y, a2.y) QMM_W(q0.z, h0.z, a0.z, a2.z) QMM_W(q0.w, h0.w, a0.w, a2.w)
            QMM_W(q1.x, h1.x, a1.x, a3.x) QMM_W(q1.y, h1.y, a1.y, a3.y) QMM_W(q1.z, h1.z, a1.z, a3.z) QMM_W(q1.w, h1.w, a1.w, a3.w)
#undef QMM_W
            const uint32_t scw = g < 2 ? sc_lo : sc_hi;
            const int s0 = (int)((scw >> (16 * (g & 1))) & 0xFFu), s1 = (int)((scw >> (16 * (g & 1) + 8)) & 0xFFu);
            tot += s0 * sl + s1 * sh;
        }
        const uint4 b = lds128(bs);
        int mins = 0;
        mins = __dp2a_lo((int)b.x, (int)mn_lo, mins); mins = __dp2a_hi((int)b.y, (int)mn_lo, mins);
        mins = __dp2a_lo((int)b.z, (int)mn_hi, mins); mins = __dp2a_hi((int)b.w, (int)mn_hi, mins);
        const float dw = __half2float(__ushort_as_half((unsigned short)(hdr.x & 0xFFFFu)));
        const float dm = __half2float(__ushort_as_half((unsigned short)(hdr.x >> 16)));
        return (dw * da) * (float)tot - (dm * da) * (float)mins;
    }
};

template <> struct BlockDot<T_Q6_K> {
    // ql[128] | qh[64] | scales[16] | d : 210 B, only 2-byte aligned -> aligned word reads + funnel shift
    __device__ __forceinline__ static float run(const uint8_t * wb, const uint8_t * act, const uint8_t * bs, float da) {
        const uint32_t * w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(wb) & ~uintptr_t(3));
        const uint32_t fs = (uint32_t)(reinterpret_cast<uintptr_t>(wb) & 2) * 8;
        int tot = 0;
        // scales: bytes 192..207 = words 48..51
        uint32_t scw[4];
        {
            uint32_t p = w[48];
#pragma unroll
            for (int i = 0; i < 4; i++) { const uint32_t n = w[49 + i]; scw[i] = __funnelshift_r(p, n, fs); p = n; }
        }
        const uint4 b0 = lds128(bs), b1 = lds128(bs + 16);           // 16 x int16 bsums (sums of 16 activations)
        const uint32_t bsw[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int h = 0; h < 2; h++) {                                // 128 weights per half
            // ql words 16h.. (64 B = 16 words): l = 0..31 -> quarters 0 (low nibble) / 2 (high); l+32 -> quarters 1 / 3
            uint32_t ql[16], qh[8];
            {
                uint32_t p = w[16 * h];
#pragma unroll
                for (int i = 0; i < 16; i++) { const uint32_t n = w[16 * h + 1 + i]; ql[i] = __funnelshift_r(p, n, fs); p = n; }
                p = w[32 + 8 * h];
#pragma unroll
                for (int i = 0; i < 8; i++) { const uint32_t n = w[32 + 8 * h + 1 + i]; qh[i] = __funnelshift_r(p, n, fs); p = n; }
            }
#pragma unroll
            for (int qtr = 0; qtr < 4; qtr++) {                      // 32 weights: elements 128h + 32qtr + l
                const uint8_t * ap = act + 128 * h + 32 * qtr;
                const uint4 a0 = lds128(ap), a1 = lds128(ap + 16);
                const uint32_t av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                int s_lo = 0, s_hi = 0;                              // l < 16 and l >= 16 use different scales
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t lo = ql[(qtr & 1) * 8 + i];
                    const uint32_t nib = (qtr < 2 ? lo : (lo >> 4)) & 0x0F0F0F0Fu;
                    const uint32_t c = nib | (((qh[i] >> (2 * qtr)) & 0x03030303u) << 4);   // 0..63
                    if (i < 4) s_lo = __dp4a((int)c, (int)av[i], s_lo); else s_hi = __dp4a((int)c, (int)av[i], s_hi);
                }
                // scale index 8h + 2qtr (+1 for l >= 16); (q - 32): subtract 32 * bsum of the same 16 activations
                const int si = 8 * h + 2 * qtr;
                const int sc0 = (int)(int8_t)((scw[si >> 2] >> (8 * (si & 3))) & 0xFFu);
                const int sc1 = (int)(int8_t)((scw[(si + 1) >> 2] >> (8 * ((si + 1) & 3))) & 0xFFu);
                const uint32_t bw = bsw[si >> 1];                    // bsums[si], bsums[si+1]
                const int bsum0 = (int)(int16_t)(bw & 0xFFFFu), bsum1 = (int)(int16_t)(bw >> 16);
                tot += sc0 * (s_lo - 32 * bsum0) + sc1 * (s_hi - 32 * bsum1);
            }
        }
        const float dw = __half2float(__ushort_as_half(*reinterpret_cast<const unsigned short *>(wb + 208)));
        return (dw * da) * (float)tot;
    }
};

}  // namespace qmm
