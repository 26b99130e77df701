// qmm_formats.cuh -- GGUF block formats as seen by the kernels.
//
// Everything here is index arithmetic on the reference's on-disk block layouts
// (ggml/src/ggml-common.h:194-376) plus the per-"unit" integer dot products the decode GEMV is built from.
// The functions are QMM_HD so the same code compiles for the host: tests/host_units.cpp runs them on the
// CPU against the oracle (the only way to check the index math without a GPU in the build container).
//
// Vocabulary
//   block    : one ggml quantisation block (32 weights for Q4_0/Q8_0, 256 for the K-quants)
//   segment  : 2048 consecutive weights of one row (64/8 blocks); its byte size is a multiple of 16 for all
//              five formats, so a segment of a 16-byte aligned row is a whole number of 16-byte HBM loads
//   unit     : 32 weights of a segment, the work item of one lane; 64 units per segment, 2 per lane
//
// Activation operand ("ActQ8", our own device layout -- never leaves the GPU):
//   qs    int8  [K]        quantised activations, exactly the CPU's block_q8_K.qs / block_q8_0.qs values
//   d     f32   [K/256] (Q8_K, = block_q8_K.d)  or  [K/32] (Q8_0, = fp16-rounded block_q8_0.d widened to f32)
//   bsums int16 [K/16] (Q8_K, = block_q8_K.bsums)  or  [K/32] (Q8_0: sum of the 32 qs, our addition so that
//                      Q4_0's "(q-8)" offset becomes  dot(q,a) - 8*bsum  in integers)
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#include <cuda_fp16.h>
#define QMM_HD __host__ __device__ __forceinline__
#else
#define QMM_HD inline
#endif

namespace qmm {

// enum ggml_type values (ggml/include/ggml.h:388-410)
enum : int { T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q8_0 = 8, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14, T_Q8_K = 15 };

constexpr int SEG_ELEMS = 2048;   // weights per segment
constexpr int SEG_UNITS = 64;     // 32-weight units per segment

template <int T> struct Fmt;
template <> struct Fmt<T_Q4_0> { static constexpr int BE = 32,  BB = 18,  ACT = T_Q8_0, ALIGN = 2;  };
template <> struct Fmt<T_Q8_0> { static constexpr int BE = 32,  BB = 34,  ACT = T_Q8_0, ALIGN = 2;  };
template <> struct Fmt<T_Q4_K> { static constexpr int BE = 256, BB = 144, ACT = T_Q8_K, ALIGN = 16; };
template <> struct Fmt<T_Q5_K> { static constexpr int BE = 256, BB = 176, ACT = T_Q8_K, ALIGN = 16; };
template <> struct Fmt<T_Q6_K> { static constexpr int BE = 256, BB = 210, ACT = T_Q8_K, ALIGN = 2;  };

QMM_HD int block_elems(int t) { return (t == T_Q4_0 || t == T_Q8_0) ? 32 : 256; }
QMM_HD int block_bytes(int t) {
    switch (t) { case T_Q4_0: return 18; case T_Q8_0: return 34; case T_Q4_K: return 144; case T_Q5_K: return 176; case T_Q6_K: return 210; }
    return 0;
}
QMM_HD bool act_is_q8_K(int t) { return t == T_Q4_K || t == T_Q5_K || t == T_Q6_K; }

// ---------------------------------------------------------------- small helpers
QMM_HD int dp4a_ss(uint32_t a, uint32_t b, int c) {   // signed x signed bytes
#if defined(__CUDA_ARCH__)
    return __dp4a((int)a, (int)b, c);
#else
    for (int i = 0; i < 4; i++) c += (int)(int8_t)(a >> (8 * i)) * (int)(int8_t)(b >> (8 * i));
    return c;
#endif
}

QMM_HD float half_bits_to_float(uint16_t h) {
#if defined(__CUDA_ARCH__)
    return __half2float(__ushort_as_half(h));
#else
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1Fu, man = h & 0x3FFu, bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else { int e = -1; do { man <<= 1; e++; } while (!(man & 0x400u)); bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3FFu) << 13); }
    } else if (exp == 31) bits = sign | 0x7F800000u | (man << 13);
    else bits = sign | ((exp + 112u) << 23) | (man << 13);
    float f; memcpy(&f, &bits, 4); return f;
#endif
}

struct U4 { uint32_t x, y, z, w; };
struct U2 { uint32_t x, y; };

// 16 bytes from a 16-byte aligned address
QMM_HD U4 ld16_a16(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
    uint4 v = *reinterpret_cast<const uint4 *>(p); return U4{v.x, v.y, v.z, v.w};
#else
    U4 v; memcpy(&v, p, 16); return v;
#endif
}
// n 32-bit words from an address that is only 2-byte aligned: read the enclosing aligned words and funnel-shift.
// Touches up to 2 bytes past the last word when misaligned (staging buffers carry 16 bytes of slack).
QMM_HD uint32_t ld4_a2(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
    const uint32_t * w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(3));
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 2) * 8;
    return __funnelshift_r(w[0], w[1], sh);
#else
    uint32_t v; memcpy(&v, p, 4); return v;
#endif
}
QMM_HD U2 ld8_a2(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
    const uint32_t * w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(3));
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 2) * 8;
    const uint32_t a = w[0], b = w[1], c = w[2];
    return U2{__funnelshift_r(a, b, sh), __funnelshift_r(b, c, sh)};
#else
    U2 v; memcpy(&v, p, 8); return v;
#endif
}
QMM_HD U4 ld16_a2(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
    const uint32_t * w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(3));
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 2) * 8;
    const uint32_t a = w[0], b = w[1], c = w[2], d = w[3], e = w[4];
    return U4{__funnelshift_r(a, b, sh), __funnelshift_r(b, c, sh), __funnelshift_r(c, d, sh), __funnelshift_r(d, e, sh)};
#else
    U4 v; memcpy(&v, p, 16); return v;
#endif
}
QMM_HD uint16_t ld2(const uint8_t * p) {
#if defined(__CUDA_ARCH__)
    return *reinterpret_cast<const uint16_t *>(p);
#else
    uint16_t v; memcpy(&v, p, 2); return v;
#endif
}

// activation loads: global memory, 16-byte aligned for K-quant units (offsets are multiples of 16), 8-byte for Q6_K
QMM_HD U4 ldg16(const int8_t * p) {
#if defined(__CUDA_ARCH__)
    int4 v = __ldg(reinterpret_cast<const int4 *>(p)); return U4{(uint32_t)v.x, (uint32_t)v.y, (uint32_t)v.z, (uint32_t)v.w};
#else
    U4 v; memcpy(&v, p, 16); return v;
#endif
}
QMM_HD U2 ldg8(const int8_t * p) {
#if defined(__CUDA_ARCH__)
    int2 v = __ldg(reinterpret_cast<const int2 *>(p)); return U2{(uint32_t)v.x, (uint32_t)v.y};
#else
    U2 v; memcpy(&v, p, 8); return v;
#endif
}

// 6-bit (scale, min) pair j of a Q4_K/Q5_K block; s0,s1,s2 = the 12 scale bytes as 3 little-endian words.
// Restates get_scale_min_k4 (ggml/src/ggml-quants.c:880-888) with shifts only (no dynamically indexed arrays,
// which would live in local memory on the device).
QMM_HD void k4_scale_min(int j, uint32_t s0, uint32_t s1, uint32_t s2, int & sc, int & mn) {
    const int sh = 8 * (j & 3);
    const uint32_t b0 = (s0 >> sh) & 0xFFu, b1 = (s1 >> sh) & 0xFFu, b2 = (s2 >> sh) & 0xFFu;
    if (j < 4) {
        sc = (int)(b0 & 63u);
        mn = (int)(b1 & 63u);
    } else {
        sc = (int)((b2 & 0x0Fu) | ((b0 >> 6) << 4));
        mn = (int)((b2 >> 4)    | ((b1 >> 6) << 4));
    }
}

// Activation operand of one column, positioned at element 0 of the row.
struct ActCol {
    const int8_t  * qs;
    const float   * d;
    const int16_t * bsums;
};

// ---------------------------------------------------------------- unit dot products
// unit_dot<T>(seg, u, kseg, act): contribution of unit u (32 weights) of the segment whose first block is at
// `seg` (shared memory on the device, alignment Fmt<T>::ALIGN) and whose first weight is element `kseg` of the
// row, against one activation column.  Integer parts are exact (they equal the CPU's int32 sums re-grouped);
// the result is  d_w * d_a * int  (- dmin * d_a * int) in fp32, i.e. the CPU's per-block combine
// (ggml-cpu/quants.c:254-255,743-767,899-902) applied per unit.
template <int T> QMM_HD float unit_dot(const uint8_t * seg, int u, int kseg, const ActCol & a);

template <> QMM_HD float unit_dot<T_Q4_K>(const uint8_t * seg, int u, int kseg, const ActCol & a) {
    const int blk = u >> 3, c = u & 7, g = c >> 1, h = c & 1;
    const uint8_t * b = seg + blk * 144;
    const U4 hdr = ld16_a16(b);                       // d | dmin<<16, scales[0..11]
    const U4 q   = ld16_a16(b + 16 + 16 * c);         // qs[32g + 16h .. +16): low nibbles = elems 64g+16h.., high = +32
    int sc0, mn0, sc1, mn1;
    k4_scale_min(2 * g, hdr.y, hdr.z, hdr.w, sc0, mn0);
    k4_scale_min(2 * g + 1, hdr.y, hdr.z, hdr.w, sc1, mn1);
    const int e0 = kseg + blk * 256 + 64 * g + 16 * h;
    const U4 alo = ldg16(a.qs + e0), ahi = ldg16(a.qs + e0 + 32);
    int s0 = 0, s1 = 0;
    s0 = dp4a_ss(q.x & 0x0F0F0F0Fu, alo.x, s0); s1 = dp4a_ss((q.x >> 4) & 0x0F0F0F0Fu, ahi.x, s1);
    s0 = dp4a_ss(q.y & 0x0F0F0F0Fu, alo.y, s0); s1 = dp4a_ss((q.y >> 4) & 0x0F0F0F0Fu, ahi.y, s1);
    s0 = dp4a_ss(q.z & 0x0F0F0F0Fu, alo.z, s0); s1 = dp4a_ss((q.z >> 4) & 0x0F0F0F0Fu, ahi.z, s1);
    s0 = dp4a_ss(q.w & 0x0F0F0F0Fu, alo.w, s0); s1 = dp4a_ss((q.w >> 4) & 0x0F0F0F0Fu, ahi.w, s1);
    const int kb = (kseg >> 8) + blk;                 // Q8_K block index in the row
    const int bs0 = a.bsums[kb * 16 + 4 * g + h], bs1 = a.bsums[kb * 16 + 4 * g + 2 + h];
    const float da = a.d[kb];
    const float dw = half_bits_to_float((uint16_t)(hdr.x & 0xFFFFu)), dminw = half_bits_to_float((uint16_t)(hdr.x >> 16));
    return (dw * da) * (float)(sc0 * s0 + sc1 * s1) - (dminw * da) * (float)(mn0 * bs0 + mn1 * bs1);
}

template <> QMM_HD float unit_dot<T_Q5_K>(const uint8_t * seg, int u, int kseg, const ActCol & a) {
    const int blk = u >> 3, c = u & 7, g = c >> 1, h = c & 1;
    const uint8_t * b = seg + blk * 176;
    const U4 hdr = ld16_a16(b);
    const U4 qh  = ld16_a16(b + 16 + 16 * h);         // qh[16h .. 16h+16): bit 2g -> low-nibble elems, bit 2g+1 -> high
    const U4 q   = ld16_a16(b + 48 + 16 * c);
    int sc0, mn0, sc1, mn1;
    k4_scale_min(2 * g, hdr.y, hdr.z, hdr.w, sc0, mn0);
    k4_scale_min(2 * g + 1, hdr.y, hdr.z, hdr.w, sc1, mn1);
    const int e0 = kseg + blk * 256 + 64 * g + 16 * h;
    const U4 alo = ldg16(a.qs + e0), ahi = ldg16(a.qs + e0 + 32);
    const int sl = 2 * g, sh = 2 * g + 1;
    int s0 = 0, s1 = 0;
#define QMM_Q5(W) \
    s0 = dp4a_ss((q.W & 0x0F0F0F0Fu) | (((qh.W >> sl) & 0x01010101u) << 4), alo.W, s0); \
    s1 = dp4a_ss(((q.W >> 4) & 0x0F0F0F0Fu) | (((qh.W >> sh) & 0x01010101u) << 4), ahi.W, s1);
    QMM_Q5(x) QMM_Q5(y) QMM_Q5(z) QMM_Q5(w)
#undef QMM_Q5
    const int kb = (kseg >> 8) + blk;
    const int bs0 = a.bsums[kb * 16 + 4 * g + h], bs1 = a.bsums[kb * 16 + 4 * g + 2 + h];
    const float da = a.d[kb];
    const float dw = half_bits_to_float((uint16_t)(hdr.x & 0xFFFFu)), dminw = half_bits_to_float((uint16_t)(hdr.x >> 16));
    return (dw * da) * (float)(sc0 * s0 + sc1 * s1) - (dminw * da) * (float)(mn0 * bs0 + mn1 * bs1);
}

template <> QMM_HD float unit_dot<T_Q6_K>(const uint8_t * seg, int u, int kseg, const ActCol & a) {
    const int blk = u >> 3, p = u & 7, h = p >> 2, lq = p & 3;
    const uint8_t * b = seg + blk * 210;               // ql[128] | qh[64] | scales[16] | d
    const U2 qa = ld8_a2(b + 64 * h + 8 * lq);         // ql[l], l = 8lq..8lq+7 : quarters 0 (low nibble), 2 (high)
    const U2 qb = ld8_a2(b + 64 * h + 32 + 8 * lq);    // ql[l+32]            : quarters 1 (low nibble), 3 (high)
    const U2 qh = ld8_a2(b + 128 + 32 * h + 8 * lq);   // 2 bits per quarter
    const int8_t * sc = reinterpret_cast<const int8_t *>(b + 192) + 8 * h + (lq >> 1);
    const int e0 = kseg + blk * 256 + 128 * h + 8 * lq;
    int tot = 0;
#define QMM_Q6(QTR, LO, SHIFTED)                                                                        \
    {                                                                                                   \
        const U2 av = ldg8(a.qs + e0 + 32 * QTR);                                                       \
        const uint32_t c0 = ((SHIFTED ? (LO.x >> 4) : LO.x) & 0x0F0F0F0Fu) | (((qh.x >> (2 * QTR)) & 0x03030303u) << 4); \
        const uint32_t c1 = ((SHIFTED ? (LO.y >> 4) : LO.y) & 0x0F0F0F0Fu) | (((qh.y >> (2 * QTR)) & 0x03030303u) << 4); \
        int s = dp4a_ss(c0, av.x, 0); s = dp4a_ss(c1, av.y, s);                                         \
        int sa = dp4a_ss(0x01010101u, av.x, 0); sa = dp4a_ss(0x01010101u, av.y, sa);                    \
        tot += (int)sc[2 * QTR] * (s - 32 * sa);                                                        \
    }
    QMM_Q6(0, qa, false) QMM_Q6(1, qb, false) QMM_Q6(2, qa, true) QMM_Q6(3, qb, true)
#undef QMM_Q6
    const int kb = (kseg >> 8) + blk;
    const float dw = half_bits_to_float(ld2(b + 208));
    return (dw * a.d[kb]) * (float)tot;
}

template <> QMM_HD float unit_dot<T_Q4_0>(const uint8_t * seg, int u, int kseg, const ActCol & a) {
    const uint8_t * b = seg + u * 18;                  // d | qs[16]: low nibble = elem j, high = elem j+16
    const U4 q = ld16_a2(b + 2);
    const int e0 = kseg + 32 * u;
    const U4 alo = ldg16(a.qs + e0), ahi = ldg16(a.qs + e0 + 16);
    int s = 0;
    s = dp4a_ss(q.x & 0x0F0F0F0Fu, alo.x, s); s = dp4a_ss((q.x >> 4) & 0x0F0F0F0Fu, ahi.x, s);
    s = dp4a_ss(q.y & 0x0F0F0F0Fu, alo.y, s); s = dp4a_ss((q.y >> 4) & 0x0F0F0F0Fu, ahi.y, s);
    s = dp4a_ss(q.z & 0x0F0F0F0Fu, alo.z, s); s = dp4a_ss((q.z >> 4) & 0x0F0F0F0Fu, ahi.z, s);
    s = dp4a_ss(q.w & 0x0F0F0F0Fu, alo.w, s); s = dp4a_ss((q.w >> 4) & 0x0F0F0F0Fu, ahi.w, s);
    const int kb = (kseg >> 5) + u;
    s -= 8 * (int)a.bsums[kb];
    return ((float)s * half_bits_to_float(ld2(b))) * a.d[kb];
}

template <> QMM_HD float unit_dot<T_Q8_0>(const uint8_t * seg, int u, int kseg, const ActCol & a) {
    const uint8_t * b = seg + u * 34;                  // d | qs[32]
    const U4 q0 = ld16_a2(b + 2), q1 = ld16_a2(b + 18);
    const int e0 = kseg + 32 * u;
    const U4 a0 = ldg16(a.qs + e0), a1 = ldg16(a.qs + e0 + 16);
    int s = 0;
    s = dp4a_ss(q0.x, a0.x, s); s = dp4a_ss(q0.y, a0.y, s); s = dp4a_ss(q0.z, a0.z, s); s = dp4a_ss(q0.w, a0.w, s);
    s = dp4a_ss(q1.x, a1.x, s); s = dp4a_ss(q1.y, a1.y, s); s = dp4a_ss(q1.z, a1.z, s); s = dp4a_ss(q1.w, a1.w, s);
    const int kb = (kseg >> 5) + u;
    return (float)s * (half_bits_to_float(ld2(b)) * a.d[kb]);
}

// ---------------------------------------------------------------- element-wise dequant (bit-exact spec)
// Value of element e (0 <= e < BE) of the block at b, computed with the reference's UNFUSED fp32 ops in its
// order (dequantize_row_*: ggml-quants.c:459-478,553-567,1529-1551,1731-1756,1939-1968).  The device build uses
// __fmul_rn/__fsub_rn so nvcc cannot contract d1*q - m1 into an FMA (SURVEY.md Appendix A).
QMM_HD float mul_rn(float x, float y) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(x, y);
#else
    volatile float r = x * y; return r;
#endif
}
QMM_HD float sub_rn(float x, float y) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(x, y);
#else
    volatile float r = x - y; return r;
#endif
}

QMM_HD float dequant_elem(int t, const uint8_t * b, int e) {
    if (t == T_Q4_0) {
        const int q = e < 16 ? (b[2 + e] & 0xF) : (b[2 + e - 16] >> 4);
        return mul_rn((float)(q - 8), half_bits_to_float((uint16_t)(b[0] | (b[1] << 8))));
    }
    if (t == T_Q8_0) {
        return mul_rn((float)(int8_t)b[2 + e], half_bits_to_float((uint16_t)(b[0] | (b[1] << 8))));
    }
    if (t == T_Q4_K || t == T_Q5_K) {
        const float d = half_bits_to_float((uint16_t)(b[0] | (b[1] << 8))), dmin = half_bits_to_float((uint16_t)(b[2] | (b[3] << 8)));
        const uint32_t s0 = (uint32_t)b[4] | (b[5] << 8) | (b[6] << 16) | ((uint32_t)b[7] << 24);
        const uint32_t s1 = (uint32_t)b[8] | (b[9] << 8) | (b[10] << 16) | ((uint32_t)b[11] << 24);
        const uint32_t s2 = (uint32_t)b[12] | (b[13] << 8) | (b[14] << 16) | ((uint32_t)b[15] << 24);
        int sc, mn; k4_scale_min(e >> 5, s0, s1, s2, sc, mn);
        const int g = e >> 6, l = e & 31, hi = (e >> 5) & 1;
        int q;
        if (t == T_Q4_K) { const uint8_t v = b[16 + 32 * g + l]; q = hi ? (v >> 4) : (v & 0xF); }
        else { const uint8_t v = b[48 + 32 * g + l]; q = (hi ? (v >> 4) : (v & 0xF)) + (((b[16 + l] >> (2 * g + hi)) & 1) ? 16 : 0); }
        return sub_rn(mul_rn(mul_rn(d, (float)sc), (float)q), mul_rn(dmin, (float)mn));
    }
    // Q6_K
    const int h = e >> 7, r = e & 127, qtr = r >> 5, l = r & 31;
    const uint8_t lo = b[64 * h + (qtr & 1) * 32 + l];
    const int nib = qtr < 2 ? (lo & 0xF) : (lo >> 4);
    const int hb = (b[128 + 32 * h + l] >> (2 * qtr)) & 3;
    const int q = (int)(int8_t)(nib | (hb << 4)) - 32;
    const float d = half_bits_to_float((uint16_t)(b[208] | (b[209] << 8)));
    return mul_rn(mul_rn(d, (float)(int8_t)b[192 + 8 * h + (l >> 4) + 2 * qtr]), (float)q);
}

}  // namespace qmm
