// decode_flow.cu -- batch-1 decode as ONE persistent DATAFLOW kernel per token.
//
// Replaces round 1's decode_mega.cu (grid barrier between phases: 196 phases x ~10 us, 0.25 of the HBM roofline).  What the
// round-1 trace showed (profiles/r01_mega_trace.md): a phase cost ~3.5 us of barrier + ~3 us of activation prologue on top of
// its weights' HBM time, the barrier's polls queued behind 150 KB/SM of weight prefetch, and while streaming an SM reached
// ~60 % of its HBM share because the block dot products read 2x more shared memory for the activations than for the weights.
//
// Design (one CTA per SM, 7 consumer warps + 1 producer warp, cooperative launch so that co-residency is guaranteed):
//
//   * NO grid barrier.  Every vector a phase produces is written as 64-bit slots (tag << 32 | f32 bits); a consumer polls
//     exactly the slots it needs until they carry  epoch + producer_phase + 1.  One L2 round trip replaces
//     store -> fence -> arrive -> poll -> load.  The epoch lives in device memory and grows by n_phases + 1 per launch, so
//     stale slots are never mistaken for fresh ones and nothing is ever reset (CUDA-graph replay safe).
//   * ONE weight stream per CTA for the whole token.  The producer warp walks the program ahead of the consumers and issues
//     cp.async.bulk copies into a ring of 18 x 9.5 KB slots (full/empty mbarriers); weights do not depend on activations,
//     so the stream crosses phase boundaries: while the consumers wait for a vector, the ring fills with the next phases'
//     rows (25 MB on chip = ~4 us of HBM time, more than a dependency hop costs).
//   * Activations live in REGISTERS.  A lane is bound to one 256-weight k-block of the activation for a whole phase
//     (K = 4096: lane l <-> block l % 16, two rows per warp step; K = 14336: two warps per row, 28 lanes each), so the
//     quantised activation block (64 words) is loaded once per phase and a block dot product reads only its 144..210
//     weight bytes from shared memory.
//   * The hidden state stays in shared memory (every CTA reads the whole vector anyway for the RMS_NORM), so the residual
//     add of attn_output / ffn_down needs no global load.
//   * Attention: head h is handled by CTA h (x nsplit parts for long contexts) as soon as ITS q/k/v rows are there.
//
// Arithmetic is that of the round-1 kernels (the CPU's Q8_K integers, exact integer block dots, fp32 combine), only the
// order of the fp32 row reduction differs.  Deterministic: every output element is produced by one fixed lane group in a
// fixed order, whatever the timing.
//
// Slot reuse: the pool of tagged slots is carved round-robin by the host (FlowBuilder).  Every mat-vec phase validates ALL of
// its input vector before it produces anything, so by the time any CTA produces the output of phase p + 2, every consumer of
// phase p's input has finished reading it; the pool holds several layers' worth of outputs, far more than that distance.
//
// All spin loops are bounded and __trap(): a lost producer must fail the launch, never hang the GPU.
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "decode_flow.cuh"
#include "gemv_blockdot.cuh"

namespace qmm {

namespace {

#ifndef FLOW_TP
#define FLOW_TP 0
#endif
constexpr int FL_NW = 7;                                   // consumer warps (7 + the producer = 256 threads: the full 255-register budget).  Tried:
                                                           // 9 warps (allocated like 12: 168 registers, spills); 8 consumer warps + a producer
                                                           // warpgroup with setmaxnreg 232 / 40 (550 bytes of spills; did not complete the 8B run
                                                           // and failed the small-model parity check on hardware, lease X: removed)
constexpr int FL_PROD_WARPS = 1;
constexpr int FL_NPAIR = FL_NW / 2;                       // warp pairs when a row is split over two warps (K > 8192)
constexpr int FL_CTHREADS = FL_NW * 32;
constexpr int FL_THREADS = FL_CTHREADS + 32 * FL_PROD_WARPS;   // + the producer warp(group)
#if defined(FLOW_AB_NSLOTS)
constexpr int FL_NSLOTS = FLOW_AB_NSLOTS;                  // (14 slots: the CTA fits the 196 KB shared-memory configuration and leaves 32 KB of L1 for the spills)
#else
constexpr int FL_NSLOTS = 18;
#endif
constexpr int FL_SLOT = 9728;                              // bytes per ring slot (multiple of 128)
constexpr int FL_MAXBLK = FLOW_MAX_K / 256;                // 64
constexpr int FL_PU = 5;                                   // activation blocks per warp and prologue pass
static_assert(FL_PU * FL_NW * 256 >= FLOW_MAX_NORM_K, "a fused RMS_NORM must fit one prologue pass");
constexpr int ACT_PITCH = 272;                             // bytes per quantised block in shared memory (skewed)
constexpr int FL_TK = 4 * FL_CTHREADS;                     // keys per attention tile
constexpr int FL_KG = FL_CTHREADS / 16;                    // key groups in the P.V pass

// shared memory map (bytes)
constexpr int OFF_BARS = 0;                                // full[NSLOTS], empty[NSLOTS]
constexpr int OFF_ACT  = 512;                              // qs: MAXBLK x 272 | bs16: MAXBLK x 32 | d: MAXBLK x 4      (aliased: attention scratch)
constexpr int ACT_BS   = FL_MAXBLK * ACT_PITCH;
constexpr int ACT_D    = ACT_BS + FL_MAXBLK * 32;
constexpr int ACT_BYTES = ACT_D + FL_MAXBLK * 4;           // 19712
constexpr int ATT_Q = 0, ATT_K = 256, ATT_V = 512, ATT_TH = 768, ATT_S = 1024, ATT_PV = ATT_S + FL_TK;   // float indices
constexpr int ATT_FLOATS = ATT_PV + FL_KG * 128;
static_assert(ATT_FLOATS * 4 <= ACT_BYTES, "attention scratch must fit the activation area");
constexpr int OFF_RED  = OFF_ACT + ACT_BYTES;              // 64 doubles
constexpr int OFF_PART = OFF_RED + 512;                    // 2 x FLOW_PART_ROWS floats
constexpr int DESC_WORDS = (int)(sizeof(FlowPhase) / 4);
static_assert(sizeof(FlowPhase) % 16 == 0 && sizeof(FlowPhase) <= 384, "FlowPhase is staged in shared memory as 16-byte words");
constexpr int OFF_DESC = OFF_PART + 2 * FLOW_PART_ROWS * 4;  // 2 x FlowPhase for the consumers + 2 x FlowPhase for the producer
constexpr int OFF_H    = OFF_DESC + 4 * 384;
constexpr int OFF_RING = (OFF_H + FLOW_MAX_H * 4 + 127) / 128 * 128;
constexpr int FL_SMEM  = OFF_RING + FL_NSLOTS * FL_SLOT;
static_assert(FL_SMEM <= 227 * 1024, "decode_flow shared memory");
static_assert(2 * FL_NSLOTS * 8 <= OFF_ACT, "mbarrier area");

// ------------------------------------------------------------------------------------------------ small PTX helpers
__device__ __forceinline__ void bar_consumers() { asm volatile("bar.sync 1, %0;\n" ::"n"(FL_CTHREADS) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint64_t ld_slot(const uint64_t * p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void ld_slot2(const uint64_t * p, uint64_t & a, uint64_t & b) {
    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];\n" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ void st_slot(uint64_t * p, uint32_t tag, float v) {
    const uint64_t w = ((uint64_t)tag << 32) | (uint64_t)__float_as_uint(v);
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;\n" ::"l"(p), "l"(w) : "memory");
}
// Bounded waits: a lost producer (or a missing bulk copy) must fail the launch, never hang the GPU.  Wall-clock bound (globaltimer,
// checked every 256 polls): 4 s is ~3 orders of magnitude above a whole token.
__device__ __forceinline__ unsigned long long gtime() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
    return t;
}
__device__ __forceinline__ void spin_fail(long long & spins) {
    if (++spins > (1ll << 23)) __trap();                     // every poll is an L2 round trip: seconds
}
__device__ __forceinline__ void fl_mbar_wait(uint64_t * bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const unsigned long long t0 = gtime();
    int n = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++n & 63) == 0 && gtime() - t0 > 4000000000ull) __trap();
    }
}
// Tags are relative to an epoch that lives in device memory and only grows.  Single GPU: one epoch (phases of this launch).  The
// tensor-parallel build (FLOW_TP, decode_flow_tp.cu) adds the collective epoch of the GPU group for vectors written by peers.
#if FLOW_TP
struct EpochT { uint32_t phase, coll; };
__device__ __forceinline__ uint32_t want_tag(const FlowVec & v, const EpochT & ep) { return ((v.flags & FLOW_VEC_COLL) ? ep.coll : ep.phase) + v.tag; }
__device__ __forceinline__ uint32_t phase_epoch(const EpochT & ep) { return ep.phase; }
__device__ __forceinline__ void st_slot_sys(uint64_t * p, uint32_t tag, float v) {       // a peer GPU's memory, over NVLink
    const uint64_t w = ((uint64_t)tag << 32) | (uint64_t)__float_as_uint(v);
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(p), "l"(w) : "memory");
}
#else
typedef uint32_t EpochT;
__device__ __forceinline__ uint32_t want_tag(const FlowVec & v, EpochT ep) { return ep + v.tag; }
__device__ __forceinline__ uint32_t phase_epoch(EpochT ep) { return ep; }
#endif
// one element of a vector (polls while the producer has not written it)
__device__ __forceinline__ float vec_ld(const FlowVec & v, int i, EpochT epoch) {
    if (v.ll != nullptr) {
        const uint32_t want = want_tag(v, epoch);
        long long spins = 0;
        uint64_t w = ld_slot(v.ll + i);
        while ((uint32_t)(w >> 32) != want) { spin_fail(spins); w = ld_slot(v.ll + i); }
        return __uint_as_float((uint32_t)w);
    }
    return __ldcg(v.plain + i);
}
// one element in two steps, so that several independent loads can be in flight before the first one is waited for
__device__ __forceinline__ uint64_t vec_peek(const FlowVec & v, int i) {
    return v.ll != nullptr ? ld_slot(v.ll + i) : (uint64_t)__float_as_uint(__ldcg(v.plain + i));
}
__device__ __forceinline__ float vec_resolve(const FlowVec & v, int i, EpochT epoch, uint64_t w) {
    if (v.ll != nullptr) {
        const uint32_t want = want_tag(v, epoch);
        long long spins = 0;
        while ((uint32_t)(w >> 32) != want) { spin_fail(spins); w = ld_slot(v.ll + i); }
    }
    return __uint_as_float((uint32_t)w);
}
__device__ __forceinline__ void out_st(const FlowOut & o, int i, uint32_t tag, float v) {
    if (o.ll != nullptr) st_slot(o.ll + i, tag, v);
    if (o.plain != nullptr) o.plain[i] = v;
}
// 8 consecutive elements (i multiple of 8).  Tagged slots: all four 16-byte loads go out together, then whatever is not there yet
// is polled.
__device__ __forceinline__ void vec_ld8_issue(const FlowVec & v, int i, uint64_t (&raw)[8]) {
    if (v.ll != nullptr) {
#pragma unroll
        for (int c = 0; c < 4; c++) ld_slot2(v.ll + i + 2 * c, raw[2 * c], raw[2 * c + 1]);
    } else {
        const float4 a = __ldcg(reinterpret_cast<const float4 *>(v.plain + i)), b = __ldcg(reinterpret_cast<const float4 *>(v.plain + i) + 1);
        raw[0] = __float_as_uint(a.x); raw[1] = __float_as_uint(a.y); raw[2] = __float_as_uint(a.z); raw[3] = __float_as_uint(a.w);
        raw[4] = __float_as_uint(b.x); raw[5] = __float_as_uint(b.y); raw[6] = __float_as_uint(b.z); raw[7] = __float_as_uint(b.w);
    }
}
__device__ __forceinline__ void vec_ld8_finish(const FlowVec & v, int i, EpochT epoch, uint64_t (&raw)[8], float (&x)[8]) {
    if (v.ll != nullptr) {
        const uint32_t want = want_tag(v, epoch);
        long long spins = 0;
#pragma unroll
        for (int c = 0; c < 4; c++) {
            while ((uint32_t)(raw[2 * c] >> 32) != want || (uint32_t)(raw[2 * c + 1] >> 32) != want) {
                spin_fail(spins);
                ld_slot2(v.ll + i + 2 * c, raw[2 * c], raw[2 * c + 1]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 8; c++) x[c] = __uint_as_float((uint32_t)raw[c]);
}

// NU blocks of 8 consecutive elements per lane (the mat-vec prologue), loads already issued by vec_ld8_issue.  What the phase trace
// showed (profiles/r02_flow_trace.md): a consumer that arrives before its producers finds EVERY first load stale, and re-polling the
// chunks one after the other costs one L2 round trip per chunk AFTER the data has landed (up to 20 in a row: 6 - 14 us per hop).
// Re-polling everything that is stale in every round floods the L2 while CTAs wait for a slow producer (lease J: -26 %).  So: spin on ONE
// chunk (one load in flight per lane, as before) until it is valid -- the producers of a vector finish within a microsecond or two of
// each other -- and only then re-load all the other stale chunks together, round after round, until none is left.
template <int NU>
__device__ __forceinline__ void vec_ld8_finish_blocks(const FlowVec & v, const int (&idx)[NU], const bool (&on)[NU], EpochT epoch, uint64_t (&raw)[NU][8], float (&x)[NU][8], unsigned long long * t_first = nullptr) {
    (void)t_first;
    if (v.ll != nullptr) {
        const uint32_t want = want_tag(v, epoch);
        long long spins = 0;
#if defined(FLOW_AB_SEQ_POLL)
#pragma unroll
        for (int u = 0; u < NU; u++) {
            if (!on[u]) continue;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                while ((uint32_t)(raw[u][2 * c] >> 32) != want || (uint32_t)(raw[u][2 * c + 1] >> 32) != want) {
                    spin_fail(spins);
                    ld_slot2(v.ll + idx[u] + 2 * c, raw[u][2 * c], raw[u][2 * c + 1]);
                }
            }
        }
#else
        if (on[0]) {                                                  // (block 0 of a pass exists for every warp that has any block in it)
            while ((uint32_t)(raw[0][0] >> 32) != want || (uint32_t)(raw[0][1] >> 32) != want) {
                spin_fail(spins);
                ld_slot2(v.ll + idx[0], raw[0][0], raw[0][1]);
            }
        }
#if defined(FLOW_FINE_TRACE)
        if (t_first != nullptr) *t_first = gtime();
#endif
        for (;;) {
            bool stale = false;
#pragma unroll
            for (int u = 0; u < NU; u++) {
                if (!on[u]) continue;
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    if ((uint32_t)(raw[u][2 * c] >> 32) != want || (uint32_t)(raw[u][2 * c + 1] >> 32) != want) {
                        ld_slot2(v.ll + idx[u] + 2 * c, raw[u][2 * c], raw[u][2 * c + 1]);
                        stale = true;
                    }
                }
            }
            if (!stale) break;
            spin_fail(spins);
        }
#endif
    }
#pragma unroll
    for (int u = 0; u < NU; u++) {
#pragma unroll
        for (int c = 0; c < 8; c++) x[u][c] = __uint_as_float((uint32_t)raw[u][c]);
    }
}

// out[i..i+8) = a[i..i+8) (+ b[i..i+8)): the tiny one-CTA phases (n is a multiple of 8 or the tail is done element-wise)
__device__ __forceinline__ void vec_copy8(const FlowVec & a, const FlowVec & b, bool add, const FlowOut & o, int i, int n, uint32_t tag, EpochT epoch) {
    if (i + 8 <= n && (i & 7) == 0) {
        uint64_t ra[8], rb[8];
        float xa[8], xb[8];
        vec_ld8_issue(a, i, ra);
        if (add) vec_ld8_issue(b, i, rb);
        vec_ld8_finish(a, i, epoch, ra, xa);
        if (add) vec_ld8_finish(b, i, epoch, rb, xb);
#pragma unroll
        for (int k = 0; k < 8; k++) out_st(o, i + k, tag, add ? __fadd_rn(xa[k], xb[k]) : xa[k]);
    } else {
        for (int k = i; k < n && k < i + 8; k++) out_st(o, k, tag, add ? __fadd_rn(vec_ld(a, k, epoch), vec_ld(b, k, epoch)) : vec_ld(a, k, epoch));
    }
}

// ------------------------------------------------------------------------------------------------ block dot products, activation in registers
// a[64]: the lane's 256 int8 activations (word i = elements 4i..4i+3); bs16[8]: 16 x int16 sums of 16; bs32[4]: 8 x int16 sums of 32.
template <int T> struct RegDot;

template <> struct RegDot<T_Q4_K> {
    __device__ __forceinline__ static float run(const uint8_t * wb, const uint32_t (&a)[64], const uint32_t (&bs16)[8], const uint32_t (&bs32)[4], float da) {
        const uint4 hdr = lds128(wb);
        // 6-bit scales/mins -> 2 x 4 packed bytes each (the reference's utmp shuffle, ggml-cpu/quants.c:726-731)
        const uint32_t sc_lo = hdr.y & 0x3f3f3f3fu, mn_lo = hdr.z & 0x3f3f3f3fu;
        const uint32_t sc_hi = (hdr.w & 0x0f0f0f0fu) | (((hdr.y >> 6) & 0x03030303u) << 4);
        const uint32_t mn_hi = ((hdr.w >> 4) & 0x0f0f0f0fu) | (((hdr.z >> 6) & 0x03030303u) << 4);
        int tot = 0;
#pragma unroll
        for (int g = 0; g < 4; g++) {                       // 64 weights: qs[32g..32g+32) low nibbles -> sub-block 2g, high -> 2g+1
            const uint4 q0 = lds128(wb + 16 + 32 * g), q1 = lds128(wb + 32 + 32 * g);
            const uint32_t qw[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
            int sl = 0, sh = 0, sl2 = 0, sh2 = 0;
#pragma unroll
            for (int i = 0; i < 8; i += 2) {
                sl  = __dp4a((int)(qw[i] & 0x0F0F0F0Fu), (int)a[16 * g + i], sl);
                sh  = dp4a_us(qw[i] & 0xF0F0F0F0u, a[16 * g + 8 + i], sh);
                sl2 = __dp4a((int)(qw[i + 1] & 0x0F0F0F0Fu), (int)a[16 * g + i + 1], sl2);
                sh2 = dp4a_us(qw[i + 1] & 0xF0F0F0F0u, a[16 * g + 8 + i + 1], sh2);
            }
            sl += sl2; sh += sh2;
            const uint32_t scw = g < 2 ? sc_lo : sc_hi;
            const int s0 = (int)((scw >> (16 * (g & 1))) & 0xFFu), s1 = (int)((scw >> (16 * (g & 1) + 8)) & 0xFFu);
            tot += s0 * sl + s1 * (sh >> 4);                // sh is an exact multiple of 16
        }
        int mins = 0;
        mins = __dp2a_lo((int)bs32[0], (int)mn_lo, mins); mins = __dp2a_hi((int)bs32[1], (int)mn_lo, mins);
        mins = __dp2a_lo((int)bs32[2], (int)mn_hi, mins); mins = __dp2a_hi((int)bs32[3], (int)mn_hi, mins);
        const float dw = __half2float(__ushort_as_half((unsigned short)(hdr.x & 0xFFFFu)));
        const float dm = __half2float(__ushort_as_half((unsigned short)(hdr.x >> 16)));
        (void)bs16;
        return (dw * da) * (float)tot - (dm * da) * (float)mins;
    }
};

template <> struct RegDot<T_Q5_K> {
    __device__ __forceinline__ static float run(const uint8_t * wb, const uint32_t (&a)[64], const uint32_t (&bs16)[8], const uint32_t (&bs32)[4], float da) {
        const uint4 hdr = lds128(wb);
        const uint4 h0 = lds128(wb + 16), h1 = lds128(wb + 32);      // qh[l], l = 0..15 / 16..31
        const uint32_t hw[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
        const uint32_t sc_lo = hdr.y & 0x3f3f3f3fu, mn_lo = hdr.z & 0x3f3f3f3fu;
        const uint32_t sc_hi = (hdr.w & 0x0f0f0f0fu) | (((hdr.y >> 6) & 0x03030303u) << 4);
        const uint32_t mn_hi = ((hdr.w >> 4) & 0x0f0f0f0fu) | (((hdr.z >> 6) & 0x03030303u) << 4);
        int tot = 0;
#pragma unroll
        for (int g = 0; g < 4; g++) {
            const uint4 q0 = lds128(wb + 48 + 32 * g), q1 = lds128(wb + 64 + 32 * g);
            const uint32_t qw[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
            int sl = 0, sh = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) {                   // bit 2g of qh[l] is the 5th bit of low-nibble element l, bit 2g+1 of the high-nibble element
                sl = __dp4a((int)((qw[i] & 0x0F0F0F0Fu) | (((hw[i] >> (2 * g)) & 0x01010101u) << 4)), (int)a[16 * g + i], sl);
                sh = __dp4a((int)(((qw[i] >> 4) & 0x0F0F0F0Fu) | (((hw[i] >> (2 * g + 1)) & 0x01010101u) << 4)), (int)a[16 * g + 8 + i], sh);
            }
            const uint32_t scw = g < 2 ? sc_lo : sc_hi;
            const int s0 = (int)((scw >> (16 * (g & 1))) & 0xFFu), s1 = (int)((scw >> (16 * (g & 1) + 8)) & 0xFFu);
            tot += s0 * sl + s1 * sh;
        }
        int mins = 0;
        mins = __dp2a_lo((int)bs32[0], (int)mn_lo, mins); mins = __dp2a_hi((int)bs32[1], (int)mn_lo, mins);
        mins = __dp2a_lo((int)bs32[2], (int)mn_hi, mins); mins = __dp2a_hi((int)bs32[3], (int)mn_hi, mins);
        const float dw = __half2float(__ushort_as_half((unsigned short)(hdr.x & 0xFFFFu)));
        const float dm = __half2float(__ushort_as_half((unsigned short)(hdr.x >> 16)));
        (void)bs16;
        return (dw * da) * (float)tot - (dm * da) * (float)mins;
    }
};

template <> struct RegDot<T_Q6_K> {
    // ql[128] | qh[64] | scales[16] | d : 210 B, only 2-byte aligned -> aligned word reads + funnel shift
    __device__ __forceinline__ static float run(const uint8_t * wb, const uint32_t (&a)[64], const uint32_t (&bs16)[8], const uint32_t (&bs32)[4], float da) {
        const uint32_t * w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(wb) & ~uintptr_t(3));
        const uint32_t fs = (uint32_t)(reinterpret_cast<uintptr_t>(wb) & 2) * 8;
        int tot = 0;
        uint32_t scw[4];                                             // scales: bytes 192..207 = words 48..51
        {
            uint32_t p = w[48];
#pragma unroll
            for (int i = 0; i < 4; i++) { const uint32_t n = w[49 + i]; scw[i] = __funnelshift_r(p, n, fs); p = n; }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {                                // 128 weights per half
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
                int s_lo = 0, s_hi = 0;                              // l < 16 and l >= 16 use different scales
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const uint32_t lo = ql[(qtr & 1) * 8 + i];
                    const uint32_t nib = (qtr < 2 ? lo : (lo >> 4)) & 0x0F0F0F0Fu;
                    const uint32_t c = nib | (((qh[i] >> (2 * qtr)) & 0x03030303u) << 4);   // 0..63
                    const uint32_t av = a[32 * h + 8 * qtr + i];
                    if (i < 4) s_lo = __dp4a((int)c, (int)av, s_lo); else s_hi = __dp4a((int)c, (int)av, s_hi);
                }
                // scale index 8h + 2qtr (+1 for l >= 16); (q - 32): subtract 32 * bsum of the same 16 activations
                const int si = 8 * h + 2 * qtr;
                const int sc0 = (int)(int8_t)((scw[si >> 2] >> (8 * (si & 3))) & 0xFFu);
                const int sc1 = (int)(int8_t)((scw[(si + 1) >> 2] >> (8 * ((si + 1) & 3))) & 0xFFu);
                const uint32_t bw = bs16[si >> 1];                   // bsums[si], bsums[si+1]
                const int bsum0 = (int)(int16_t)(bw & 0xFFFFu), bsum1 = (int)(int16_t)(bw >> 16);
                tot += sc0 * (s_lo - 32 * bsum0) + sc1 * (s_hi - 32 * bsum1);
            }
        }
        const float dw = __half2float(__ushort_as_half(*reinterpret_cast<const unsigned short *>(wb + 208)));
        (void)bs32;
        return (dw * da) * (float)tot;
    }
};

// ------------------------------------------------------------------------------------------------ geometry shared by producer and consumers
// first row of CTA `cta` of matrix m: the host planned rq = M / grid rows per CTA and gives the first rr = M % grid CTAs one more
__device__ __forceinline__ int row_begin(const FlowMatvec & p, int m, int cta) { const int r = p.rr[m]; return cta * p.rq[m] + (cta < r ? cta : r); }

struct PieceGeom {
    int nblk, contiguous[3], row_bytes[3], sub;
};

__device__ __forceinline__ int seg_len(const FlowMatvec & p, int nblk, int s) { const int l = nblk - s * p.seg; return l < p.seg ? l : p.seg; }

// bytes layout of a piece inside its slot: sub-piece j (SwiGLU: 0 gate, 1 up), row r
//   contiguous (one k-segment, dense rows): one copy per sub-piece, pitch sub_pitch
//   otherwise: one copy per (j, r), pitch row_pitch
__device__ __forceinline__ int sub_pitch(int R, int row_bytes) { return (R * row_bytes + 16 + 15) & ~15; }
__device__ __forceinline__ int row_pitch(int seg, int bb) { return (seg * bb + 16 + 15) & ~15; }

// Which consumer warp takes piece q of a phase.  One k-segment per row: round robin, q % 7.  Two segments (K > 8192): piece q = (chunk,
// s); a warp is bound to one segment for the whole phase (its lanes hold that segment's activation blocks), so six warps form three
// pairs -- warp 2 (chunk % 3) + s -- and the seventh idles.  (consume_matrix walks exactly these.)

// ------------------------------------------------------------------------------------------------ producer warp
// The phase descriptors live in global memory; every field read behind an mbarrier wait ("memory" clobber) would be re-fetched
// from L2 (the L1 is tiny next to 227 KB of shared memory and is swept by the activation polls): the first hardware run spent
// ~700 cycles per 7 KB piece on that.  So the producer keeps the descriptor of its current mat-vec phase in shared memory (its
// own two slots) and fetches the next one while it issues the current phase's copies.
__device__ __forceinline__ int next_matvec(const FlowPhase * __restrict__ ph, int from, int n_phases) {
    while (from < n_phases && __ldg(&ph[from].kind) != FLOW_MATVEC) from++;
    return from;
}
#if defined(FLOW_AB_SERIAL_PRODUCER)
__device__ __forceinline__ void producer_loop(const FlowPhase * __restrict__ ph, int n_phases, uint8_t * smem, int lane, int throttle) {
    uint64_t * full = reinterpret_cast<uint64_t *>(smem + OFF_BARS), * empty = full + FL_NSLOTS;
    uint8_t * ring = smem + OFF_RING;
    uint32_t * pdesc = reinterpret_cast<uint32_t *>(smem + OFF_DESC + 2 * 384);
    const int cta = (int)blockIdx.x, grid = (int)gridDim.x;
    unsigned g = 0;                                                  // pieces issued so far (this CTA, whole program)
    int pi = next_matvec(ph, 0, n_phases), buf = 0;
    if (pi < n_phases) {
        const uint32_t * src = reinterpret_cast<const uint32_t *>(ph + pi);
        for (int i = lane; i < DESC_WORDS; i += 32) pdesc[i] = __ldg(src + i);
    }
    __syncwarp();
    while (pi < n_phases) {
        const int pn = next_matvec(ph, pi + 1, n_phases);
        uint32_t nxt[(DESC_WORDS + 31) / 32];
        if (pn < n_phases) {
            const uint32_t * src = reinterpret_cast<const uint32_t *>(ph + pn);
#pragma unroll
            for (int i = 0; i < (DESC_WORDS + 31) / 32; i++) if (lane + 32 * i < DESC_WORDS) nxt[i] = __ldg(src + lane + 32 * i);
        }
        const FlowMatvec & p = reinterpret_cast<const FlowPhase *>(pdesc + buf * 96)->mv;
        const int nblk = p.K >> 8, S = p.S, seg = p.seg;
        const int nenum = p.mode == 2 ? 1 : p.nmat, sub = p.mode == 2 ? 2 : 1;
        for (int m = 0; m < nenum; m++) {
            // per-matrix constants in registers (the piece loop below must be lean: it has to stay ahead of 7 consumer warps)
            const int Mm = p.M[m], R = p.R[m], bb = block_bytes(p.type[m]);
            const int rb = row_begin(p, m, cta), re = row_begin(p, m, cta + 1);
            const int row_bytes = nblk * bb;
            const uint8_t * w0 = p.w[m], * w1 = p.w[1];
            const int64_t rs0 = p.row_stride[m], rs1 = p.row_stride[1];
            const bool contiguous = S == 1 && rs0 == (int64_t)row_bytes && (sub == 1 || rs1 == (int64_t)row_bytes);
            const int spitch = sub_pitch(R, row_bytes), rpitch = row_pitch(seg, bb);
            for (int r0 = rb; r0 < re; r0 += R) {
                const int nr = min(R, re - r0);
                // the piece is one or a few contiguous runs (dense rows: one per sub-piece; otherwise one per row segment); lane rj
                // copies run rj.  (Cutting runs into smaller chunks issued side by side was measured and is slower: 268 tok/s at
                // 1 KB chunks, 296 at 4 KB, 343 unchunked -- the copy engine prefers few large copies.)
                const int nruns = contiguous ? sub : sub * nr;
                for (int sgm = 0; sgm < S; sgm++) {
                    const unsigned slot = g % FL_NSLOTS, use = g / FL_NSLOTS;
                    if (use > 0) fl_mbar_wait(empty + slot, (use - 1) & 1u);
                    if (throttle > 0 && g >= (unsigned)throttle) {   // at most `throttle` pieces in flight: keeps the SM's memory queue short
                        const unsigned og = g - (unsigned)throttle;
                        fl_mbar_wait(full + og % FL_NSLOTS, (og / FL_NSLOTS) & 1u);
                    }
                    uint8_t * sl = ring + (size_t)slot * FL_SLOT;
                    const uint8_t * src = nullptr;
                    uint8_t * dst = nullptr;
                    uint32_t cnt = 0;
                    if (lane < nruns) {
                        const uint8_t * gp;
                        uint32_t total;
                        if (contiguous) {
                            gp = (sub == 2 && lane == 1 ? w1 : w0) + (int64_t)r0 * (sub == 2 && lane == 1 ? rs1 : rs0);
                            dst = sl + lane * spitch;
                            total = (uint32_t)(nr * row_bytes);
                        } else {
                            const int j = lane >= nr ? 1 : 0, r = lane - j * nr;
                            gp = (sub == 2 && j ? w1 : w0) + (int64_t)(r0 + r) * (sub == 2 && j ? rs1 : rs0) + (int64_t)sgm * seg * bb;
                            dst = sl + (j * R + r) * rpitch;
                            total = (uint32_t)(seg_len(p, nblk, sgm) * bb);
                        }
                        const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(gp) & 15);
                        cnt = (off + total + 15u) & ~15u;
                        src = gp - off;
                    }
                    uint32_t tx = cnt;
                    if (nruns <= 2) {
                        tx += __shfl_xor_sync(0xffffffffu, tx, 1);
                    } else {
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) tx += __shfl_xor_sync(0xffffffffu, tx, o);
                    }
                    if (lane == 0) mbar_expect_tx(full + slot, tx);
                    __syncwarp();
                    if (cnt) bulk_g2s(dst, src, cnt, full + slot);
                    g++;
                }
            }
        }
        // hand over to the next mat-vec phase: its descriptor has long arrived
        if (pn < n_phases) {
#pragma unroll
            for (int i = 0; i < (DESC_WORDS + 31) / 32; i++) if (lane + 32 * i < DESC_WORDS) pdesc[(buf ^ 1) * 96 + lane + 32 * i] = nxt[i];
        }
        __syncwarp();
        buf ^= 1;
        pi = pn;
    }
}

#else
// What the trace and the bulk-copy micro-benchmark showed together (profiles/r02_flow_trace.md, r02_ubench.md): one lane streaming 9 KB
// copies saturates HBM, yet every mat-vec phase advanced at one ring piece per ~560 - 710 cycles whatever the piece size (Q6_K pieces of
// 6.7 KB: 2.7 TB/s, Q4_K pieces of 9.2 KB: 3.8 - 4.6 TB/s).  That is the latency of ONE trip through the serial producer loop (barrier
// wait, address arithmetic, shuffles, expect_tx, copy).  So FL_PL lanes now walk FL_PL consecutive pieces side by side: each lane
// decodes its own piece (matrix, row chunk, k-segment), waits for its own slot and issues that piece's copies itself.  The numbering of
// the pieces (matrix-major, then row chunk, then segment) is unchanged, so the consumers need no change.
#if defined(FLOW_AB_PL)
constexpr int FL_PL = FLOW_AB_PL;
#else
constexpr int FL_PL = 8;
#endif
__device__ __forceinline__ void producer_loop(const FlowPhase * __restrict__ ph, int n_phases, uint8_t * smem, int lane, int throttle) {
    (void)throttle;
    uint64_t * full = reinterpret_cast<uint64_t *>(smem + OFF_BARS), * empty = full + FL_NSLOTS;
    uint8_t * ring = smem + OFF_RING;
    uint32_t * pdesc = reinterpret_cast<uint32_t *>(smem + OFF_DESC + 2 * 384);
    const int cta = (int)blockIdx.x, grid = (int)gridDim.x;
    unsigned gbase = 0;                                              // pieces of the phases before the current one (this CTA)
    int pi = next_matvec(ph, 0, n_phases), buf = 0;
    if (pi < n_phases) {
        const uint32_t * src = reinterpret_cast<const uint32_t *>(ph + pi);
        for (int i = lane; i < DESC_WORDS; i += 32) pdesc[i] = __ldg(src + i);
    }
    __syncwarp();
    while (pi < n_phases) {
        const int pn = next_matvec(ph, pi + 1, n_phases);
        uint32_t nxt[(DESC_WORDS + 31) / 32];
        if (pn < n_phases) {
            const uint32_t * src = reinterpret_cast<const uint32_t *>(ph + pn);
#pragma unroll
            for (int i = 0; i < (DESC_WORDS + 31) / 32; i++) if (lane + 32 * i < DESC_WORDS) nxt[i] = __ldg(src + lane + 32 * i);
        }
        const FlowMatvec & p = reinterpret_cast<const FlowPhase *>(pdesc + buf * 96)->mv;
        const int nblk = p.K >> 8, S = p.S, seg = p.seg;
        const int nenum = p.mode == 2 ? 1 : p.nmat, sub = p.mode == 2 ? 2 : 1;
        // this CTA's rows and piece count per matrix (warp-uniform)
        int rb0 = 0, re0 = 0, rb1 = 0, re1 = 0, rb2 = 0, re2 = 0, n0 = 0, n1 = 0, n2 = 0;
        rb0 = row_begin(p, 0, cta); re0 = row_begin(p, 0, cta + 1); n0 = (re0 - rb0 + p.R[0] - 1) / p.R[0] * S;
        if (nenum > 1) { rb1 = row_begin(p, 1, cta); re1 = row_begin(p, 1, cta + 1); n1 = (re1 - rb1 + p.R[1] - 1) / p.R[1] * S; }
        if (nenum > 2) { rb2 = row_begin(p, 2, cta); re2 = row_begin(p, 2, cta + 1); n2 = (re2 - rb2 + p.R[2] - 1) / p.R[2] * S; }
        const int P = n0 + n1 + n2;
        for (int q0 = 0; q0 < P; q0 += FL_PL) {
            const int q = q0 + lane;
            if (lane < FL_PL && q < P) {
                const int m = q < n0 ? 0 : (q < n0 + n1 ? 1 : 2);
                const int t = q - (m == 0 ? 0 : (m == 1 ? n0 : n0 + n1));
                const int rb = m == 0 ? rb0 : (m == 1 ? rb1 : rb2), re = m == 0 ? re0 : (m == 1 ? re1 : re2);
                const int R = p.R[m], bb = block_bytes(p.type[m]);
                const int ch = S == 1 ? t : t >> 1, sgm = S == 1 ? 0 : (t & 1);
                const int r0 = rb + ch * R, nr = min(R, re - r0);
                const int row_bytes = nblk * bb;
                const uint8_t * w0 = p.w[m], * w1 = p.w[1];
                const int64_t rs0 = p.row_stride[m], rs1 = p.row_stride[1];
                const bool contiguous = S == 1 && rs0 == (int64_t)row_bytes && (sub == 1 || rs1 == (int64_t)row_bytes);
                const unsigned g = gbase + (unsigned)q, slot = g % FL_NSLOTS, use = g / FL_NSLOTS;
                if (use > 0) fl_mbar_wait(empty + slot, (use - 1) & 1u);
                uint8_t * sl = ring + (size_t)slot * FL_SLOT;
                if (contiguous) {
                    // dense rows: one copy per sub-piece (SwiGLU: gate rows, up rows)
                    const uint8_t * g0 = w0 + (int64_t)r0 * rs0, * g1 = w1 + (int64_t)r0 * rs1;
                    const uint32_t total = (uint32_t)(nr * row_bytes);
                    const uint32_t off0 = (uint32_t)(reinterpret_cast<uintptr_t>(g0) & 15), off1 = (uint32_t)(reinterpret_cast<uintptr_t>(g1) & 15);
                    const uint32_t c0 = (off0 + total + 15u) & ~15u, c1 = sub == 2 ? ((off1 + total + 15u) & ~15u) : 0u;
                    mbar_expect_tx(full + slot, c0 + c1);
                    bulk_g2s(sl, g0 - off0, c0, full + slot);
                    if (sub == 2) bulk_g2s(sl + sub_pitch(R, row_bytes), g1 - off1, c1, full + slot);
                } else {
                    // one copy per (sub-piece, row): this segment's blocks of the row
                    const int rpitch = row_pitch(seg, bb);
                    const uint32_t total = (uint32_t)(seg_len(p, nblk, sgm) * bb);
                    const int64_t koff = (int64_t)sgm * seg * bb;
                    uint32_t tx = 0;
                    for (int j = 0; j < sub; j++)
                        for (int r = 0; r < nr; r++) {
                            const uint8_t * gp = (j ? w1 : w0) + (int64_t)(r0 + r) * (j ? rs1 : rs0) + koff;
                            tx += ((uint32_t)(reinterpret_cast<uintptr_t>(gp) & 15) + total + 15u) & ~15u;
                        }
                    mbar_expect_tx(full + slot, tx);
                    for (int j = 0; j < sub; j++)
                        for (int r = 0; r < nr; r++) {
                            const uint8_t * gp = (j ? w1 : w0) + (int64_t)(r0 + r) * (j ? rs1 : rs0) + koff;
                            const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(gp) & 15);
                            bulk_g2s(sl + (j * R + r) * rpitch, gp - off, (off + total + 15u) & ~15u, full + slot);
                        }
                }
            }
            __syncwarp();
        }
        gbase += (unsigned)P;
        // hand over to the next mat-vec phase: its descriptor has long arrived
        if (pn < n_phases) {
#pragma unroll
            for (int i = 0; i < (DESC_WORDS + 31) / 32; i++) if (lane + 32 * i < DESC_WORDS) pdesc[(buf ^ 1) * 96 + lane + 32 * i] = nxt[i];
        }
        __syncwarp();
        buf ^= 1;
        pi = pn;
    }
}
#endif

// ------------------------------------------------------------------------------------------------ Q8_K quantisation of one 256-block held by a warp
// quantize_row_q8_K_ref (ggml-quants.c:2768-2805): lane l holds elements 8l..8l+7; the FIRST element of largest magnitude decides
// scale and sign.  Writes the int8 values (skewed pitch), the 16 sums of 16 and the scale to shared memory.
__device__ __forceinline__ void quant_block(const float (&v)[8], int b, int lane, uint8_t * act) {
    unsigned mloc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) { const unsigned a = (v[i] == v[i]) ? (__float_as_uint(v[i]) & 0x7fffffffu) : 0u; mloc = a > mloc ? a : mloc; }
    const unsigned mall = __reduce_max_sync(0xffffffffu, mloc);
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
    uint2 packed;
    packed.x = (uint32_t)(q[0] & 0xFF) | ((uint32_t)(q[1] & 0xFF) << 8) | ((uint32_t)(q[2] & 0xFF) << 16) | ((uint32_t)(q[3] & 0xFF) << 24);
    packed.y = (uint32_t)(q[4] & 0xFF) | ((uint32_t)(q[5] & 0xFF) << 8) | ((uint32_t)(q[6] & 0xFF) << 16) | ((uint32_t)(q[7] & 0xFF) << 24);
    *reinterpret_cast<uint2 *>(act + (size_t)b * ACT_PITCH + 8 * lane) = packed;
    const int s8 = q[0] + q[1] + q[2] + q[3] + q[4] + q[5] + q[6] + q[7];
    const int s16 = s8 + __shfl_xor_sync(0xffffffffu, s8, 1);
    if ((lane & 1) == 0) reinterpret_cast<int16_t *>(act + ACT_BS + (size_t)b * 32)[lane >> 1] = (int16_t)s16;
    if (lane == 0) reinterpret_cast<float *>(act + ACT_D)[b] = d;
}

// (FLOW_AB_BATCH_QUANT builds only: measured 420 vs 426 tok/s for the serial form, lease X -- the extra live registers cost more than the
// overlapped chains gain.)  The same for NU blocks at once, stage by stage: one block is a serial latency chain (redux -> ballot -> shuffle -> IEEE division ->
// convert -> division -> pack -> store, ~500 cycles) and a warp quantises 3 - 8 blocks per phase while 147 other CTAs wait for nobody
// but themselves -- the fine-grained trace put 2.0 us (K = 4096) and 5.3 us (K = 14336) of every dependency hop here.  With the
// stages of the NU blocks interleaved the chains overlap.  Same arithmetic, bit for bit (blocks that do not exist compute on zeros and
// store nothing).
template <int NU>
__device__ __forceinline__ void quant_blocks(const float (&v)[NU][8], const int (&b)[NU], const bool (&on)[NU], int lane, uint8_t * act) {
    unsigned mloc[NU], mall[NU];
#pragma unroll
    for (int u = 0; u < NU; u++) {
        mloc[u] = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) { const unsigned a = (v[u][i] == v[u][i]) ? (__float_as_uint(v[u][i]) & 0x7fffffffu) : 0u; mloc[u] = a > mloc[u] ? a : mloc[u]; }
    }
#pragma unroll
    for (int u = 0; u < NU; u++) mall[u] = __reduce_max_sync(0xffffffffu, mloc[u]);
    float mine[NU], maxv[NU];
    int wl[NU];
#pragma unroll
    for (int u = 0; u < NU; u++) {
        wl[u] = __ffs((int)__ballot_sync(0xffffffffu, mloc[u] == mall[u])) - 1;
        mine[u] = 0.0f;
#pragma unroll
        for (int i = 7; i >= 0; i--) mine[u] = ((__float_as_uint(v[u][i]) & 0x7fffffffu) == mall[u] && v[u][i] == v[u][i]) ? v[u][i] : mine[u];
    }
#pragma unroll
    for (int u = 0; u < NU; u++) maxv[u] = __shfl_sync(0xffffffffu, mine[u], wl[u]);
    float iscale[NU], d[NU];
#pragma unroll
    for (int u = 0; u < NU; u++) {
        const bool nz = __uint_as_float(mall[u]) > 0.0f;
        iscale[u] = nz ? __fdiv_rn(-127.0f, maxv[u]) : 0.0f;            // (all-zero block: every q becomes 0, d = 0)
        d[u] = nz ? __fdiv_rn(1.0f, iscale[u]) : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < NU; u++) {
        int q[8];
#pragma unroll
        for (int i = 0; i < 8; i++) { const int t = __float2int_rn(__fmul_rn(iscale[u], v[u][i])); q[i] = t > 127 ? 127 : t; }
        uint2 packed;
        packed.x = (uint32_t)(q[0] & 0xFF) | ((uint32_t)(q[1] & 0xFF) << 8) | ((uint32_t)(q[2] & 0xFF) << 16) | ((uint32_t)(q[3] & 0xFF) << 24);
        packed.y = (uint32_t)(q[4] & 0xFF) | ((uint32_t)(q[5] & 0xFF) << 8) | ((uint32_t)(q[6] & 0xFF) << 16) | ((uint32_t)(q[7] & 0xFF) << 24);
        const int s8 = q[0] + q[1] + q[2] + q[3] + q[4] + q[5] + q[6] + q[7];
        const int s16 = s8 + __shfl_xor_sync(0xffffffffu, s8, 1);
        if (on[u]) {
            *reinterpret_cast<uint2 *>(act + (size_t)b[u] * ACT_PITCH + 8 * lane) = packed;
            if ((lane & 1) == 0) reinterpret_cast<int16_t *>(act + ACT_BS + (size_t)b[u] * 32)[lane >> 1] = (int16_t)s16;
            if (lane == 0) reinterpret_cast<float *>(act + ACT_D)[b[u]] = d[u];
        }
    }
}

// ------------------------------------------------------------------------------------------------ mat-vec phase (consumer warps)
struct Ctx {
    EpochT epoch;
    unsigned g;                        // pieces consumed so far by the CTA (all warps count all pieces)
    bool h_ok;                         // this CTA's shared-memory copy of the hidden state is the one the program refers to
    unsigned long long * trace;
};

__device__ __forceinline__ void stamp(const Ctx & c, int pi, int k) {
    if (c.trace != nullptr && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
        c.trace[((size_t)pi * FLOW_TRACE_N + k) * 160 + blockIdx.x] = t;
    }
}

// Everything a warp needs to turn the pieces of ONE matrix of a phase into output rows, hoisted into registers once per matrix (the
// first version re-read these from the descriptor for every piece: ~1 000 cycles of dependent shared/global loads per 7 KB piece).
struct MatCtx {
    const uint8_t * w0, * w1;          // weights (w1: the "up" matrix of a SwiGLU pair)
    int64_t rs0, rs1;                  // row strides
    FlowOut out;
    FlowVec residual;
    const float * h;                   // != nullptr: the residual is the hidden state in shared memory
    float * part;                      // S == 2: partial sums [2][FLOW_PART_ROWS]
    int mode, S, seg, RP, rp_shift, R, rb, rb_end, row_bytes, spitch, rpitch;
    bool contiguous;
    uint32_t tag;
    EpochT epoch;
#if FLOW_TP
    const FlowMatvec * desc;           // shared-memory descriptor (peer pointers of a tensor-parallel partial result)
#endif
};

__device__ __forceinline__ void mv_epilogue(const MatCtx & mc, int row, float v, float gate) {
    if (mc.mode == 2) {
        const float silu = __fdiv_rn(gate, __fadd_rn(1.0f, expf(-gate)));
        out_st(mc.out, row, mc.tag, __fmul_rn(silu, v));
    } else {
        if (mc.mode == 1) v = __fadd_rn(v, mc.h != nullptr ? mc.h[row] : vec_ld(mc.residual, row, mc.epoch));
        out_st(mc.out, row, mc.tag, v);
#if FLOW_TP
        const int npeer = mc.desc->npeer;
        if (npeer > 0) {                                       // tensor-parallel partial: one tagged slot per GPU of the group, over NVLink
            const uint32_t ctag = mc.epoch.coll + mc.desc->coll + 1u;
            for (int d = 0; d < npeer; d++) st_slot_sys(mc.desc->peer[d] + row, ctag, v);
        }
#endif
    }
}

// One ring piece: rows r0 .. r0 + nr of k-segment s (SUB = 2: the same rows of the gate and the up matrix).
template <int T, int SUB>
__device__ __forceinline__ void consume_piece(const MatCtx & mc, int r0, int nr, int s, const uint8_t * sl, const uint32_t (&a)[64], const uint32_t (&bs16)[8],
                                              const uint32_t (&bs32)[4], float da, int kl, int lr, bool lane_on, int lane) {
    constexpr int BB = Fmt<T>::BB;
    const int steps = (nr + mc.RP - 1) >> mc.rp_shift;
    for (int u = 0; u < steps; u++) {
        const int r = (u << mc.rp_shift) + lr;
        const bool on = lane_on && r < nr;
        float acc[2] = {0.0f, 0.0f};
#pragma unroll
        for (int j = 0; j < SUB; j++) {
            if (on) {
                const uint8_t * wb;
                // offset of the copy inside its 16-byte granule: only Q6_K rows / segments can start off a 16-byte boundary
                if (mc.contiguous) {
                    const int off = T == T_Q6_K ? (int)(reinterpret_cast<uintptr_t>((j ? mc.w1 : mc.w0) + (int64_t)r0 * (j ? mc.rs1 : mc.rs0)) & 15) : 0;
                    wb = sl + j * mc.spitch + off + r * mc.row_bytes + kl * BB;
                } else {
                    const int off = T == T_Q6_K ? (int)(reinterpret_cast<uintptr_t>((j ? mc.w1 : mc.w0) + (int64_t)(r0 + r) * (j ? mc.rs1 : mc.rs0) + (int64_t)s * mc.seg * BB) & 15) : 0;
                    wb = sl + (j * mc.R + r) * mc.rpitch + off + kl * BB;
                }
                acc[j] = RegDot<T>::run(wb, a, bs16, bs32, da);
            }
        }
        // sum over the k-blocks of the row: the lanes of one row are lr's group (RP > 1: aligned groups of seg lanes) or the whole warp
        if (mc.RP > 1) {
            for (int o = mc.seg >> 1; o > 0; o >>= 1) {
                acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], o);
                if (SUB == 2) acc[1] += __shfl_xor_sync(0xffffffffu, acc[1], o);
            }
        } else {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], o);
                if (SUB == 2) acc[1] += __shfl_xor_sync(0xffffffffu, acc[1], o);
            }
        }
        if (kl == 0 && r < nr && (mc.RP > 1 || lane == 0)) {
            const int row = r0 + r;
            if (mc.S == 1) mv_epilogue(mc, row, SUB == 2 ? acc[1] : acc[0], acc[0]);
            else mc.part[s * FLOW_PART_ROWS + (row - mc.rb)] = acc[0];
        }
    }
}

// All of this warp's pieces of one matrix.  Piece t of the matrix (chunk t / S, segment t % S) is piece qbase + t of the phase and goes
// to warp piece_warp(S, qbase + t); the warp walks only its own.
template <int T, int SUB>
__device__ __forceinline__ void consume_matrix(const MatCtx & mc, int nch, unsigned gbase, unsigned qbase, uint8_t * smem, const uint32_t (&a)[64],
                                               const uint32_t (&bs16)[8], const uint32_t (&bs32)[4], float da, int kl, int lr, bool lane_on, int warp, int lane,
                                               bool timed, long long & t_wait, long long & t_comp) {
    uint64_t * full = reinterpret_cast<uint64_t *>(smem + OFF_BARS), * empty = full + FL_NSLOTS;
    const uint8_t * ring = smem + OFF_RING;
    const int re_rows = nch;                                            // (chunks of R rows)
    int t, tstep;
    if (mc.S == 1) { t = (warp + FL_NW - (int)(qbase % FL_NW)) % FL_NW; tstep = FL_NW; }
    else { if (warp >= 2 * FL_NPAIR) return; t = 2 * (warp >> 1) + (warp & 1); tstep = 2 * FL_NPAIR; }      // (S == 2: single matrix, qbase == 0)
    for (; t < re_rows * mc.S; t += tstep) {
        const int ch = mc.S == 1 ? t : t >> 1, sgm = mc.S == 1 ? 0 : t & 1;
        const unsigned g = gbase + qbase + (unsigned)t, slot = g % FL_NSLOTS, use = g / FL_NSLOTS;
        const long long tw0 = timed ? clock64() : 0;
        // The warps take pieces round-robin, so the consumer of the slot's previous use is another warp, and this warp can get here while
        // that use's copy is still landing.  A parity wait on `full` alone would then see the phase before it (same parity) and pass.  Wait
        // first for the previous use to be released.  That wait cannot alias: every mat-vec phase starts with a barrier of all consumer
        // warps, and inside a phase a warp takes every FL_NW-th (S == 2: every 2 FL_NPAIR-th) piece, so this warp's previous piece is fewer
        // than FL_NSLOTS pieces back -- then it, and before it the slot's previous use, were issued, which the producer did only after the
        // use before was released -- or the previous use lies before this phase and was consumed at that barrier.
        if (use > 0) fl_mbar_wait(empty + slot, (use - 1) & 1u);
        fl_mbar_wait(full + slot, use & 1u);
        const long long tw1 = timed ? clock64() : 0;
        const int r0 = mc.rb + ch * mc.R;
        consume_piece<T, SUB>(mc, r0, min(mc.R, mc.rb_end - r0), sgm, ring + (size_t)slot * FL_SLOT, a, bs16, bs32, da, kl, lr, lane_on, lane);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + slot);
        if (timed) { t_wait += tw1 - tw0; t_comp += clock64() - tw1; }
    }
}

__device__ __forceinline__ void matvec_phase(const FlowMatvec & p, int pi, Ctx & c, uint8_t * smem) {   // p: the shared-memory copy
    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = (int)blockIdx.x, grid = (int)gridDim.x;
    const int nblk = p.K >> 8;
    const EpochT epoch = c.epoch;
    const uint32_t tag = phase_epoch(epoch) + (uint32_t)pi + 1u;
    uint8_t * act = smem + OFF_ACT;
    double * red = reinterpret_cast<double *>(smem + OFF_RED);
    float * part = reinterpret_cast<float *>(smem + OFF_PART);
    float * h = reinterpret_cast<float *>(smem + OFF_H);

    // does this CTA have rows in this phase at all?  (it still counts the pieces of nobody: none exist for it)
    bool any = false;
    const int nenum = p.mode == 2 ? 1 : p.nmat;
    for (int m = 0; m < nenum; m++) any = any || row_begin(p, m, cta + 1) > row_begin(p, m, cta);
    // A CTA without rows does not touch the phase at all (only CTAs that also PRODUCE may read a vector: that is what makes the
    // reuse of slots and of in-place ggml buffers safe); it then has no copy of the hidden state this phase hands on.
    if (!any) { if (p.keep_h) c.h_ok = false; return; }
    if (p.keep_h) c.h_ok = true;
    const float * hres = (p.mode == 1 && p.resid_h && c.h_ok) ? h : nullptr;

    // ---- activation prologue: warp w owns blocks w, w + 8, ...; lane l owns elements 8l..8l+7 of a block.  Passes of 35 blocks
    //      (5 per warp); a fused RMS_NORM needs the whole vector before anything is quantised, so it is limited to one pass
    //      (K <= FLOW_MAX_NORM_K = 8192 = 32 blocks).
    const bool norm = p.norm_w != nullptr;
    for (int base = 0; base < nblk; base += FL_PU * FL_NW) {
        float xv[FL_PU][8];
        uint64_t raw[FL_PU][8];
#pragma unroll
        for (int u = 0; u < FL_PU; u++) {
            const int b = base + warp + u * FL_NW;
            if (b < nblk) vec_ld8_issue(p.x, 256 * b + 8 * lane, raw[u]);
        }
        double acc = 0.0;
        {
            int idx[FL_PU];
            bool on[FL_PU];
#pragma unroll
            for (int u = 0; u < FL_PU; u++) { const int b = base + warp + u * FL_NW; on[u] = b < nblk; idx[u] = 256 * b + 8 * lane; }
#if defined(FLOW_FINE_TRACE)
            unsigned long long * tf = (c.trace != nullptr && tid == 0 && base == 0) ? &c.trace[((size_t)pi * FLOW_TRACE_N + 6) * 160 + blockIdx.x] : nullptr;
            vec_ld8_finish_blocks<FL_PU>(p.x, idx, on, epoch, raw, xv, tf);
#else
            vec_ld8_finish_blocks<FL_PU>(p.x, idx, on, epoch, raw, xv);
#endif
        }
        // the norm weights of this warp's blocks: requested now, so that their L2 round trip runs under the sum-of-squares reduction
        // and its barrier (there is practically no L1 next to 227 KB of shared memory)
#if defined(FLOW_AB_NW_EARLY)
        float4 nw[FL_PU][2];
        if (norm) {
#pragma unroll
            for (int u = 0; u < FL_PU; u++) {
                const int b = base + warp + u * FL_NW;
                if (b < nblk) {
                    nw[u][0] = __ldg(reinterpret_cast<const float4 *>(p.norm_w + 256 * b + 8 * lane));
                    nw[u][1] = __ldg(reinterpret_cast<const float4 *>(p.norm_w + 256 * b + 8 * lane) + 1);
                }
            }
        }
#endif
#pragma unroll
        for (int u = 0; u < FL_PU; u++) {
            const int b = base + warp + u * FL_NW;
            if (b < nblk) {
                if (norm) {
#pragma unroll
                    for (int i = 0; i < 8; i++) acc += (double)__fmul_rn(xv[u][i], xv[u][i]);
                }
                if (p.keep_h) {
                    float4 * hp = reinterpret_cast<float4 *>(h + 256 * b + 8 * lane);
                    hp[0] = make_float4(xv[u][0], xv[u][1], xv[u][2], xv[u][3]);
                    hp[1] = make_float4(xv[u][4], xv[u][5], xv[u][6], xv[u][7]);
                }
            }
        }
        if (base == 0) stamp(c, pi, 1);
        float scale = 1.0f;
        if (norm) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) red[warp] = acc;
            bar_consumers();
            double tot = 0.0;
#pragma unroll
            for (int i = 0; i < FL_NW; i++) tot += red[i];
            const float mean = (float)(tot / (double)p.K);
            scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, p.eps)));
#if defined(FLOW_FINE_TRACE)
            if (base == 0) stamp(c, pi, 7);
#endif
        }
#if !defined(FLOW_AB_BATCH_QUANT)
        {
#pragma unroll
            for (int u = 0; u < FL_PU; u++) {
                const int b = base + warp + u * FL_NW;
                if (b < nblk) {
                    float v[8];
                    if (norm) {
#if defined(FLOW_AB_NW_EARLY)
                        const float4 w0 = nw[u][0], w1 = nw[u][1];
#else
                        const float4 w0 = __ldg(reinterpret_cast<const float4 *>(p.norm_w + 256 * b + 8 * lane)), w1 = __ldg(reinterpret_cast<const float4 *>(p.norm_w + 256 * b + 8 * lane) + 1);
#endif
                        const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                        for (int i = 0; i < 8; i++) v[i] = __fmul_rn(__fmul_rn(xv[u][i], scale), wv[i]);
                        if (p.norm_out != nullptr && cta == 0) {
                            float4 * op = reinterpret_cast<float4 *>(p.norm_out + 256 * b + 8 * lane);
                            op[0] = make_float4(v[0], v[1], v[2], v[3]);
                            op[1] = make_float4(v[4], v[5], v[6], v[7]);
                        }
                    } else {
#pragma unroll
                        for (int i = 0; i < 8; i++) v[i] = xv[u][i];
                    }
                    quant_block(v, b, lane, act);
                }
            }
        }
#else
        {
            float v[FL_PU][8];
            int bi[FL_PU];
            bool onb[FL_PU];
#pragma unroll
            for (int u = 0; u < FL_PU; u++) { bi[u] = base + warp + u * FL_NW; onb[u] = bi[u] < nblk; }
            if (norm) {
                float4 w0[FL_PU], w1[FL_PU];
#pragma unroll
                for (int u = 0; u < FL_PU; u++) {                        // all the norm-weight loads of the warp go out together
                    if (onb[u]) {
                        w0[u] = __ldg(reinterpret_cast<const float4 *>(p.norm_w + 256 * bi[u] + 8 * lane));
                        w1[u] = __ldg(reinterpret_cast<const float4 *>(p.norm_w + 256 * bi[u] + 8 * lane) + 1);
                    } else { w0[u] = make_float4(0.f, 0.f, 0.f, 0.f); w1[u] = w0[u]; }
                }
#pragma unroll
                for (int u = 0; u < FL_PU; u++) {
                    const float wv[8] = {w0[u].x, w0[u].y, w0[u].z, w0[u].w, w1[u].x, w1[u].y, w1[u].z, w1[u].w};
#pragma unroll
                    for (int i = 0; i < 8; i++) v[u][i] = onb[u] ? __fmul_rn(__fmul_rn(xv[u][i], scale), wv[i]) : 0.0f;
                    if (onb[u] && p.norm_out != nullptr && cta == 0) {
                        float4 * op = reinterpret_cast<float4 *>(p.norm_out + 256 * bi[u] + 8 * lane);
                        op[0] = make_float4(v[u][0], v[u][1], v[u][2], v[u][3]);
                        op[1] = make_float4(v[u][4], v[u][5], v[u][6], v[u][7]);
                    }
                }
            } else {
#pragma unroll
                for (int u = 0; u < FL_PU; u++) {
#pragma unroll
                    for (int i = 0; i < 8; i++) v[u][i] = onb[u] ? xv[u][i] : 0.0f;
                }
            }
            quant_blocks<FL_PU>(v, bi, onb, lane, act);
        }
#endif
    }
#if defined(FLOW_FINE_TRACE)
    stamp(c, pi, 8);
#endif
    bar_consumers();

    // ---- bind the lane to its k-block and pull that block of the quantised activation into registers
    const int s_w = p.S == 2 ? (warp & 1) : 0;                          // this warp's k-segment (see piece_warp)
    const int kl = p.RP > 1 ? (lane & (p.seg - 1)) : lane;
    const int lr = p.RP > 1 ? lane / p.seg : 0;
    const bool lane_on = kl < seg_len(p, nblk, s_w);
    const int kb = s_w * p.seg + (lane_on ? kl : 0);
    uint32_t a[64], bs16[8], bs32[4];
    {
        const uint4 * ap = reinterpret_cast<const uint4 *>(act + (size_t)kb * ACT_PITCH);
#pragma unroll
        for (int i = 0; i < 16; i++) { const uint4 t = ap[i]; a[4 * i] = t.x; a[4 * i + 1] = t.y; a[4 * i + 2] = t.z; a[4 * i + 3] = t.w; }
        const uint4 * bp = reinterpret_cast<const uint4 *>(act + ACT_BS + (size_t)kb * 32);
        const uint4 b0 = bp[0], b1 = bp[1];
        bs16[0] = b0.x; bs16[1] = b0.y; bs16[2] = b0.z; bs16[3] = b0.w; bs16[4] = b1.x; bs16[5] = b1.y; bs16[6] = b1.z; bs16[7] = b1.w;
#pragma unroll
        for (int i = 0; i < 4; i++) {                                    // sums of 32 = pairs of sums of 16 (they fit int16: |sum| <= 32 * 127)
            const int lo = (int)(int16_t)(bs16[2 * i] & 0xFFFFu) + (int)(int16_t)(bs16[2 * i] >> 16);
            const int hi = (int)(int16_t)(bs16[2 * i + 1] & 0xFFFFu) + (int)(int16_t)(bs16[2 * i + 1] >> 16);
            bs32[i] = ((uint32_t)lo & 0xFFFFu) | ((uint32_t)hi << 16);
        }
    }
    const float da = reinterpret_cast<const float *>(act + ACT_D)[kb];
    stamp(c, pi, 2);

    // ---- consume this warp's pieces, matrix by matrix (same enumeration as the producer)
    unsigned q = 0;
    long long t_wait = 0, t_comp = 0;
    const bool timed = c.trace != nullptr;
    MatCtx mc;
    mc.mode = p.mode; mc.S = p.S; mc.seg = p.seg; mc.RP = p.RP; mc.rp_shift = 31 - __clz(p.RP);
    mc.h = hres; mc.part = part; mc.tag = tag; mc.epoch = epoch;
#if FLOW_TP
    mc.desc = &p;
#endif
    mc.residual = p.residual;
    for (int m = 0; m < nenum; m++) {
        const int Mm = p.M[m], T = p.type[m];
        mc.R = p.R[m];
        mc.rb = row_begin(p, m, cta); mc.rb_end = row_begin(p, m, cta + 1);
        mc.row_bytes = nblk * block_bytes(T);
        mc.w0 = p.w[m]; mc.rs0 = p.row_stride[m];
        mc.w1 = p.w[1]; mc.rs1 = p.row_stride[1];
        mc.out = p.mode == 2 ? p.out[0] : p.out[m];
        mc.contiguous = p.S == 1 && mc.rs0 == (int64_t)mc.row_bytes && (p.mode != 2 || mc.rs1 == (int64_t)mc.row_bytes);
        mc.spitch = sub_pitch(mc.R, mc.row_bytes); mc.rpitch = row_pitch(p.seg, block_bytes(T));
        const int nch = (mc.rb_end - mc.rb + mc.R - 1) / mc.R;
#if defined(FLOW_FINE_TRACE)
        if (m == 0) stamp(c, pi, 9);
#endif
        if (p.mode == 2) {
            switch (T) {
                case T_Q4_K: consume_matrix<T_Q4_K, 2>(mc, nch, c.g, q, smem, a, bs16, bs32, da, kl, lr, lane_on, warp, lane, timed, t_wait, t_comp); break;
                case T_Q5_K: consume_matrix<T_Q5_K, 2>(mc, nch, c.g, q, smem, a, bs16, bs32, da, kl, lr, lane_on, warp, lane, timed, t_wait, t_comp); break;
                default:     consume_matrix<T_Q6_K, 2>(mc, nch, c.g, q, smem, a, bs16, bs32, da, kl, lr, lane_on, warp, lane, timed, t_wait, t_comp); break;
            }
        } else {
            switch (T) {
                case T_Q4_K: consume_matrix<T_Q4_K, 1>(mc, nch, c.g, q, smem, a, bs16, bs32, da, kl, lr, lane_on, warp, lane, timed, t_wait, t_comp); break;
                case T_Q5_K: consume_matrix<T_Q5_K, 1>(mc, nch, c.g, q, smem, a, bs16, bs32, da, kl, lr, lane_on, warp, lane, timed, t_wait, t_comp); break;
                default:     consume_matrix<T_Q6_K, 1>(mc, nch, c.g, q, smem, a, bs16, bs32, da, kl, lr, lane_on, warp, lane, timed, t_wait, t_comp); break;
            }
        }
        q += (unsigned)(nch * p.S);
    }
#if defined(FLOW_FINE_TRACE)
    if (timed && lane == 0) atomicMax(&c.trace[((size_t)pi * FLOW_TRACE_N + 10) * 160 + blockIdx.x], gtime());
#endif
    if (timed && tid == 0) {                             // warp 0's cycles waiting for weight bytes / computing, this phase
        c.trace[((size_t)pi * FLOW_TRACE_N + 4) * 160 + blockIdx.x] = (unsigned long long)t_wait;
        c.trace[((size_t)pi * FLOW_TRACE_N + 5) * 160 + blockIdx.x] = (unsigned long long)t_comp;
    }
    c.g += q;
    if (p.S == 2) {                                                      // rows split over two warps: combine the halves in a fixed order
        bar_consumers();
        const int rb = row_begin(p, 0, cta), re = row_begin(p, 0, cta + 1);
        mc.out = p.out[0];
        for (int t = tid; t < re - rb; t += FL_CTHREADS) mv_epilogue(mc, rb + t, __fadd_rn(part[t], part[FLOW_PART_ROWS + t]), 0.0f);
    }
    stamp(c, pi, 3);
}

// pieces of a phase this CTA does NOT consume because it returned early: none -- a CTA without rows has no pieces.

// ------------------------------------------------------------------------------------------------ attention phase
__device__ __forceinline__ float block_max(float v, float * red, int warp, int lane) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    bar_consumers();                                                  // red[] free
    if (lane == 0) red[warp] = v;
    bar_consumers();
    float m = red[0];
#pragma unroll
    for (int i = 1; i < FL_NW; i++) m = fmaxf(m, red[i]);
    return m;
}
__device__ __forceinline__ float block_sum(float v, float * red, int warp, int lane) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    bar_consumers();
    if (lane == 0) red[warp] = v;
    bar_consumers();
    float t = 0.0f;
#pragma unroll
    for (int i = 0; i < FL_NW; i++) t += red[i];
    return t;
}

__device__ __forceinline__ void attn_phase(const FlowAttn & a, int pi, const Ctx & c, uint8_t * smem) {
    const int nsplit = a.nsplit;
    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = (int)blockIdx.x;
    const int D = a.head_dim;                                         // 128 (checked on the host)
    if (cta >= a.n_head * nsplit) return;
    const EpochT epoch = c.epoch;
    const uint32_t tag = phase_epoch(epoch) + (uint32_t)pi + 1u;
    const int h = cta / nsplit, part = cta % nsplit;
    const int gqa = a.n_head / a.n_head_kv, hk = h / gqa;
    float * att = reinterpret_cast<float *>(smem + OFF_ACT);
    float * sQ = att + ATT_Q, * sK = att + ATT_K, * sV = att + ATT_V, * sTh = att + ATT_TH, * sS = att + ATT_S, * sPV = att + ATT_PV;
    float * red = reinterpret_cast<float *>(smem + OFF_RED);
    // ---- ROPE of this head's q and of its kv head's new k (ggml ROPE, CPU's iterated theta), new v; f16 rounding as the cache / the
    //      CPU's q conversion.  One CTA of the GQA group stores the cache rows.  The ROPE nodes' own outputs are not materialised:
    //      they are consumed only here.
    const int64_t kpos = __ldcg(a.k_idx), vpos = __ldcg(a.v_idx);
    const bool writer_kv = part == 0 && (h % gqa) == 0;
    const int half = a.n_dims / 2;
    if (tid == 0) {
        float theta = (float)__ldcg(a.pos);
        for (int i = 0; i < half; i++) { sTh[i] = theta; theta = __fmul_rn(theta, a.theta_scale); }
    }
    bar_consumers();
    __half * kc = reinterpret_cast<__half *>(reinterpret_cast<char *>(a.k_cache) + kpos * a.k_row_bytes) + (int64_t)hk * D;
    __half * vc = reinterpret_cast<__half *>(reinterpret_cast<char *>(a.v_cache) + vpos * a.v_row_bytes) + (int64_t)hk * D;
    const int qo = h * D, ko = hk * D;
    // ---- this CTA's key range; the mask entry of the first key this thread scores does not depend on this token: requested now, so that
    //      the key row's loads need not wait for it later (one L2 round trip less on the critical path of a pure-latency phase)
    const int n_kv = a.n_kv;
    const int chunk = ((n_kv + nsplit - 1) / nsplit + 31) & ~31;
    const int k0 = part * chunk, k1 = min(n_kv, k0 + chunk);
    const char * kbase = reinterpret_cast<const char *>(a.kview) + (int64_t)hk * a.k_nb2;
    const char * vbase = reinterpret_cast<const char *>(a.vview) + (int64_t)hk * a.v_nb2;
    const __half * mp = reinterpret_cast<const __half *>(a.mask);
    const int dc = tid & 15, kg = tid >> 4;                           // P.V ownership: dims 8dc..8dc+7, keys kg, kg + FL_KG, ...
    const int key_pf = k0 + tid;
    const float mv_pf = (mp && key_pf < k1) ? __half2float(mp[key_pf]) : 0.0f;
#if defined(FLOW_AB_ATTN_PREFETCH_V)
    uint4 vpf[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int key = k0 + kg + u * FL_KG;
        vpf[u] = make_uint4(0u, 0u, 0u, 0u);
        if (key < k1 && key != (int)vpos) vpf[u] = __ldg(reinterpret_cast<const uint4 *>(vbase + (int64_t)key * a.v_nb1) + dc);
    }
#endif
    // every load of this thread goes out first (q pair, k pair, v element), then whatever is still stale is re-polled as a batch: the three
    // vectors come from the same mat-vec phase, so they land together and sequential re-polls would only add L2 round trips
    const bool has_v = tid < D;
    uint64_t rv = has_v ? vec_peek(a.v, ko + tid) : 0ull;
    for (int i = tid; i < half; i += FL_CTHREADS) {
        const float theta_extrap = a.freq_factors ? __fdiv_rn(sTh[i], a.freq_factors[i]) : sTh[i];
        const float theta_interp = __fmul_rn(a.freq_scale, theta_extrap);
        float theta = theta_interp, mscale = a.attn_factor;
        if (a.ext_factor != 0.0f) {
            const float yv = ((float)i - a.corr0) / fmaxf(0.001f, a.corr1 - a.corr0);
            const float ramp_mix = (1.0f - fminf(1.0f, fmaxf(0.0f, yv))) * a.ext_factor;
            theta = theta_interp * (1.0f - ramp_mix) + theta_extrap * ramp_mix;
            mscale *= 1.0f + 0.1f * logf(1.0f / a.freq_scale);
        }
        const int ia = a.rope_mode == 0 ? 2 * i : i, ib = a.rope_mode == 0 ? 2 * i + 1 : i + half;
        uint64_t rq0 = vec_peek(a.q, qo + ia), rq1 = vec_peek(a.q, qo + ib), rk0 = vec_peek(a.k, ko + ia), rk1 = vec_peek(a.k, ko + ib);
        const float cs = cosf(theta) * mscale, sn = sinf(theta) * mscale;
        {
            const uint32_t wq = want_tag(a.q, epoch), wk = want_tag(a.k, epoch), wv = want_tag(a.v, epoch);
            const bool pq = a.q.ll != nullptr, pk = a.k.ll != nullptr, pv = has_v && a.v.ll != nullptr;
            long long spins = 0;
            for (;;) {
                bool stale = false;
                if (pq && (uint32_t)(rq0 >> 32) != wq) { rq0 = ld_slot(a.q.ll + qo + ia); stale = true; }
                if (pq && (uint32_t)(rq1 >> 32) != wq) { rq1 = ld_slot(a.q.ll + qo + ib); stale = true; }
                if (pk && (uint32_t)(rk0 >> 32) != wk) { rk0 = ld_slot(a.k.ll + ko + ia); stale = true; }
                if (pk && (uint32_t)(rk1 >> 32) != wk) { rk1 = ld_slot(a.k.ll + ko + ib); stale = true; }
                if (pv && (uint32_t)(rv >> 32) != wv) { rv = ld_slot(a.v.ll + ko + tid); stale = true; }
                if (!stale) break;
                spin_fail(spins);
            }
        }
        {
            const float x0 = __uint_as_float((uint32_t)rq0), x1 = __uint_as_float((uint32_t)rq1);
            const float y0 = __fsub_rn(__fmul_rn(x0, cs), __fmul_rn(x1, sn)), y1 = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, cs));
            sQ[ia] = __half2float(__float2half_rn(y0)); sQ[ib] = __half2float(__float2half_rn(y1));
        }
        {
            const float x0 = __uint_as_float((uint32_t)rk0), x1 = __uint_as_float((uint32_t)rk1);
            const float y0 = __fsub_rn(__fmul_rn(x0, cs), __fmul_rn(x1, sn)), y1 = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, cs));
            const __half h0 = __float2half_rn(y0), h1 = __float2half_rn(y1);
            if (writer_kv) { kc[ia] = h0; kc[ib] = h1; }
            sK[ia] = __half2float(h0); sK[ib] = __half2float(h1);
        }
    }
    for (int i = a.n_dims + tid; i < D; i += FL_CTHREADS) {
        const float qv = vec_ld(a.q, qo + i, epoch), kv = vec_ld(a.k, ko + i, epoch);
        sQ[i] = __half2float(__float2half_rn(qv));
        const __half hh = __float2half_rn(kv);
        if (writer_kv) kc[i] = hh;
        sK[i] = __half2float(hh);
    }
    if (has_v) {
        const __half hv = __float2half_rn(vec_resolve(a.v, ko + tid, epoch, rv));
        if (writer_kv) vc[tid] = hv;
        sV[tid] = __half2float(hv);
    }
    bar_consumers();

    float M = -INFINITY, L = 0.0f, o[8];
#pragma unroll
    for (int i = 0; i < 8; i++) o[i] = 0.0f;

    for (int t0 = k0; t0 < k1; t0 += FL_TK) {
        const int t1 = min(k1, t0 + FL_TK);
        float lmax = -INFINITY;
        for (int key = t0 + tid; key < t1; key += FL_CTHREADS) {      // scores: one key per thread
            const float mv = key == key_pf ? mv_pf : (mp ? __half2float(mp[key]) : 0.0f);
            float sc = -INFINITY;
            if (mv != -INFINITY) {
                float dot = 0.0f;
                if (key == (int)kpos) {
                    for (int d = 0; d < D; d++) dot += sQ[d] * sK[d];
                } else {
                    const uint4 * kr = reinterpret_cast<const uint4 *>(kbase + (int64_t)key * a.k_nb1);
                    uint4 kreg[16];                                   // the whole key row in flight at once (the phase is latency-bound)
#pragma unroll
                    for (int cc = 0; cc < 16; cc++) kreg[cc] = __ldg(kr + cc);
#pragma unroll
                    for (int cc = 0; cc < 16; cc++) {
                        const uint4 kk = kreg[cc];
                        const __half2 * k2 = reinterpret_cast<const __half2 *>(&kk);
                        const float4 q0 = *reinterpret_cast<const float4 *>(sQ + 8 * cc), q1 = *reinterpret_cast<const float4 *>(sQ + 8 * cc + 4);
                        const float2 f0 = __half22float2(k2[0]), f1 = __half22float2(k2[1]), f2 = __half22float2(k2[2]), f3 = __half22float2(k2[3]);
                        dot += q0.x * f0.x; dot += q0.y * f0.y; dot += q0.z * f1.x; dot += q0.w * f1.y;
                        dot += q1.x * f2.x; dot += q1.y * f2.y; dot += q1.z * f3.x; dot += q1.w * f3.y;
                    }
                }
                sc = dot * a.scale;
                if (a.softcap != 0.0f) sc = a.softcap * tanhf(sc);
                sc += mv;
            }
            sS[key - t0] = sc;
            lmax = fmaxf(lmax, sc);
        }
        const float Mt = block_max(lmax, red, warp, lane);
        const float Mnew = fmaxf(M, Mt);
        const float muse = Mnew == -INFINITY ? 0.0f : Mnew;
        const float alpha = expf(M - muse);                           // M = -inf -> 0
        float lsum = 0.0f;
        for (int key = t0 + tid; key < t1; key += FL_CTHREADS) {
            const float pv = expf(sS[key - t0] - muse);
            sS[key - t0] = pv;
            lsum += pv;
        }
        const float Lt = block_sum(lsum, red, warp, lane);            // the syncs inside also publish sS
        L = L * alpha + Lt;
        M = Mnew;
#pragma unroll
        for (int i = 0; i < 8; i++) o[i] *= alpha;
        for (int key0 = t0 + kg; key0 < t1; key0 += 8 * FL_KG) {     // 8 keys of this thread's group per round: their V chunks in flight together
            float pvv[8];
            uint4 rawv[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int key = key0 + u * FL_KG;
                pvv[u] = key < t1 ? sS[key - t0] : 0.0f;
                rawv[u] = make_uint4(0u, 0u, 0u, 0u);
#if defined(FLOW_AB_ATTN_PREFETCH_V)
                if (key0 == k0 + kg) { rawv[u] = vpf[u]; continue; }
#endif
                if (pvv[u] != 0.0f && key != (int)vpos) rawv[u] = __ldg(reinterpret_cast<const uint4 *>(vbase + (int64_t)key * a.v_nb1) + dc);
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {                             // keys in ascending order: the sum is the same whatever the timing
                const int key = key0 + u * FL_KG;
                if (pvv[u] == 0.0f) continue;
                float vv[8];
                if (key == (int)vpos) {
#pragma unroll
                    for (int i = 0; i < 8; i++) vv[i] = sV[8 * dc + i];
                } else {
                    const __half2 * v2 = reinterpret_cast<const __half2 *>(&rawv[u]);
                    const float2 f0 = __half22float2(v2[0]), f1 = __half22float2(v2[1]), f2 = __half22float2(v2[2]), f3 = __half22float2(v2[3]);
                    vv[0] = f0.x; vv[1] = f0.y; vv[2] = f1.x; vv[3] = f1.y; vv[4] = f2.x; vv[5] = f2.y; vv[6] = f3.x; vv[7] = f3.y;
                }
#pragma unroll
                for (int i = 0; i < 8; i++) o[i] += pvv[u] * vv[i];
            }
        }
        bar_consumers();                                              // sS is rewritten by the next tile
    }
    // ---- reduce the FL_KG partial outputs per dim
#pragma unroll
    for (int i = 0; i < 8; i++) sPV[kg * 128 + 8 * dc + i] = o[i];
    bar_consumers();
    float outv = 0.0f;
    if (tid < D) {
        for (int q = 0; q < FL_KG; q++) outv += sPV[q * 128 + tid];
    }
    if (nsplit == 1) {
        if (tid < D) out_st(a.out, qo + tid, tag, L > 0.0f ? outv / L : 0.0f);
        bar_consumers();                                              // scratch is the next phase's activation area
        return;
    }
    // ---- split head: every part publishes (partial, M, L) as tagged slots; part 0 combines all parts in a fixed order
    uint64_t * my = a.part_ll + (int64_t)(h * nsplit + part) * (D + 2);
    if (part != 0) {
        if (tid < D) st_slot(my + tid, tag, outv);
        if (tid == 0) { st_slot(my + D, tag, M); st_slot(my + D + 1, tag, L); }
        bar_consumers();
        return;
    }
    if (tid < D) {
        FlowVec pv;
        pv.plain = nullptr; pv.tag = (uint32_t)pi + 1u; pv.flags = 0;
        float Ms = M;
        for (int q = 1; q < nsplit; q++) { pv.ll = a.part_ll + (int64_t)(h * nsplit + q) * (D + 2); Ms = fmaxf(Ms, vec_ld(pv, D, epoch)); }
        const float mu = Ms == -INFINITY ? 0.0f : Ms;
        float f = expf(M - mu);
        float accv = f * outv, Ls = f * L;
        for (int q = 1; q < nsplit; q++) {
            pv.ll = a.part_ll + (int64_t)(h * nsplit + q) * (D + 2);
            f = expf(vec_ld(pv, D, epoch) - mu);
            accv += f * vec_ld(pv, tid, epoch);
            Ls += f * vec_ld(pv, D + 1, epoch);
        }
        out_st(a.out, qo + tid, tag, Ls > 0.0f ? accv / Ls : 0.0f);
    }
    bar_consumers();
}

// ------------------------------------------------------------------------------------------------ the kernel
__global__ void __launch_bounds__(FL_THREADS, 1) decode_flow_kernel(const FlowPhase * __restrict__ ph, int n_phases, unsigned * sync, unsigned long long * trace, int throttle, int n_coll) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint64_t * full = reinterpret_cast<uint64_t *>(smem + OFF_BARS), * empty = full + FL_NSLOTS;
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < FL_NSLOTS; i++) { mbar_init(full + i, 1); mbar_init(empty + i, 1); }
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    if (tid < DESC_WORDS) reinterpret_cast<uint32_t *>(smem + OFF_DESC)[tid] = __ldg(reinterpret_cast<const uint32_t *>(ph) + tid);
    __syncthreads();
#if FLOW_TP
    EpochT epoch;
    epoch.phase = __ldcg(sync);                                       // left by the previous launch (0 after allocation)
    epoch.coll = __ldcg(sync + 2);
#else
    const EpochT epoch = __ldcg(sync);                                // left by the previous launch (0 after allocation)
#endif

    if (warp >= FL_NW) {
        if (warp == FL_NW) producer_loop(ph, n_phases, smem, lane, throttle);
    } else {
        // The consumers read the current phase's descriptor from shared memory (two slots); the next one is fetched at phase entry
        // and parked in a register until the phase's work is done (see producer_loop for why).
        uint32_t * cdesc = reinterpret_cast<uint32_t *>(smem + OFF_DESC);
        Ctx c;
        c.epoch = epoch; c.g = 0; c.trace = trace; c.h_ok = false;
        for (int pi = 0; pi < n_phases; pi++) {
            bar_consumers();                                          // every warp has left phase pi - 1 (and its descriptor slot is written)
            const bool pre = pi + 1 < n_phases && tid < DESC_WORDS;
            uint32_t nextw = 0;
            if (pre) nextw = __ldg(reinterpret_cast<const uint32_t *>(ph + pi + 1) + tid);
            const FlowPhase & d = *reinterpret_cast<const FlowPhase *>(cdesc + (pi & 1) * 96);
            const int kind = d.kind;
            stamp(c, pi, 0);
            if (kind == FLOW_MATVEC) {
                matvec_phase(d.mv, pi, c, smem);
            } else if (kind == FLOW_ATTN) {
                attn_phase(d.at, pi, c, smem);
#if FLOW_TP
            } else if (kind == FLOW_SUM) {
                // out = src[0] + src[1] + ... (rank order: bit-identical on every GPU of the group), 8 elements per thread, the vector
                // spread over all CTAs: the reduce half of the fused all-reduce (and the ADD that follows it, when the host folded it in)
                const FlowSum & sm = d.sm;
                const uint32_t tag = phase_epoch(epoch) + (uint32_t)pi + 1u;
                const int nunits = sm.n >> 3;
                const int u0 = (int)(((long long)nunits * blockIdx.x) / gridDim.x), u1 = (int)(((long long)nunits * (blockIdx.x + 1)) / gridDim.x);
                for (int u = u0 + tid; u < u1; u += FL_CTHREADS) {
                    float acc[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) acc[k] = 0.0f;
                    for (int s0 = 0; s0 < sm.nsrc; s0 += 3) {             // three sources' loads in flight together
                        uint64_t raw[3][8];
                        float x[8];
#pragma unroll
                        for (int j = 0; j < 3; j++) if (s0 + j < sm.nsrc) vec_ld8_issue(sm.src[s0 + j], 8 * u, raw[j]);
#pragma unroll
                        for (int j = 0; j < 3; j++) {
                            if (s0 + j < sm.nsrc) {
                                vec_ld8_finish(sm.src[s0 + j], 8 * u, epoch, raw[j], x);
#pragma unroll
                                for (int k = 0; k < 8; k++) acc[k] = (s0 + j) == 0 ? x[k] : __fadd_rn(acc[k], x[k]);
                                if (s0 + j + 1 == sm.n_first) {
#pragma unroll
                                    for (int k = 0; k < 8; k++) out_st(sm.out, 8 * u + k, tag, acc[k]);
                                }
                            }
                        }
                    }
                    if (sm.n_first < sm.nsrc) {
#pragma unroll
                        for (int k = 0; k < 8; k++) out_st(sm.out2, 8 * u + k, tag, acc[k]);
                    }
                }
                if (blockIdx.x == 0) {                                      // ragged tail
                    for (int i = 8 * nunits + tid; i < sm.n; i += FL_CTHREADS) {
                        float a = vec_ld(sm.src[0], i, epoch);
                        if (sm.n_first == 1) out_st(sm.out, i, tag, a);
                        for (int s1 = 1; s1 < sm.nsrc; s1++) {
                            a = __fadd_rn(a, vec_ld(sm.src[s1], i, epoch));
                            if (s1 + 1 == sm.n_first) out_st(sm.out, i, tag, a);
                        }
                        if (sm.n_first < sm.nsrc) out_st(sm.out2, i, tag, a);
                    }
                }
#endif
            } else if (blockIdx.x == 0) {
                const uint32_t tag = phase_epoch(epoch) + (uint32_t)pi + 1u;
                if (kind == FLOW_COPY) {
                    const FlowCopy & cp = d.cp;
                    for (int i = 8 * tid; i < cp.n; i += 8 * FL_CTHREADS) vec_copy8(cp.src, cp.src, false, cp.out, i, cp.n, tag, epoch);
                } else if (kind == FLOW_ADD) {
                    const FlowAdd & ad = d.ad;
                    for (int i = 8 * tid; i < ad.n; i += 8 * FL_CTHREADS) vec_copy8(ad.a, ad.b, true, ad.out, i, ad.n, tag, epoch);
                }
            }
            if (pre) cdesc[((pi + 1) & 1) * 96 + tid] = nextw;
        }
    }
    // ---- hand the epoch to the next launch: the last CTA to get here advances it past every tag of this launch
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        const unsigned old = atomicAdd(sync + 1, 1u);
        if (old == gridDim.x - 1) {
            sync[1] = 0u; sync[0] = phase_epoch(epoch) + (unsigned)n_phases + 1u;
#if FLOW_TP
            sync[2] = epoch.coll + (unsigned)n_coll;
#endif
            __threadfence();
        }
    }
}

int sm_count_of(int dev) {
    static int cnt[64] = {};
    dev &= 63;
    if (!cnt[dev]) {
        int n = 132;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        cnt[dev] = n;
    }
    return cnt[dev];
}

}  // namespace

#ifndef FLOW_SECONDARY
size_t flow_sync_bytes() { return 256; }
size_t flow_slot_bytes() { return FL_SLOT; }
int    flow_grid(int device) { return sm_count_of(device); }
cudaError_t launch_decode_flow_tp(const FlowProgram & prog, cudaStream_t st);   // decode_flow_tp.cu: the same kernel built with FLOW_TP (peer stores, collective epoch, sum phase)
#endif

#ifdef FLOW_SECONDARY
cudaError_t launch_decode_flow_tp(const FlowProgram & prog, cudaStream_t st) {
#else
cudaError_t launch_decode_flow(const FlowProgram & prog, cudaStream_t st) {
    if (prog.n_coll > 0) return launch_decode_flow_tp(prog, st);      // programs with a fused all-reduce need the tensor-parallel build
#endif
    if (prog.n_phases <= 0) return cudaSuccess;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr[64] = {};
    static int coop[64] = {};
    if (!attr[dev & 63]) {
        cudaError_t e = cudaFuncSetAttribute(decode_flow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FL_SMEM);
        if (e != cudaSuccess) return e;
        // the consumers of one CTA wait for producers in other CTAs: every CTA must be resident.  One CTA fits per SM by construction;
        // the cooperative launch makes the driver refuse the launch (instead of deadlocking) if the device cannot host the whole grid.
        int per_sm = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decode_flow_kernel, FL_THREADS, FL_SMEM);
        if (e != cudaSuccess) return e;
        if (per_sm < 1) return cudaErrorCooperativeLaunchTooLarge;
        cudaDeviceGetAttribute(&coop[dev & 63], cudaDevAttrCooperativeLaunch, dev);
        const char * ce = getenv("GGML_B200_FLOW_COOP");
        if (ce != nullptr && ce[0] == '0') coop[dev & 63] = 0;
        attr[dev & 63] = true;
    }
    static const int throttle = [] { const char * e = getenv("GGML_B200_FLOW_THROTTLE"); return e ? atoi(e) : 0; }();
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)sm_count_of(dev));
    cfg.blockDim = dim3(FL_THREADS);
    cfg.dynamicSmemBytes = FL_SMEM;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = coop[dev & 63] ? 1 : 0;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    note_launch();
    return cudaLaunchKernelEx(&cfg, decode_flow_kernel, prog.phases, prog.n_phases, prog.sync, prog.trace, throttle, prog.n_coll);
}

#ifndef FLOW_SECONDARY
// ================================================================================================ host: program builder
void FlowBuilder::reset(uint64_t * ll_pool, size_t ll_elems, int grid) {
    phases_.clear();
    produced_.clear();
    h_ptr_ = nullptr; h_ptr_copy_ = nullptr;
    pool_ = ll_pool; pool_elems_ = ll_elems; head_ = 0; seg_start_ = 0; n_coll_ = 0;
    grid_ = grid > 0 ? grid : 132;
}

void FlowBuilder::cut() {
    n_coll_ = 0;
    produced_.clear();
    h_ptr_ = nullptr; h_ptr_copy_ = nullptr;
    seg_start_ = phases_.size();
}

uint64_t * FlowBuilder::carve(size_t n) {
    n = (n + 1) & ~size_t(1);                                          // 16-byte granules (vector loads of two slots)
    if (pool_ == nullptr || n > pool_elems_) return nullptr;
    if (head_ + n > pool_elems_) head_ = 0;
    uint64_t * p = pool_ + head_;
    head_ += n;
    return p;
}

bool FlowBuilder::needs_cut(const void * p) const {
    auto it = produced_.find(p);
    return it != produced_.end() && it->second.ll == nullptr && it->second.plain_alias == nullptr;
}

FlowVec FlowBuilder::vec(const float * p) const {
    FlowVec v;
    v.plain = p; v.ll = nullptr; v.tag = 0; v.flags = 0;
    auto it = produced_.find(p);
    if (it != produced_.end()) {
        if (it->second.ll != nullptr) { v.ll = it->second.ll; v.tag = it->second.tag; }
        else if (it->second.plain_alias != nullptr) v.plain = it->second.plain_alias;
    }
    return v;
}

// The output of the phase about to be pushed (its index is phases_.size()).
FlowOut FlowBuilder::out(float * p, int n, bool want_ll) {
    FlowOut o;
    o.plain = p;
    o.ll = (want_ll && n <= 65536) ? carve((size_t)n) : nullptr;
    produced_[p] = Produced{o.ll, (uint32_t)(phases_.size() - seg_start_) + 1u, n, nullptr};
    if (p == h_ptr_) h_ptr_ = nullptr;                                 // (an in-place result replaces the vector the CTAs hold)
    if (p == h_ptr_copy_) h_ptr_copy_ = nullptr;
    return o;
}

static int flow_block_bytes(int t) { return t == T_Q4_K ? 144 : (t == T_Q5_K ? 176 : (t == T_Q6_K ? 210 : 0)); }

bool FlowBuilder::matvec_ok(const MatvecDesc & d) const {
    if (d.nmat < 1 || d.nmat > 3 || d.K <= 0 || d.K % 256 || d.K > FLOW_MAX_K) return false;
    if (d.norm_w && (d.K > FLOW_MAX_NORM_K || (reinterpret_cast<uintptr_t>(d.norm_w) & 15))) return false;
    if (d.norm_out && (!d.norm_w || (reinterpret_cast<uintptr_t>(d.norm_out) & 15))) return false;
    if (d.x == nullptr || (reinterpret_cast<uintptr_t>(d.x) & 15)) return false;
    if (d.mode == 2 && (d.nmat != 2 || d.M[0] != d.M[1] || d.type[0] != d.type[1])) return false;
    if (d.mode == 1 && (d.nmat != 1 || d.residual == nullptr)) return false;
    if (d.mode < 0 || d.mode > 2) return false;
    const int nblk = d.K / 256;
    if (nblk > 32 && (d.nmat != 1 || d.mode == 2)) return false;       // rows split over two warps: single matrix only
    for (int i = 0; i < d.nmat; i++) {
        const int bb = flow_block_bytes(d.type[i]);
        if (!bb || d.M[i] <= 0) return false;
        const uintptr_t wa = reinterpret_cast<uintptr_t>(d.w[i]);
        if (d.type[i] == T_Q6_K) { if ((wa & 1) || (d.row_stride[i] & 1)) return false; }
        else if ((wa & 15) || (d.row_stride[i] & 15)) return false;
        if (d.row_stride[i] < (int64_t)nblk * bb) return false;
        if (nblk > 32 && (d.M[i] + grid_ - 1) / grid_ + 1 > FLOW_PART_ROWS) return false;
    }
    if (needs_cut(d.x) || (d.residual && needs_cut(d.residual))) return false;
    return true;
}

bool FlowBuilder::add_matvec(const MatvecDesc & d) {
    if (!matvec_ok(d)) return false;
    FlowPhase ph;
    memset(&ph, 0, sizeof(ph));
    ph.kind = FLOW_MATVEC;
    FlowMatvec & m = ph.mv;
    const int nblk = d.K / 256;
    m.K = d.K; m.nmat = d.nmat; m.mode = d.mode; m.eps = d.eps; m.norm_w = d.norm_w; m.norm_out = d.norm_out;
    // plan: k-segments per row, blocks per segment, rows per warp step
    m.S = nblk > 32 ? 2 : 1;
    m.seg = (nblk + m.S - 1) / m.S;
    m.RP = (m.S == 1 && m.seg <= 16 && (m.seg & (m.seg - 1)) == 0) ? 32 / m.seg : 1;
    const int sub = d.mode == 2 ? 2 : 1;
    for (int i = 0; i < d.nmat; i++) {
        m.w[i] = d.w[i]; m.row_stride[i] = d.row_stride[i]; m.M[i] = d.M[i]; m.type[i] = d.type[i];
        m.rq[i] = d.M[i] / grid_; m.rr[i] = d.M[i] % grid_;
        const int bb = flow_block_bytes(d.type[i]);
        const int row_bytes = nblk * bb;
        const bool contiguous = m.S == 1 && d.row_stride[i] == row_bytes && (sub == 1 || d.row_stride[1] == row_bytes);
        int r_fit;
        if (contiguous) r_fit = (FL_SLOT / sub - 31) / row_bytes;
        else {
            const int pitch = (m.seg * bb + 16 + 15) & ~15;
            r_fit = FL_SLOT / (sub * pitch);
            if (r_fit * sub > 32) r_fit = 32 / sub;                    // one copy per lane of the producer warp
        }
        if (r_fit < 1) return false;
        const int rpc = (d.M[i] + grid_ - 1) / grid_;                  // rows per CTA
        int r_bal = rpc * m.S / (m.S == 1 ? FL_NW : 2 * FL_NPAIR);                // aim for at least one piece per consumer warp
        int R = r_fit < r_bal ? r_fit : r_bal;
        if (R < m.RP) R = m.RP <= r_fit ? m.RP : r_fit;
        if (R > m.RP) R = R / m.RP * m.RP;
        if (R < 1) R = 1;
        m.R[i] = R;
    }
    if (d.mode == 2) m.R[1] = m.R[0];
    m.x = vec(d.x);
    if (d.mode == 1) {
        m.resid_h = (h_ptr_ != nullptr && (d.residual == h_ptr_ || d.residual == h_ptr_copy_) && d.M[0] <= FLOW_MAX_H) ? 1 : 0;
        m.residual = vec(d.residual);
    }
    // the hidden state: a normalised input of at most FLOW_MAX_H floats is what later residual adds refer to
    m.keep_h = (d.norm_w != nullptr && d.K <= FLOW_MAX_H) ? 1 : 0;
    if (m.keep_h) { h_ptr_ = d.x; h_ptr_copy_ = nullptr; }
    if (d.norm_out != nullptr) produced_[d.norm_out] = Produced{nullptr, (uint32_t)(phases_.size() - seg_start_) + 1u, d.K, nullptr};   // plain only: readers must cut
    if (d.mode == 2) {
        m.out[0] = out(d.dst[0], d.M[0]);
    } else {
        for (int i = 0; i < d.nmat; i++) m.out[i] = out(d.dst[i], d.M[i]);
    }
    phases_.push_back(ph);
    return true;
}

bool FlowBuilder::attn_ok(const FlowAttn & a) const {
    if (a.head_dim != 128 || a.n_dims > 128 || a.n_dims % 2 || a.n_dims / 2 > 256) return false;
    if (a.rope_mode != 0 && a.rope_mode != 2) return false;
    if (a.n_head_kv <= 0 || a.n_head % a.n_head_kv || a.n_head > grid_) return false;
    if ((reinterpret_cast<uintptr_t>(a.kview) & 15) || (reinterpret_cast<uintptr_t>(a.vview) & 15) || a.k_nb1 % 16 || a.k_nb2 % 16 || a.v_nb1 % 16 || a.v_nb2 % 16) return false;
    if (a.n_kv <= 0) return false;
    return true;
}

bool FlowBuilder::add_attn(FlowAttn a, const float * q, const float * k, const float * v, float * dst, const FlowVec * q_vec) {
    if (!attn_ok(a) || (q_vec == nullptr && needs_cut(q)) || needs_cut(k) || needs_cut(v)) return false;
    // CTAs per head: split only when one CTA's 256 threads would walk more than 512 keys
    int n = grid_ / a.n_head;
    n = n < 1 ? 1 : (n > 8 ? 8 : n);
    const int want = (a.n_kv + 511) / 512;
    a.nsplit = want < n ? (want < 1 ? 1 : want) : n;
    a.part_ll = nullptr;
    if (a.nsplit > 1) {
        a.part_ll = carve((size_t)a.n_head * a.nsplit * (a.head_dim + 2));
        if (a.part_ll == nullptr) return false;
    }
    FlowPhase ph;
    memset(&ph, 0, sizeof(ph));
    ph.kind = FLOW_ATTN;
    a.q = q_vec ? *q_vec : vec(q); a.k = vec(k); a.v = vec(v);
    a.out = out(dst, a.n_head * a.head_dim);
    ph.at = a;
    phases_.push_back(ph);
    return true;
}

bool FlowBuilder::add_copy(const float * src, float * dst, int n) {
    if (needs_cut(src) || n <= 0) return false;
    // Inside the program the copy is an ALIAS: later phases read the source's slots (or its memory, if it was complete before
    // the launch), so nothing waits for this phase; it only materialises the ggml tensor for whoever reads it after the launch.
    FlowPhase ph;
    memset(&ph, 0, sizeof(ph));
    ph.kind = FLOW_COPY;
    ph.cp.src = vec(src); ph.cp.n = n;
    ph.cp.out.plain = dst; ph.cp.out.ll = nullptr;
    Produced pr{ph.cp.src.ll ? const_cast<uint64_t *>(ph.cp.src.ll) : nullptr, ph.cp.src.tag, n, ph.cp.src.ll ? nullptr : ph.cp.src.plain};
    const bool was_h = h_ptr_ == src;
    produced_[dst] = pr;
    if (dst == h_ptr_) h_ptr_ = nullptr;
    if (was_h && dst != src) h_ptr_copy_ = dst;                        // the copy names the same values the CTAs hold as hidden state
    phases_.push_back(ph);
    return true;
}

bool FlowBuilder::fuse_allreduce(FlowBuilder * const * fb, int n, float * const * tensors, int nelem, uint64_t * const * xpool, size_t xpool_elems, size_t & xoff) {
    if (n < 2 || n > FLOW_MAX_PEERS || nelem <= 0 || nelem > 65536) return false;
    const size_t need = ((size_t)n * nelem + 1) & ~size_t(1);
    if (xoff + need > xpool_elems) return false;
    const int coll = fb[0]->n_coll_;
    for (int d = 0; d < n; d++) {
        FlowBuilder & b = *fb[d];
        if (b.phases_.size() <= b.seg_start_ || b.n_coll_ != coll || xpool[d] == nullptr) return false;
        const FlowPhase & last = b.phases_.back();
        if (last.kind != FLOW_MATVEC || last.mv.nmat != 1 || last.mv.mode == 2 || last.mv.npeer != 0 || last.mv.M[0] != nelem || last.mv.out[0].plain != tensors[d]) return false;
    }
    for (int d = 0; d < n; d++) {
        FlowBuilder & b = *fb[d];
        FlowMatvec & mv = b.phases_.back().mv;
        for (int j = 0; j < n; j++) mv.peer[j] = xpool[j] + xoff + (size_t)d * nelem;     // GPU d's partial lands in slot d of every GPU
        mv.npeer = n; mv.coll = (uint32_t)coll;
        FlowPhase ph;
        memset(&ph, 0, sizeof(ph));
        ph.kind = FLOW_SUM;
        for (int s = 0; s < n; s++) {
            FlowVec & v = ph.sm.src[s];
            v.plain = nullptr; v.ll = xpool[d] + xoff + (size_t)s * nelem; v.tag = (uint32_t)coll + 1u; v.flags = FLOW_VEC_COLL;
        }
        ph.sm.nsrc = n; ph.sm.n = nelem; ph.sm.n_first = n;
        ph.sm.out = b.out(tensors[d], nelem);              // the reduced vector replaces the partial one under the same name
        b.phases_.push_back(ph);
        b.n_coll_++;
    }
    xoff += need;
    return true;
}

bool FlowBuilder::add_add(const float * a, const float * b, float * dst, int n) {
    if (needs_cut(a) || needs_cut(b) || n <= 0) return false;
    if (phases_.size() > seg_start_) {
        // the residual ADD right after a fused all-reduce joins its sum phase as one more source (same order of additions: the reduced
        // vector first, then the residual) -- one dependency hop less per all-reduce; the reduced vector itself is still written
        FlowPhase & last = phases_.back();
        if (last.kind == FLOW_SUM && last.sm.n == n && last.sm.n_first == last.sm.nsrc && last.sm.nsrc < FLOW_MAX_PEERS + 1 &&
            (last.sm.out.plain == a || last.sm.out.plain == b)) {
            const float * other = last.sm.out.plain == a ? b : a;
            last.sm.src[last.sm.nsrc++] = vec(other);
            last.sm.out2 = out(dst, n);
            return true;
        }
    }
    FlowPhase ph;
    memset(&ph, 0, sizeof(ph));
    ph.kind = FLOW_ADD;
    ph.ad.a = vec(a); ph.ad.b = vec(b); ph.ad.n = n;
    ph.ad.out = out(dst, n);
    phases_.push_back(ph);
    return true;
}

#endif  // FLOW_SECONDARY

}  // namespace qmm
