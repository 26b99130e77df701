// gemv3.cu -- the fused decode mat-vec: what one Llama layer needs per token, in as few launches as possible.
//
// The first whole-model run through the plugin showed decode is not bandwidth- but LAUNCH-bound: ~600 kernels per token
// (19 per layer), most of them 3-4 us stubs around 5-10 us mat-vecs.  This kernel folds the stubs into the mat-vec:
//
//   prologue   the activation arrives as f32.  Optionally RMS_NORM * weight (ggml RMS_NORM + MUL) is applied, then the
//              vector is quantised to the CPU's Q8_K integers -- by every CTA for itself, in shared memory, while the
//              weight stream is already in flight (the cp.async.bulk ring is primed BEFORE the activation is touched;
//              with programmatic dependent launch that prefetch even overlaps the previous kernel's tail).
//              No separate rms_norm / quantize launches, no round trip of the quantised vector through HBM.
//   body       gemv2's bulk-copy ring + block-per-lane dot products, over up to 3 weight matrices of the same type that
//              share the activation (attn_q|k|v, ffn_gate|up) -- one launch instead of three.
//   epilogue   store | + residual (ggml ADD) | SwiGLU pair: rows r of matrix 0 (gate) and matrix 1 (up) are produced by
//              the same warp and written as silu(gate) * up (ggml GLU SWIGLU) -- the gate/up vectors never reach HBM.
//
// Arithmetic is unchanged (same Q8_K integers, same integer dot products, same fp32 combine), so the parity bounds of
// gemv2 apply; the fused RMS_NORM sums float squares in double like the CPU (ops.cpp ggml_compute_forward_rms_norm_f32).
// N = 1 only (the decode regime).  Algorithmic bytes: sum_i M_i * K/256 * BB.  Roofline: HBM.
#include <cstdio>
#include <cstdlib>

#include "gemv_blockdot.cuh"

namespace qmm {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

template <int T>
__global__ void __launch_bounds__(G2<T>::WARPS * 32) gemv3_kernel(const FusedGemvArgs p) {
    using C = G2<T>;
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ int gqueue[C::WARPS][8];                               // per warp: ids of the row groups it has claimed, in order
    __shared__ double red[C::WARPS];
    pdl_launch_dependents();                                          // let the next kernel's CTAs queue up behind ours
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int K = p.K;
    const int nblk = K >> 8;
    const int nks = (nblk + 7) >> 3;
    const int nsub = p.mode == 2 ? 2 : 1;                             // SwiGLU pair: gate group then up group

    uint64_t * bars = reinterpret_cast<uint64_t *>(smem);
    uint8_t * act_qs = smem + 256;
    uint8_t * act_bs = act_qs + (size_t)nblk * C::ACTB;
    float * act_d = reinterpret_cast<float *>(act_bs + (size_t)nblk * C::BSB);
    float * xf = reinterpret_cast<float *>((reinterpret_cast<uintptr_t>(act_d + nblk) + 15) & ~uintptr_t(15));   // K floats when x is f32
    uint8_t * ring0 = reinterpret_cast<uint8_t *>(xf + (p.x ? K : 0));
    ring0 = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ring0) + 127) & ~uintptr_t(127));
    uint8_t * ring = ring0 + (size_t)warp * C::STAGES * C::SLOT;
    uint64_t * mybar = bars + warp * C::STAGES;


    // ---- row groups over the concatenated matrices (SwiGLU: groups of matrix 0, each paired with the same rows of matrix 1)
    const int G0 = (p.M[0] + 3) >> 2, G1 = p.nmat > 1 ? (p.M[1] + 3) >> 2 : 0, G2_ = p.nmat > 2 ? (p.M[2] + 3) >> 2 : 0;
    const int ngroups = p.mode == 2 ? G0 : G0 + G1 + G2_;
    const int nwarps_total = (int)gridDim.x * C::WARPS;
    // Work distribution: the first group of every warp is static (group = global warp id, consecutive warps stream
    // consecutive rows); every further group is claimed from a global ticket counter, so no warp idles while another
    // still has two groups to go (a static split left ~1/3 of the machine idle in the last third of mid-size mat-vecs).
    auto next_group = [&](int prev) -> int {
        if (p.counter) return nwarps_total + (int)atomicAdd(p.counter, 1u);
        return prev + nwarps_total;
    };

    // kernel parameters are indexed with selects, not dynamically (dynamic indexing would spill the struct to local memory)
    auto Wp = [&](int m) { return m == 0 ? p.w[0] : (m == 1 ? p.w[1] : p.w[2]); };
    auto RS = [&](int m) { return m == 0 ? p.row_stride[0] : (m == 1 ? p.row_stride[1] : p.row_stride[2]); };
    auto Mm = [&](int m) { return m == 0 ? p.M[0] : (m == 1 ? p.M[1] : p.M[2]); };
    auto Dp = [&](int m) { return m == 0 ? p.dst[0] : (m == 1 ? p.dst[1] : p.dst[2]); };
    auto Rp = [&](int m) { return m == 0 ? p.residual[0] : (m == 1 ? p.residual[1] : p.residual[2]); };
    auto locate = [&](int g, int sub, int & mat, int & row0) {
        if (p.mode == 2) { mat = sub; row0 = 4 * g; return; }
        if (g < G0) { mat = 0; row0 = 4 * g; }
        else if (g < G0 + G1) { mat = 1; row0 = 4 * (g - G0); }
        else { mat = 2; row0 = 4 * (g - G0 - G1); }
    };

    auto issue = [&](int g, int sub, int ks, int slot) {              // lane 0 only
        int mat, row0;
        locate(g, sub, mat, row0);
        const int nb = min(8, nblk - 8 * ks);
        uint8_t * sl = ring + slot * C::SLOT;
        uint32_t tx = 0, cnt[4];
        const uint8_t * src[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            cnt[r] = 0;
            if (row0 + r < Mm(mat)) {
                const uint8_t * gp = Wp(mat) + (int64_t)(row0 + r) * RS(mat) + (int64_t)ks * C::PIECEB;
                const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(gp) & 15);
                src[r] = gp - off;
                cnt[r] = (off + (uint32_t)(nb * C::BB) + 15u) & ~15u;
                tx += cnt[r];
            }
        }
        mbar_expect_tx(mybar + slot, tx);
#pragma unroll
        for (int r = 0; r < 4; r++)
            if (cnt[r]) bulk_g2s(sl + r * C::PIECE, src[r], cnt[r], mybar + slot);
    };

    // ---- prime the weight stream: it depends on nothing the previous kernel produced
    int ig = (int)blockIdx.x * C::WARPS + warp, isub = 0, iks = 0, islot = 0, qtail = 1;   // lane 0's issue cursor
    auto advance_issue = [&]() {
        if (++iks == nks) {
            iks = 0;
            if (++isub == nsub) { isub = 0; ig = next_group(ig); gqueue[warp][qtail & 7] = ig; qtail++; }
        }
        islot = islot + 1 == C::STAGES ? 0 : islot + 1;
    };
    bool primed = false;
    auto prime = [&]() {
        if (primed) return;
        primed = true;
        if (lane == 0) {
#pragma unroll
            for (int s = 0; s < C::STAGES; s++) mbar_init(mybar + s, 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
        if (lane == 0) {
            gqueue[warp][0] = ig;
#pragma unroll
            for (int s = 0; s < C::STAGES - 1; s++)
                if (ig < ngroups) { issue(ig, isub, iks, islot); advance_issue(); }
        }
    };

    // ---- keep HBM busy across the launch boundary: ask the L2 to start pulling in the NEXT launch's weights now.  A decode
    //      mat-vec is a latency chain (launch -> prologue -> first bytes -> compute -> tail) during which HBM mostly idles;
    //      the next launch then finds its weights in the 50 MB L2.  Fire-and-forget bulk prefetches, one slice per CTA.
    if (warp == C::WARPS - 1) {
#pragma unroll
        for (int m = 0; m < 3; m++) {
            const uint8_t * nw = m == 0 ? p.next_w[0] : (m == 1 ? p.next_w[1] : p.next_w[2]);
            const int64_t nbytes = m == 0 ? p.next_bytes[0] : (m == 1 ? p.next_bytes[1] : p.next_bytes[2]);
            if (nw == nullptr || nbytes <= 0) continue;
            const int64_t per_cta = ((nbytes + gridDim.x - 1) / gridDim.x + 4095) & ~int64_t(4095);
            const int64_t lo = (int64_t)blockIdx.x * per_cta;
            const int64_t hi = lo + per_cta < nbytes ? lo + per_cta : nbytes;
            for (int64_t off = lo + (int64_t)lane * 4096; off < hi; off += 32 * 4096) {
                const uint32_t sz = (uint32_t)((hi - off < 4096 ? hi - off : 4096) & ~int64_t(15));
                if (sz) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;\n" ::"l"(nw + off), "r"(sz) : "memory");
            }
        }
    }

    // ---- activation prologue (everything below reads the previous kernel's output)
    // PDL note: this grid was scheduled (and its SMs' L1 invalidated) BEFORE the producer finished, and producer CTAs
    // sharing an SM with us may since have pulled lines of the very buffers we are about to read into that L1 (e.g. the
    // in-place residual add reads 4 floats of a line whose other 28 floats are written by other SMs).  Every load of
    // producer data after the wait therefore bypasses L1 (ld.global.cg).
    pdl_wait();
    if (p.x != nullptr) {
        // phase 1: x -> shared memory (coalesced float4), sum of squares in double when normalising; the norm weights are
        // requested in the same breath so that both L2 round trips overlap
        constexpr int NV = 8;                                         // float4 per thread: K <= 8192 with 192 threads needs 11 -> two rounds
        double acc = 0.0;
        const int nf4 = K / 4;
        for (int base = 0; base < nf4; base += NV * (int)blockDim.x) {
            float4 xv[NV], wv[NV];
#pragma unroll
            for (int u = 0; u < NV; u++) {
                const int i = base + u * (int)blockDim.x + (int)threadIdx.x;
                if (i < nf4) {
                    xv[u] = __ldcg(reinterpret_cast<const float4 *>(p.x) + i);      // L2 only: see the PDL note above
                    if (p.has_norm) wv[u] = __ldg(reinterpret_cast<const float4 *>(p.norm_w) + i);
                }
            }
            // The activation loads above are in flight; only NOW flood the memory system with the weight stream.  (Priming
            // first put ~16 MB of bulk copies ahead of these few KB in the memory queues and the prologue waited ~10 us.)
            prime();
            if (p.has_norm) {
#pragma unroll
                for (int u = 0; u < NV; u++) {
                    const int i = base + u * (int)blockDim.x + (int)threadIdx.x;
                    if (i < nf4) acc += (double)__fmul_rn(xv[u].x, xv[u].x) + (double)__fmul_rn(xv[u].y, xv[u].y) + (double)__fmul_rn(xv[u].z, xv[u].z) + (double)__fmul_rn(xv[u].w, xv[u].w);
                }
            }
            if (p.has_norm && nf4 <= NV * (int)blockDim.x) {
                // single round (K <= 6144): finish the norm here with x and w still in registers
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
                if (lane == 0) red[warp] = acc;
                __syncthreads();
                double tot = 0.0;
#pragma unroll
                for (int i = 0; i < C::WARPS; i++) tot += red[i];
                const float mean = (float)(tot / (double)K);
                const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, p.eps)));
#pragma unroll
                for (int u = 0; u < NV; u++) {
                    const int i = base + u * (int)blockDim.x + (int)threadIdx.x;
                    if (i < nf4) {
                        float4 v = xv[u];
                        v.x = __fmul_rn(__fmul_rn(v.x, scale), wv[u].x); v.y = __fmul_rn(__fmul_rn(v.y, scale), wv[u].y);
                        v.z = __fmul_rn(__fmul_rn(v.z, scale), wv[u].z); v.w = __fmul_rn(__fmul_rn(v.w, scale), wv[u].w);
                        reinterpret_cast<float4 *>(xf)[i] = v;
                    }
                }
            } else {
#pragma unroll
                for (int u = 0; u < NV; u++) {
                    const int i = base + u * (int)blockDim.x + (int)threadIdx.x;
                    if (i < nf4) reinterpret_cast<float4 *>(xf)[i] = xv[u];
                }
            }
        }
        if (p.has_norm && nf4 > NV * (int)blockDim.x) {
            // multi-round (K > 6144): x is staged raw; reduce, then normalise in place
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) red[warp] = acc;
            __syncthreads();
            double tot = 0.0;
#pragma unroll
            for (int i = 0; i < C::WARPS; i++) tot += red[i];
            const float mean = (float)(tot / (double)K);
            const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, p.eps)));
            for (int i = threadIdx.x; i < nf4; i += blockDim.x) {
                float4 v = reinterpret_cast<float4 *>(xf)[i];
                const float4 w = __ldg(reinterpret_cast<const float4 *>(p.norm_w) + i);
                v.x = __fmul_rn(__fmul_rn(v.x, scale), w.x); v.y = __fmul_rn(__fmul_rn(v.y, scale), w.y);
                v.z = __fmul_rn(__fmul_rn(v.z, scale), w.z); v.w = __fmul_rn(__fmul_rn(v.w, scale), w.w);
                reinterpret_cast<float4 *>(xf)[i] = v;
            }
        }
        __syncthreads();
        // phase 3: one warp per 256-block, from shared memory; lane l owns elements 8l .. 8l+7
        for (int b = warp; b < nblk; b += C::WARPS) {
            float v[8];
            const float4 a0 = reinterpret_cast<const float4 *>(xf + 256 * b)[2 * lane], a1 = reinterpret_cast<const float4 *>(xf + 256 * b)[2 * lane + 1];
            v[0] = a0.x; v[1] = a0.y; v[2] = a0.z; v[3] = a0.w; v[4] = a1.x; v[5] = a1.y; v[6] = a1.z; v[7] = a1.w;
            // quantize_row_q8_K_ref (ggml-quants.c:2768-2805): the FIRST element of largest magnitude decides scale and sign.
            // |v| as uint orders like the float; NaN never wins (mapped to 0).
            unsigned mloc = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) { const unsigned a = (v[i] == v[i]) ? (__float_as_uint(v[i]) & 0x7fffffffu) : 0u; mloc = a > mloc ? a : mloc; }
            unsigned mall = mloc;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { const unsigned t = __shfl_xor_sync(0xffffffffu, mall, o); mall = t > mall ? t : mall; }
            const unsigned holders = __ballot_sync(0xffffffffu, mloc == mall);
            const int wl = __ffs((int)holders) - 1;                    // first lane holding the maximum
            float mine = 0.0f;
#pragma unroll
            for (int i = 7; i >= 0; i--) mine = ((__float_as_uint(v[i]) & 0x7fffffffu) == mall && v[i] == v[i]) ? v[i] : mine;   // first index in this lane
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
            *reinterpret_cast<uint2 *>(act_qs + (size_t)b * C::ACTB + 8 * lane) = packed;
            const int s8 = q[0] + q[1] + q[2] + q[3] + q[4] + q[5] + q[6] + q[7];
            const int s16 = s8 + __shfl_xor_sync(0xffffffffu, s8, 1);              // bsums: groups of 16 = lane pairs
            if (T == T_Q6_K) {
                if ((lane & 1) == 0) reinterpret_cast<int16_t *>(act_bs + (size_t)b * C::BSB)[lane >> 1] = (int16_t)s16;
            } else {
                const int s32_ = s16 + __shfl_xor_sync(0xffffffffu, s16, 2);       // Q4_K/Q5_K use sums of 32
                if ((lane & 3) == 0) reinterpret_cast<int16_t *>(act_bs + (size_t)b * C::BSB)[lane >> 2] = (int16_t)s32_;
            }
            if (lane == 0) act_d[b] = d;
        }
    } else {
        const int8_t * gq = p.act.qs;
        for (int i = threadIdx.x; i < nblk * 16; i += blockDim.x)
            *reinterpret_cast<uint4 *>(act_qs + (size_t)(i >> 4) * C::ACTB + 16 * (i & 15)) = __ldcg(reinterpret_cast<const uint4 *>(gq + 16 * (size_t)i));
        const int16_t * gb = p.act.bsums;
        if (T == T_Q6_K) {
            for (int i = threadIdx.x; i < nblk * 16; i += blockDim.x) reinterpret_cast<int16_t *>(act_bs + (size_t)(i >> 4) * C::BSB)[i & 15] = __ldcg(gb + i);
        } else {
            for (int i = threadIdx.x; i < nblk * 8; i += blockDim.x)
                reinterpret_cast<int16_t *>(act_bs + (size_t)(i >> 3) * C::BSB)[i & 7] = (int16_t)(__ldcg(gb + 2 * i) + __ldcg(gb + 2 * i + 1));
        }
        for (int i = threadIdx.x; i < nblk; i += blockDim.x) act_d[i] = __ldcg(p.act.d + i);
    }
    prime();
    __syncthreads();

    const int r = lane >> 3, j = lane & 7;
    float acc = 0.0f, gate = 0.0f;
    int qhead = 0, csub = 0, cks = 0, cslot = 0;
    int cg = gqueue[warp][0];
    uint32_t phase_bits = 0;
    while (cg < ngroups) {
        if (lane == 0 && ig < ngroups) { issue(ig, isub, iks, islot); advance_issue(); }
        mbar_wait(mybar + cslot, (phase_bits >> cslot) & 1u);
        phase_bits ^= 1u << cslot;

        int mat, row0;
        locate(cg, csub, mat, row0);
        const int row = row0 + r;
        const int kb = 8 * cks + j;
        if (row < Mm(mat) && kb < nblk) {
            const uint8_t * gp = Wp(mat) + (int64_t)row * RS(mat) + (int64_t)cks * C::PIECEB;
            const uint8_t * wb = ring + cslot * C::SLOT + r * C::PIECE + (int)(reinterpret_cast<uintptr_t>(gp) & 15) + j * C::BB;
            acc += BlockDot<T>::run(wb, act_qs + (size_t)kb * C::ACTB, act_bs + (size_t)kb * C::BSB, act_d[kb]);
        }
        if (cks + 1 == nks) {                                         // rows of this (group, sub) are complete
            float v = acc;
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            acc = 0.0f;
            if (p.mode == 2 && csub == 0) {
                gate = v;                                             // keep silu input until the paired "up" rows arrive
            } else if (j == 0 && row < Mm(mat)) {
                if (p.mode == 2) {
                    const float silu = __fdiv_rn(gate, __fadd_rn(1.0f, expf(-gate)));
                    p.dst[0][row] = __fmul_rn(silu, v);
                } else if (p.mode == 1) {
                    Dp(mat)[row] = __fadd_rn(v, __ldcg(Rp(mat) + row));
                } else {
                    Dp(mat)[row] = v;
                }
            }
        }
        __syncwarp();                                                 // slot reusable; lane 0's queue writes visible to the warp
        cslot = cslot + 1 == C::STAGES ? 0 : cslot + 1;
        if (++cks == nks) {
            cks = 0;
            if (++csub == nsub) { csub = 0; qhead++; cg = gqueue[warp][qhead & 7]; }
        }
    }
}

template <int T>
static cudaError_t launch3(const FusedGemvArgs & a, cudaStream_t st) {
    using C = G2<T>;
    const int nblk = a.K >> 8;
    const size_t smem = 256 + (size_t)nblk * (C::ACTB + C::BSB + 4) + (a.x ? (size_t)a.K * 4 + 16 : 0) + 128 + (size_t)C::WARPS * C::STAGES * C::SLOT;
    if (smem > 227 * 1024 - 512) return cudaErrorNotSupported;
    static int sm_count[64] = {};
    static bool attr[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (!attr[dev]) {
        int n = 132;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sm_count[dev] = n;
        cudaError_t e = cudaFuncSetAttribute(gemv3_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 512);   // the kernel also has a little static shared memory
        if (e != cudaSuccess) { if (getenv("GGML_B200_DEBUG")) fprintf(stderr, "gemv3 cudaFuncSetAttribute failed: %s\n", cudaGetErrorString(e)); return e; }
        attr[dev] = true;
    }
    int per_sm = (int)((227 * 1024) / (smem + 1024));
    static const int cap = getenv("GGML_B200_GEMV_CTAS_PER_SM") ? atoi(getenv("GGML_B200_GEMV_CTAS_PER_SM")) : 4;
    if (per_sm > cap) per_sm = cap;
    int gx = sm_count[dev] * (per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm));
    int ngroups = (a.M[0] + 3) / 4;
    if (a.mode != 2) for (int i = 1; i < a.nmat; i++) ngroups += (a.M[i] + 3) / 4;
    if (gx > ngroups) gx = ngroups;
    if (gx < 1) gx = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)gx);
    cfg.blockDim = dim3(C::WARPS * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = a.pdl ? 1 : 0;
    cfg.attrs = at;
    cfg.numAttrs = (a.pdl || pdl_attr_always()) ? 1 : 0;
    note_launch();
    const cudaError_t e = cudaLaunchKernelEx(&cfg, gemv3_kernel<T>, a);
    if (e != cudaSuccess && getenv("GGML_B200_DEBUG"))
        fprintf(stderr, "gemv3 launch failed: %s  grid=%d block=%d smem=%zu nmat=%d K=%d M0=%d mode=%d pdl=%d norm=%d\n", cudaGetErrorString(e), gx,
                C::WARPS * 32, smem, a.nmat, a.K, a.M[0], a.mode, a.pdl, a.has_norm);
    return e;
}

// cudaErrorNotSupported: the caller falls back to separate kernels.
cudaError_t launch_fused_gemv(int type, const FusedGemvArgs & a, cudaStream_t st) {
    if (a.nmat < 1 || a.nmat > 3 || a.K <= 0 || a.K % 256) return cudaErrorNotSupported;
    if (a.mode == 2 && (a.nmat != 2 || a.M[0] != a.M[1])) return cudaErrorInvalidValue;
    if (a.x != nullptr && (reinterpret_cast<uintptr_t>(a.x) & 15)) return cudaErrorNotSupported;
    if (a.has_norm && (a.x == nullptr || a.norm_w == nullptr || (reinterpret_cast<uintptr_t>(a.norm_w) & 15))) return cudaErrorNotSupported;
    for (int i = 0; i < a.nmat; i++) {
        const uintptr_t wa = reinterpret_cast<uintptr_t>(a.w[i]);
        if (type == T_Q4_K || type == T_Q5_K) { if ((wa & 15) || (a.row_stride[i] & 15)) return cudaErrorNotSupported; }
        else if ((wa & 1) || (a.row_stride[i] & 1)) return cudaErrorNotSupported;
    }
    switch (type) {
        case T_Q4_K: return launch3<T_Q4_K>(a, st);
        case T_Q5_K: return launch3<T_Q5_K>(a, st);
        case T_Q6_K: return launch3<T_Q6_K>(a, st);
    }
    return cudaErrorNotSupported;
}

}  // namespace qmm
