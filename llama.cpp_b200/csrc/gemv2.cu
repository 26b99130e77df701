// gemv2.cu -- decode mat-vec, second generation ("block per lane, bulk-copy ring"), K-quant formats.
//
// Same contract as gemv.cu (dst[M, n] = W[M, K] . act[K, n], n <= NCOLS_MAX) but organised around what the first
// ncu/bench pass showed: gemv.cu is ISSUE-bound (~1.4 instructions per weight: per-lane cp.async address math,
// per-32-weight header decode, activation re-loads), not HBM-bound.  Here:
//
//   * HBM -> shared memory moves with cp.async.bulk (the TMA unit's 1-D bulk copy): ONE instruction by ONE lane per
//     row piece, completion on an mbarrier (complete_tx).  No per-lane address math, no LSU issue slots.
//     A warp owns 4 consecutive rows ("row group"); per k-step it brings in 4 pieces of 8 blocks (2048 weights,
//     1152 B for Q4_K) into a private ring of D slots; (D-1) slots x 4.6 KB x resident warps stay in flight.
//   * lane = (row-in-group r = lane/8, block j = lane%8): a lane consumes one WHOLE 256-weight block per k-step, so
//     the fp16 super-scales and the 6-bit scale/min unpacking are done once per 256 weights, not per 32.
//   * high nibbles are multiplied in place: dp4a((q & 0xF0F0F0F0) as unsigned, a) = 16 * sum(hi*a), shifted down once
//     per sub-block -- one LOP instead of SHF+LOP per word.
//   * the quantised activations (CPU-identical Q8_K integers) are staged ONCE per CTA into shared memory in a skewed
//     layout (272-byte block pitch) so the 8 lanes of a row read 8 different blocks bank-conflict free.
//   * reduction: 3 xor-shuffles inside each 8-lane group per row group (not 5 per row).
//
// Algorithmic bytes per launch: M * K/256 * BB (weights once).  Roofline: HBM.
#include "gemv_blockdot.cuh"

namespace qmm {

// ---------------------------------------------------------------- kernel
template <int T, int NCOLS>
__global__ void __launch_bounds__(G2<T>::WARPS * 32) gemv2_kernel(const GemvArgs p) {
    using C = G2<T>;
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int K = p.K, M = p.M;
    const int nblk = K >> 8;
    const int nks = (nblk + 7) >> 3;                                  // k-steps per row group
    const int row_bytes = nblk * C::BB;

    // smem carve: barriers | act qs (NCOLS x nblk x 272) | act bsums (NCOLS x nblk x BSB) | act d (NCOLS x nblk x 4) | ring
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem);
    static_assert(C::WARPS * C::STAGES * 8 <= 256, "barrier area");
    uint8_t * act_qs = smem + 256;
    uint8_t * act_bs = act_qs + (size_t)NCOLS * nblk * C::ACTB;
    float * act_d = reinterpret_cast<float *>(act_bs + (size_t)NCOLS * nblk * C::BSB);
    uint8_t * ring0 = reinterpret_cast<uint8_t *>(act_d + (size_t)NCOLS * nblk);
    ring0 = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(ring0) + 127) & ~uintptr_t(127));
    uint8_t * ring = ring0 + (size_t)warp * C::STAGES * C::SLOT;
    uint64_t * mybar = bars + warp * C::STAGES;

    const int z = blockIdx.y;
    const uint8_t * wbase = p.w;
    int col0 = 0;
    if (p.ids != nullptr) {
        const int t = z / p.n_used, s = z - t * p.n_used;
        const int e = p.ids[(int64_t)t * p.ids_stride + s];
        if (e < 0 || e >= p.n_expert) return;
        wbase += (int64_t)e * p.expert_stride;
        col0 = t * p.nb1 + (s % p.nb1);
    }

    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < C::STAGES; s++) mbar_init(mybar + s, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");

    // ---- this warp's row groups: group id g = blockIdx.x + gridDim.x * (warp + WARPS * i)
    const int ngroups = (M + 3) >> 2;
    const int gstride = (int)gridDim.x * C::WARPS;
    const int g0 = (int)blockIdx.x + (int)gridDim.x * warp;
    const int ngw = g0 < ngroups ? (ngroups - 1 - g0) / gstride + 1 : 0;
    const int total = ngw * nks;

    auto issue = [&](int gi, int ks, int slot) {                      // lane 0 only
        const int row0 = 4 * (g0 + gi * gstride);
        const int nb = min(8, nblk - 8 * ks);
        uint8_t * sl = ring + slot * C::SLOT;
        uint32_t tx = 0;
        uint32_t offs[4], cnt[4];
        const uint8_t * src[4];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            cnt[r] = 0;
            if (row0 + r < M) {
                const uint8_t * g = wbase + (int64_t)(row0 + r) * p.row_stride + (int64_t)ks * C::PIECEB;
                const uint32_t off = (uint32_t)(reinterpret_cast<uintptr_t>(g) & 15);
                src[r] = g - off; offs[r] = off;
                cnt[r] = (off + (uint32_t)(nb * C::BB) + 15u) & ~15u;
                tx += cnt[r];
            }
        }
        mbar_expect_tx(mybar + slot, tx);
#pragma unroll
        for (int r = 0; r < 4; r++)
            if (cnt[r]) bulk_g2s(sl + r * C::PIECE, src[r], cnt[r], mybar + slot);
        (void)offs;
    };

    // ---- start the weight stream first (it does not depend on the activations), then stage the activations
    int igi = 0, iks = 0, islot = 0;
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < C::STAGES - 1; s++) {
            if (igi < ngw) { issue(igi, iks, islot); if (++iks == nks) { iks = 0; igi++; } islot = islot + 1 == C::STAGES ? 0 : islot + 1; }
        }
    }

    for (int n = 0; n < NCOLS; n++) {
        const int8_t * gq = p.act.qs + (int64_t)(col0 + n) * p.act.qs_stride;
        for (int i = threadIdx.x; i < nblk * 16; i += blockDim.x) {   // 16-byte chunks
            const int blk = i >> 4, c = i & 15;
            *reinterpret_cast<uint4 *>(act_qs + ((size_t)n * nblk + blk) * C::ACTB + 16 * c) = *reinterpret_cast<const uint4 *>(gq + 16 * (size_t)i);
        }
        const int16_t * gb = p.act.bsums + (int64_t)(col0 + n) * p.act.bs_stride;
        if (T == T_Q6_K) {
            for (int i = threadIdx.x; i < nblk * 16; i += blockDim.x)
                reinterpret_cast<int16_t *>(act_bs + ((size_t)n * nblk + (i >> 4)) * C::BSB)[i & 15] = gb[i];
        } else {
            for (int i = threadIdx.x; i < nblk * 8; i += blockDim.x)       // sums over sub-blocks of 32
                reinterpret_cast<int16_t *>(act_bs + ((size_t)n * nblk + (i >> 3)) * C::BSB)[i & 7] = (int16_t)(gb[2 * i] + gb[2 * i + 1]);
        }
        const float * gd = p.act.d + (int64_t)(col0 + n) * p.act.d_stride;
        for (int i = threadIdx.x; i < nblk; i += blockDim.x) act_d[(size_t)n * nblk + i] = gd[i];
    }
    __syncthreads();                                                  // barriers initialised + activations staged
    if (total == 0) return;

    const int r = lane >> 3, j = lane & 7;
    float * dst = p.dst + (int64_t)z * NCOLS * p.ldd;
    const float * res = p.residual ? p.residual + (int64_t)z * NCOLS * p.ldd : nullptr;

    float acc[NCOLS];
#pragma unroll
    for (int n = 0; n < NCOLS; n++) acc[n] = 0.0f;

    int cgi = 0, cks = 0, cslot = 0;
    uint32_t phase_bits = 0;                                          // bit s = parity to wait for on slot s
    for (int i = 0; i < total; i++) {
        if (lane == 0 && igi < ngw) {
            issue(igi, iks, islot);
            if (++iks == nks) { iks = 0; igi++; }
            islot = islot + 1 == C::STAGES ? 0 : islot + 1;
        }
        mbar_wait(mybar + cslot, (phase_bits >> cslot) & 1u);
        phase_bits ^= 1u << cslot;

        const int row = 4 * (g0 + cgi * gstride) + r;
        const int kb = 8 * cks + j;
        if (row < M && kb < nblk) {
            const uint8_t * g = wbase + (int64_t)row * p.row_stride + (int64_t)cks * C::PIECEB;
            const uint8_t * wb = ring + cslot * C::SLOT + r * C::PIECE + (int)(reinterpret_cast<uintptr_t>(g) & 15) + j * C::BB;
#pragma unroll
            for (int n = 0; n < NCOLS; n++) {
                const size_t ab = (size_t)n * nblk + kb;
                acc[n] += BlockDot<T>::run(wb, act_qs + ab * C::ACTB, act_bs + ab * C::BSB, act_d[ab]);
            }
        }
        if (cks + 1 == nks) {                                         // row group finished
#pragma unroll
            for (int n = 0; n < NCOLS; n++) {
                float v = acc[n];
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                if (j == 0 && row < M) {
                    const int64_t di = (int64_t)n * p.ldd + row;
                    dst[di] = res ? v + res[di] : v;
                }
                acc[n] = 0.0f;
            }
        }
        __syncwarp();                                                 // all lanes done with cslot before lane 0 refills it
        cslot = cslot + 1 == C::STAGES ? 0 : cslot + 1;
        if (++cks == nks) { cks = 0; cgi++; }
    }
}

template <int T, int NCOLS>
static cudaError_t launch2_one(const GemvArgs & a, cudaStream_t st) {
    using C = G2<T>;
    const int nblk = a.K >> 8;
    const size_t act_bytes = (size_t)NCOLS * nblk * (C::ACTB + C::BSB + 4);
    const size_t smem = 256 + act_bytes + 128 + (size_t)C::WARPS * C::STAGES * C::SLOT;
    if (smem > 227 * 1024) return cudaErrorInvalidValue;
    static int sm_count[64] = {};
    static size_t smem_set[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (sm_count[dev] == 0) {
        int n = 132;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sm_count[dev] = n;
    }
    if (smem_set[dev] < smem) {
        cudaError_t e = cudaFuncSetAttribute(gemv2_kernel<T, NCOLS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return e;
        smem_set[dev] = 227 * 1024;
    }
    const int per_sm = (int)((227 * 1024) / (smem + 1024));           // CTAs that fit one SM
    int gx = sm_count[dev] * (per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm));
    if (a.nz > 1) gx = (gx + a.nz - 1) / a.nz;
    const int ngroups = (a.M + 3) / 4;
    if (gx > ngroups) gx = ngroups;
    if (gx < 1) gx = 1;
    note_launch();
    gemv2_kernel<T, NCOLS><<<dim3((unsigned)gx, (unsigned)a.nz), C::WARPS * 32, smem, st>>>(a);
    return cudaGetLastError();
}

template <int T>
static cudaError_t launch2_type(const GemvArgs & a, cudaStream_t st) {
    switch (a.ncols) {
        case 1: return launch2_one<T, 1>(a, st);
        case 2: return launch2_one<T, 2>(a, st);
        case 3: return launch2_one<T, 3>(a, st);
        case 4: return launch2_one<T, 4>(a, st);
    }
    return cudaErrorNotSupported;
}

// Returns cudaErrorNotSupported when this generation does not cover the case (caller falls back to gemv.cu).
cudaError_t launch_gemv2(int type, const GemvArgs & a, cudaStream_t st) {
    if (a.M == 0 || a.nz == 0) return cudaSuccess;
    if (a.K <= 0 || a.K % 256 || a.ncols > 4) return cudaErrorNotSupported;
    const uintptr_t wa = reinterpret_cast<uintptr_t>(a.w);
    if (type == T_Q4_K || type == T_Q5_K) {
        if ((wa & 15) || (a.row_stride & 15) || (a.expert_stride & 15)) return cudaErrorNotSupported;
    } else if ((wa & 1) || (a.row_stride & 1) || (a.expert_stride & 1)) return cudaErrorNotSupported;
    // activations must fit next to the ring
    switch (type) {
        case T_Q4_K: return launch2_type<T_Q4_K>(a, st);
        case T_Q5_K: return launch2_type<T_Q5_K>(a, st);
        case T_Q6_K: return launch2_type<T_Q6_K>(a, st);
    }
    return cudaErrorNotSupported;
}

}  // namespace qmm
