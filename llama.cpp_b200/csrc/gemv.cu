// gemv.cu -- decode mat-vec for GGUF block formats on sm_90a:  dst[M, n] = W[M, K] . act[K, n],  n <= 8.
//
// Replaces, for the batch-1 regime, the inner loop of ggml_compute_forward_mul_mat
// (ggml/src/ggml-cpu/ggml-cpu.c:1254-1452 -> ggml_vec_dot_q*_q8_* , ggml-cpu/quants.c:225-904); the closest analogue
// in the reference's CUDA backend is mul_mat_vec_q (ggml-cuda/mmvq.cu:544-765), which this does NOT port:
//
//   * HBM-bound by construction.  Algorithmic bytes per launch = M * K/BE * BB (every weight byte read once);
//     activations (K int8) stay in L1/L2.
//   * Each warp owns whole rows.  A row is cut into segments of 2048 weights (1152..2176 B, always a multiple of 16 B);
//     a segment is streamed HBM -> shared memory with 16-byte cp.async (L1-bypassing .cg) into a private per-warp
//     ring of D slots, so (D-1) segments per warp -- ~100 KB per SM with 32 resident warps -- are in flight while
//     the warp computes on the oldest one.  No block-level barrier exists anywhere in the kernel: a warp only ever
//     waits on its own cp.async groups (+ __syncwarp), so slow rows never stall neighbours.
//   * The ring lives in shared memory because three of the five formats (Q4_0 18 B, Q8_0 34 B, Q6_K 210 B blocks)
//     are only 2-byte aligned in HBM: the copy engine moves aligned 16-byte chunks, the unaligned reads happen
//     on-chip (ld*_a2 funnel shifts in qmm_formats.cuh).
//   * Per segment a lane handles 2 of the 64 "units" of 32 weights: integer dp4a against the CPU-identical
//     Q8_K/Q8_0 activations, one fp32 FMA per unit, warp-shuffle reduction at the end of the row.
//   * Rows are dealt round-robin over CTAs (row r -> CTA r % grid), grid = 4 CTAs x 132 SMs, so every SM streams
//     the same number of bytes +-1 row.
#include "qmm_formats.cuh"
#include "qmm_kernels.cuh"

namespace qmm {

constexpr int GEMV_WARPS   = 8;
constexpr int GEMV_THREADS = GEMV_WARPS * 32;

template <int T> struct GemvCfg {
    static constexpr int SEGB   = SEG_ELEMS / Fmt<T>::BE * Fmt<T>::BB;     // bytes per full segment
    static constexpr int SLOT   = (SEGB + 16 + 16 + 15) / 16 * 16;          // + align-down offset (<16) + read slack (16)
    static constexpr int STAGES = (SEGB > 1500) ? 3 : 4;
    static constexpr int SMEM   = GEMV_WARPS * STAGES * SLOT;
};

__device__ __forceinline__ void cp_async16(void * smem, const void * gmem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

template <int T, int NCOLS>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_q_kernel(const GemvArgs p) {
    using C = GemvCfg<T>;
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t * ring = smem + warp * (C::STAGES * C::SLOT);

    // ---- which weight matrix / activation column(s) this z-slice uses (MUL_MAT_ID routing, mmid semantics:
    //      dst[:, s, t] = as[:, :, ids[s, t]] . b[:, s % nb1, t], test-backend-ops.cpp:4713-4732)
    const int z = blockIdx.y;
    const uint8_t * wbase = p.w;
    int col0 = 0;
    if (p.ids != nullptr) {
        const int t = z / p.n_used, s = z - t * p.n_used;
        const int e = p.ids[(int64_t)t * p.ids_stride + s];
        if (e < 0 || e >= p.n_expert) return;             // invalid id: leave dst untouched (the CPU asserts)
        wbase += (int64_t)e * p.expert_stride;
        col0 = t * p.nb1 + (s % p.nb1);
    }
    ActCol act[NCOLS];
#pragma unroll
    for (int n = 0; n < NCOLS; n++) {
        act[n].qs = p.act.qs + (int64_t)(col0 + n) * p.act.qs_stride;
        act[n].d = p.act.d + (int64_t)(col0 + n) * p.act.d_stride;
        act[n].bsums = p.act.bsums + (int64_t)(col0 + n) * p.act.bs_stride;
    }
    float * dst = p.dst + (int64_t)z * NCOLS * p.ldd;
    const float * res = p.residual ? p.residual + (int64_t)z * NCOLS * p.ldd : nullptr;

    const int K = p.K, M = p.M;
    const int row_bytes = K / Fmt<T>::BE * Fmt<T>::BB;
    const int spr = (K + SEG_ELEMS - 1) / SEG_ELEMS;                       // segments per row
    // rows of this CTA: blockIdx.x + i*gridDim.x ; this warp takes i = warp, warp + 8, ...
    const int nrb = (int)blockIdx.x < M ? (M - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int nrw = warp < nrb ? (nrb - 1 - warp) / GEMV_WARPS + 1 : 0;
    const int total = nrw * spr;                                          // segments this warp streams
    if (total == 0) return;

    // issue one segment: row index ri (warp-local), segment s -> slot
    auto issue = [&](int ri, int s, int slot) {
        const int row = (int)blockIdx.x + (warp + GEMV_WARPS * ri) * (int)gridDim.x;
        const uint8_t * g = wbase + (int64_t)row * p.row_stride + (int64_t)s * C::SEGB;
        const int nbytes = min(C::SEGB, row_bytes - s * C::SEGB);
        const int off = (int)(reinterpret_cast<uintptr_t>(g) & 15);
        const uint8_t * g0 = g - off;
        const int nchunks = (off + nbytes + 15) >> 4;
        uint8_t * sl = ring + slot * C::SLOT;
        for (int c = lane; c < nchunks; c += 32) cp_async16(sl + 16 * c, g0 + 16 * c);
    };

    int iri = 0, is = 0;                 // next segment to issue (row, seg)
    int islot = 0;
#pragma unroll
    for (int k = 0; k < C::STAGES - 1; k++) {
        if (iri < nrw) { issue(iri, is, islot); if (++is == spr) { is = 0; iri++; } }
        cp_async_commit();
        islot = islot + 1 == C::STAGES ? 0 : islot + 1;
    }

    float acc[NCOLS];
#pragma unroll
    for (int n = 0; n < NCOLS; n++) acc[n] = 0.0f;

    int cslot = 0, cs = 0, cri = 0;      // segment being consumed
    for (int i = 0; i < total; i++) {
        if (iri < nrw) { issue(iri, is, islot); if (++is == spr) { is = 0; iri++; } }
        cp_async_commit();
        islot = islot + 1 == C::STAGES ? 0 : islot + 1;

        cp_async_wait<C::STAGES - 1>();
        __syncwarp();

        {
            const int row = (int)blockIdx.x + (warp + GEMV_WARPS * cri) * (int)gridDim.x;
            const uint8_t * g = wbase + (int64_t)row * p.row_stride + (int64_t)cs * C::SEGB;
            const uint8_t * seg = ring + cslot * C::SLOT + (int)(reinterpret_cast<uintptr_t>(g) & 15);
            const int kseg = cs * SEG_ELEMS;
#pragma unroll
            for (int uu = 0; uu < 2; uu++) {
                const int u = lane + 32 * uu;
                if (kseg + 32 * u < K) {
#pragma unroll
                    for (int n = 0; n < NCOLS; n++) acc[n] += unit_dot<T>(seg, u, kseg, act[n]);
                }
            }
            if (cs + 1 == spr) {         // row finished: reduce over lanes, write
#pragma unroll
                for (int n = 0; n < NCOLS; n++) {
                    float v = acc[n];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    if (lane == 0) {
                        const int64_t di = (int64_t)n * p.ldd + row;
                        dst[di] = res ? v + res[di] : v;
                    }
                    acc[n] = 0.0f;
                }
            }
        }
        __syncwarp();                    // every lane is done with cslot before it is refilled next iteration
        cslot = cslot + 1 == C::STAGES ? 0 : cslot + 1;
        if (++cs == spr) { cs = 0; cri++; }
    }
    cp_async_wait<0>();
}

template <int T, int NCOLS>
static cudaError_t launch_one(const GemvArgs & a, cudaStream_t st) {
    using C = GemvCfg<T>;
    static bool attr_done[64] = {};                      // per device: one host process may drive all 8 GPUs
    static int  sm_count[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (!attr_done[dev & 63]) {
        cudaError_t e = cudaFuncSetAttribute(gemv_q_kernel<T, NCOLS>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM);
        if (e != cudaSuccess) return e;
        int n = 132;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sm_count[dev & 63] = n;
        attr_done[dev & 63] = true;
    }
    const int sms = sm_count[dev & 63];
    int gx = sms * 4;
    if (a.nz > 1) gx = (gx + a.nz - 1) / a.nz;          // keep the whole launch near 4 CTAs/SM
    if (gx > a.M) gx = a.M;
    if (gx < 1) gx = 1;
    note_launch();
    gemv_q_kernel<T, NCOLS><<<dim3((unsigned)gx, (unsigned)a.nz), GEMV_THREADS, C::SMEM, st>>>(a);
    return cudaGetLastError();
}

template <int T>
static cudaError_t launch_type(const GemvArgs & a, cudaStream_t st) {
    switch (a.ncols) {
        case 1: return launch_one<T, 1>(a, st);
        case 2: return launch_one<T, 2>(a, st);
        case 3: return launch_one<T, 3>(a, st);
        case 4: return launch_one<T, 4>(a, st);
        case 5: return launch_one<T, 5>(a, st);
        case 6: return launch_one<T, 6>(a, st);
        case 7: return launch_one<T, 7>(a, st);
        case 8: return launch_one<T, 8>(a, st);
    }
    return cudaErrorInvalidValue;
}

static int g_gemv_variant = 2;          // 2 = gemv2.cu where it applies (default), 1 = always this file
void set_gemv_variant(int v) { g_gemv_variant = v; }
cudaError_t launch_gemv2(int type, const GemvArgs & a, cudaStream_t st);

cudaError_t launch_gemv(int type, const GemvArgs & a, cudaStream_t st) {
    if (a.M == 0 || a.nz == 0) return cudaSuccess;
    if (g_gemv_variant == 2) {
        const cudaError_t e = launch_gemv2(type, a, st);
        if (e != cudaErrorNotSupported) return e;
    }
    if (a.K <= 0 || a.K % block_elems(type)) return cudaErrorInvalidValue;
    // 16-byte formats need 16-byte aligned rows (true for every ggml tensor: base alignment >= 32, row bytes % 16 == 0);
    // the 2-byte formats only need even addresses.
    const uintptr_t wa = reinterpret_cast<uintptr_t>(a.w);
    if (type == T_Q4_K || type == T_Q5_K) {
        if ((wa & 15) || (a.row_stride & 15) || (a.expert_stride & 15)) return cudaErrorMisalignedAddress;
    } else if ((wa & 1) || (a.row_stride & 1) || (a.expert_stride & 1)) return cudaErrorMisalignedAddress;
    switch (type) {
        case T_Q4_0: return launch_type<T_Q4_0>(a, st);
        case T_Q8_0: return launch_type<T_Q8_0>(a, st);
        case T_Q4_K: return launch_type<T_Q4_K>(a, st);
        case T_Q5_K: return launch_type<T_Q5_K>(a, st);
        case T_Q6_K: return launch_type<T_Q6_K>(a, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace qmm
