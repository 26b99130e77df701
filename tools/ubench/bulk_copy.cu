// Micro-benchmark (sm_90a; nvcc -O3 -gencode arch=compute_90a,code=sm_90a): HBM -> shared memory throughput of cp.async.bulk as a function of who issues the copies.
// One CTA per SM; W warps x L lanes are "issuers"; every issuer streams its own disjoint part of a large buffer through its own
// ring of D slots of S bytes (one mbarrier per slot; the data is not consumed -- a slot is re-armed as soon as its copy has landed).
// Prints achieved TB/s over the whole chip.  Question it answers: does a decode kernel need MANY issuing lanes / warps, or deep rings,
// or large copies, to keep every SM's share of HBM busy?
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t s32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t * b, int c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t * b, uint32_t n) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(s32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t * b, uint32_t par) {
    uint32_t ok = 0;
    while (!ok) asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.b32 %0, 1, 0, P1;\n\t}\n" : "=r"(ok) : "r"(s32(b)), "r"(par) : "memory");
}
__device__ __forceinline__ void bulk(void * dst, const void * src, uint32_t n, uint64_t * b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(s32(dst)), "l"(src), "r"(n), "r"(s32(b)) : "memory");
}

__global__ void __launch_bounds__(1024, 1) stream_kernel(const uint8_t * __restrict__ src, size_t bytes_per_issuer, int L, int D, int S) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, W = blockDim.x >> 5;
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem);                   // [W][L][D]
    uint8_t * ring = smem + 8 * 32 * 8 * 16;                                 // up to 32 warps x 8 lanes x 16 slots of barriers
    const bool issuer = lane < L;
    const int id = warp * L + lane;                                          // issuer id inside the CTA
    uint64_t * mybar = bars + (size_t)id * 16;
    uint8_t * myring = ring + (size_t)id * D * S;
    if (issuer) for (int i = 0; i < D; i++) mbar_init(mybar + i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    __syncthreads();
    if (!issuer) return;
    const uint8_t * p = src + ((size_t)blockIdx.x * W * L + id) * bytes_per_issuer;
    const int n = (int)(bytes_per_issuer / S);
    for (int i = 0; i < n; i++) {
        const int slot = i % D, use = i / D;
        if (use > 0) mbar_wait(mybar + slot, (use - 1) & 1);
        mbar_expect_tx(mybar + slot, (uint32_t)S);
        bulk(myring + (size_t)slot * S, p + (size_t)i * S, (uint32_t)S, mybar + slot);
    }
    for (int i = n > D ? n - D : 0; i < n; i++) mbar_wait(mybar + i % D, (i / D) & 1);
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const size_t total = 3ull << 30;
    uint8_t * buf;
    cudaMalloc(&buf, total);
    cudaMemset(buf, 1, total);
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    printf("SMs %d; buffer %.1f GiB; columns: warps lanes depth size | in flight per SM | TB/s\n", sms, total / 1073741824.0);
    const int sizes[] = {1024, 2304, 4608, 9216, 18432};
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int W : {1, 2, 4, 8, 16})
        for (int L : {1, 2, 4, 8})
            for (int S : sizes)
                for (int D : {2, 4, 8, 16}) {
                    const size_t ring = (size_t)W * L * D * S;
                    if (ring > 192 * 1024 || W * L > 64) continue;
                    const size_t smem = 8 * 32 * 8 * 16 + ring;
                    const size_t issuers = (size_t)sms * W * L;
                    size_t per = total / issuers / S * S;
                    if (per > (64u << 20)) per = (64u << 20) / S * S;            // enough to be far larger than the L2 in total
                    if (per * issuers < (1ull << 30)) { /* small but fine */ }
                    stream_kernel<<<sms, W * 32, smem>>>(buf, per, L, D, S);     // warm-up / fault-in
                    cudaEventRecord(e0);
                    stream_kernel<<<sms, W * 32, smem>>>(buf, per, L, D, S);
                    cudaEventRecord(e1);
                    cudaEventSynchronize(e1);
                    float ms = 0;
                    cudaEventElapsedTime(&ms, e0, e1);
                    if (cudaGetLastError() != cudaSuccess) { printf("%2d %d %2d %5d | error\n", W, L, D, S); continue; }
                    printf("%2d %d %2d %5d | %6.1f KB | %6.3f\n", W, L, D, S, ring / 1024.0, per * issuers / (ms * 1e-3) / 1e12);
                }
    return 0;
}
