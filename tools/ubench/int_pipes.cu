// Micro-benchmark (sm_90a; nvcc -O3 -gencode arch=compute_90a,code=sm_90a): issue rate of the integer dot-product paths a quantised GEMV can use.
//   dp4a            IDP.4A on the CUDA cores (what round 1's decode kernels were built on)
//   imad            IMAD (full-rate integer pipe), for scale
//   mma.s8 k32      mma.sync.m16n8k32 s8 x s8 -> s32 (legacy tensor-core path)
//   mma.f16 k16     mma.sync.m16n8k16 f16 x f16 -> f32
//   ffma            scalar fp32 FMA (the prefill GEMMs' per-block rescale)
// Every warp runs `iters` x 16 independent chains; prints warp-instructions per cycle per SM for 1, 2, 4, 8 warps per SMSP.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

template <int MODE>
__global__ void bench(int iters, unsigned long long * cycles, int * sink) {
    int acc[16];
    float facc[16];
#pragma unroll
    for (int i = 0; i < 16; i++) { acc[i] = threadIdx.x + i; facc[i] = (float)i; }
    unsigned a = threadIdx.x * 0x01010101u + 7u, b = blockIdx.x * 0x01030507u + 3u;
    __syncthreads();
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (MODE == 0) acc[i] = __dp4a((int)(a + i), (int)b, acc[i]);
            if (MODE == 1) acc[i] = acc[i] * (int)(a | 1) + (int)b;
            if (MODE == 2) {
                int c0 = acc[i], c1 = 0, c2 = 0, c3 = 0;
                asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(c3) : "r"(a), "r"(a + 1), "r"(a + 2), "r"(a + 3), "r"(b), "r"(b + 1));
                acc[i] = c0 + c1 + c2 + c3;
            }
            if (MODE == 5) facc[i] = fmaf(facc[i], 1.0001f, 0.5f);
            if (MODE == 3) {
                float c0 = facc[i], c1 = 0.f, c2 = 0.f, c3 = 0.f;
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                             : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3) : "r"(a), "r"(a + 1), "r"(a + 2), "r"(a + 3), "r"(b), "r"(b + 1));
                facc[i] = c0 + c1 + c2 + c3;
            }
        }
        a += 0x00010001u;
    }
    const long long t1 = clock64();
    int s = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) s += acc[i] + (int)facc[i];
    if (s == 0x7fffffff) sink[0] = s;
    if (threadIdx.x == 0) cycles[blockIdx.x] = (unsigned long long)(t1 - t0);
}

template <int MODE>
static void run(const char * name, int sms) {
    unsigned long long * cyc;
    int * sink;
    cudaMalloc(&cyc, 1024 * 8);
    cudaMalloc(&sink, 4);
    const int iters = 2000;
    for (int warps = 4; warps <= 32; warps *= 2) {
        bench<MODE><<<sms, warps * 32>>>(iters, cyc, sink);
        bench<MODE><<<sms, warps * 32>>>(iters, cyc, sink);
        cudaDeviceSynchronize();
        unsigned long long h[1024];
        cudaMemcpy(h, cyc, sms * 8, cudaMemcpyDeviceToHost);
        double avg = 0;
        for (int i = 0; i < sms; i++) avg += (double)h[i];
        avg /= sms;
        const double winstr = (double)iters * 16 * warps;
        printf("%-12s %2d warps/SM: %8.0f cycles, %6.3f warp-instr/cycle/SM (%6.1f lanes/cycle/SM)%s\n", name, warps, avg, winstr / avg, 32.0 * winstr / avg,
               cudaGetLastError() == cudaSuccess ? "" : "  [CUDA error]");
    }
    cudaFree(cyc);
    cudaFree(sink);
}

int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    printf("SMs: %d\n", sms);
    run<0>("dp4a", sms);
    run<1>("imad", sms);
    run<2>("mma.s8.k32", sms);
    run<3>("mma.f16.k16", sms);
    run<5>("ffma", sms);
    return 0;
}
