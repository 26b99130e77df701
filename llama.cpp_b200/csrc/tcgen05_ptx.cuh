// tcgen05_ptx.cuh (a historical name) -- the PTX wrappers shared by the prefill GEMM kernels (gemm_tcgen05.cu: K-quants, exact-integer operands;
// gemm_legacy_wgmma.cu: Q4_0 / Q8_0, hi/lo fp16 operands): mbarriers, 1-D bulk copies (TMA), the sm_90a warpgroup MMA
// (wgmma.mma_async m64n128k16, fp16 in, fp32 accumulators in registers) and its fences, and the shared-memory descriptor of the
// canonical K-major SWIZZLE_128B layout.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace qmm {

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t s32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void g_mbar_init(uint64_t * bar, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(s32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void g_mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(s32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void g_mbar_wait(uint64_t * bar, uint32_t parity) {
    uint32_t ok = 0;
    long long spins = 0;
    while (!ok) {
        asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.b32 %0, 1, 0, P1;\n\t}\n"
                     : "=r"(ok) : "r"(s32(bar)), "r"(parity) : "memory");
        if (!ok && ++spins > (1ll << 22)) __trap();
    }
}
__device__ __forceinline__ void g_mbar_arrive(uint64_t * bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(s32(bar)) : "memory"); }
__device__ __forceinline__ void g_bulk_g2s(void * dst, const void * src, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 ::"r"(s32(dst)), "l"(src), "r"(bytes), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
// barrier among the 128 threads of one warpgroup (ids 1.. are free: __syncthreads uses 0)
__device__ __forceinline__ void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;\n" ::"r"(1 + wg) : "memory"); }

// ------------------------------------------------------------------------------------------------ warpgroup MMA
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// Pins the accumulator registers at this point of the program: the compiler may not move their reads above a wgmma_wait or
// their writes below the wgmma that follows.
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, both K-major in shared memory, fp16 in, fp32 accumulate.  Thread t of the warpgroup
// holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) and columns 8 i + 2 (t % 4) (+ 1): d[4 i + 2 hi + c] = D[row + 8 hi][8 i + 2 (t % 4) + c].
__device__ __forceinline__ void wgmma_m64n128k16_f16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, "
        "%29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, "
        "%56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
          "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate)
        : "memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor of sm_90 (cute::GMMA::DescriptorSM90): start address >> 4 in bits [0,14),
// LBO (unused for swizzled K-major) = 1 in [16,30), SBO = 1024 B (8 rows x 128 B) >> 4 in [32,46), base offset 0 (atoms are
// 1024-byte aligned), layout type SWIZZLE_128B = 1 in [62,64).  A k16 slice inside the 128-byte row is selected by adding its byte
// offset (32 per slice) to the start address.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

}  // namespace qmm
