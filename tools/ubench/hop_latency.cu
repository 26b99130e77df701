// hop_latency.cu (sm_90a; nvcc -O3 -gencode arch=compute_90a,code=sm_90a) -- how long does a tagged-slot vector take from one CTA's stores to every other CTA having read it, while every
// SM streams weights with cp.async.bulk?  (The persistent decode kernel pays this once per phase: 160 times per token.)
//
//   hop_latency <cap> <poll_mode> <rounds> [n_slots]
//     cap        pieces (9728 B) each SM keeps in flight (0 = no streaming)
//     poll_mode  0: every thread loads its slots once and re-polls stale ones one after the other (the kernel's prologue)
//                1: one thread per CTA polls the LAST slot; when it is valid the CTA loads everything once (lower bound on traffic;
//                   not a valid protocol -- stores of one writer are unordered -- but the writer here stores that slot last + fence)
//                2: like 0, but the stale slots are re-loaded as a batch
// Prints the mean / min / max latency (writer's timestamp before its first store -> reader's timestamp after its last valid load)
// and the streaming bandwidth reached meanwhile.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

constexpr int THREADS = 256, CTHREADS = 224, PIECE = 9728, MAXCAP = 20;

__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void ld2(const uint64_t * p, uint64_t & a, uint64_t & b) { asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory"); }
__device__ __forceinline__ uint64_t ld1(const uint64_t * p) { uint64_t v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st1(uint64_t * p, uint64_t v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory"); }

__global__ void __launch_bounds__(THREADS) hop_kernel(const uint8_t * __restrict__ weights, size_t wbytes, uint64_t * slots, int n_slots, int cap, int poll_mode, int rounds,
                                                      unsigned long long * t_w, unsigned long long * t_r, unsigned long long * copied, volatile int * stop) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem);
    uint8_t * ring = smem + 256;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, cta = blockIdx.x, grid = gridDim.x;
    const unsigned long long deadline = gtime() + 8000000000ull;      // a lost round must fail the launch, not hang the GPU
    unsigned spin = 0;
#define WATCHDOG() do { if (((++spin) & 0x3fffu) == 0 && gtime() > deadline) __trap(); } while (0)
    if (tid == 0) for (int i = 0; i < MAXCAP; i++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bars + i)));
    __syncthreads();
    if (warp == 7) {                                                  // streaming warp
        if (cap == 0) return;
        unsigned long long g = 0;
        const size_t per_cta = (wbytes / grid) / PIECE * PIECE;
        const uint8_t * base = weights + (size_t)cta * per_cta;
        size_t off = 0;
        while (true) {
            if ((g & 31) == 0 && (*stop != 0 || gtime() > deadline)) break;
            const int s = (int)(g % cap);
            if (g >= (unsigned long long)cap) {
                const uint32_t par = (uint32_t)((g / cap - 1) & 1);
                uint32_t ok = 0;
                while (!ok) asm volatile("{ .reg .pred P; mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2; selp.b32 %0, 1, 0, P; }" : "=r"(ok) : "r"(smem_u32(bars + s)), "r"(par) : "memory");
            }
            if (lane == 0) {
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bars + s)), "r"(PIECE) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(ring + (size_t)s * PIECE)), "l"(base + off), "r"(PIECE), "r"(smem_u32(bars + s)) : "memory");
            }
            __syncwarp();
            off += PIECE; if (off + PIECE > per_cta) off = 0;
            g++;
        }
        // drain
        for (unsigned long long q = (g > (unsigned long long)cap ? g - cap : 0); q < g; q++) {
            const int s = (int)(q % cap); const uint32_t par = (uint32_t)((q / cap) & 1);
            uint32_t ok = 0;
            while (!ok) asm volatile("{ .reg .pred P; mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2; selp.b32 %0, 1, 0, P; }" : "=r"(ok) : "r"(smem_u32(bars + s)), "r"(par) : "memory");
        }
        if (lane == 0) copied[cta] = g * PIECE;
        return;
    }
    // ---- hop rounds: CTA (r % grid) writes vector r (tag r + 1) into array r % 4; everyone else reads it
    const int per_thread = (n_slots + CTHREADS - 1) / CTHREADS;       // slots per thread, in pairs
    for (int r = 0; r < rounds; r++) {
        uint64_t * arr = slots + (size_t)(r & 15) * n_slots;
        const uint64_t tag = (uint64_t)(r + 1) << 32;
        if (cta == r % grid) {
            const unsigned long long t0 = gtime();
            while (gtime() - t0 < 6000) { }                           // the readers are already polling when the data is written
            asm volatile("bar.sync 1, %0;" ::"n"(CTHREADS));
            if (tid == 0) t_w[r] = gtime();
            for (int i = tid; i < n_slots - 1; i += CTHREADS) st1(arr + i, tag | (uint32_t)i);
            asm volatile("bar.sync 1, %0;" ::"n"(CTHREADS));
            if (tid == 0) { __threadfence(); st1(arr + n_slots - 1, tag | (uint32_t)(n_slots - 1)); }
            continue;
        }
        if (poll_mode == 1) {
            if (tid == 0) { while ((ld1(arr + n_slots - 1) >> 32) != (uint64_t)(r + 1)) { WATCHDOG(); } }
            asm volatile("bar.sync 1, %0;" ::"n"(CTHREADS));
            uint64_t acc = 0;
            for (int i = 2 * tid; i < n_slots; i += 2 * CTHREADS) { uint64_t a, b; ld2(arr + i, a, b); acc += a + b; }
            if (acc == 12345) t_r[0] = acc;
        } else {
            // thread t owns pairs t, t + CTHREADS, ... (coalesced 16-byte loads across the warp)
            constexpr int MAXP = 32;
            uint64_t a[MAXP], b[MAXP];
            const int npairs = n_slots / 2;
#pragma unroll
            for (int u = 0; u < MAXP; u++) { const int p = tid + u * CTHREADS; if (p < npairs) ld2(arr + 2 * p, a[u], b[u]); }
            if (poll_mode == 0) {
#pragma unroll
                for (int u = 0; u < MAXP; u++) {
                    const int p = tid + u * CTHREADS;
                    if (p < npairs) while ((a[u] >> 32) != (uint64_t)(r + 1) || (b[u] >> 32) != (uint64_t)(r + 1)) { WATCHDOG(); ld2(arr + 2 * p, a[u], b[u]); }
                }
            } else {
                for (;;) {
                    const uint64_t * first = nullptr;
#pragma unroll
                    for (int u = 0; u < MAXP; u++) { const int p = tid + u * CTHREADS; if (p < npairs && first == nullptr && ((a[u] >> 32) != (uint64_t)(r + 1) || (b[u] >> 32) != (uint64_t)(r + 1))) first = arr + 2 * p; }
                    if (first == nullptr) break;
                    uint64_t x, y; ld2(first, x, y);
                    while ((x >> 32) != (uint64_t)(r + 1) || (y >> 32) != (uint64_t)(r + 1)) { WATCHDOG(); ld2(first, x, y); }
#pragma unroll
                    for (int u = 0; u < MAXP; u++) { const int p = tid + u * CTHREADS; if (p < npairs && ((a[u] >> 32) != (uint64_t)(r + 1) || (b[u] >> 32) != (uint64_t)(r + 1))) ld2(arr + 2 * p, a[u], b[u]); }
                }
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(CTHREADS));
        if (tid == 0) t_r[(size_t)r * grid + cta] = gtime();
    }
    (void)per_thread;
}

__global__ void set_stop(int * stop) { *stop = 1; }

int main(int argc, char ** argv) {
    const int cap = argc > 1 ? atoi(argv[1]) : 0, mode = argc > 2 ? atoi(argv[2]) : 0, rounds = argc > 3 ? atoi(argv[3]) : 600, n_slots = argc > 4 ? atoi(argv[4]) : 4096;
    if (cap > MAXCAP || n_slots > 2 * 32 * CTHREADS) { fprintf(stderr, "cap <= %d, n_slots <= %d\n", MAXCAP, 2 * 32 * CTHREADS); return 2; }
    int grid = 132;
    cudaDeviceGetAttribute(&grid, cudaDevAttrMultiProcessorCount, 0);
    const size_t wbytes = (size_t)4 << 30;
    uint8_t * w; uint64_t * slots; unsigned long long * t_w, * t_r, * copied; int * stop;
    cudaMalloc(&w, wbytes); cudaMemset(w, 1, wbytes);
    cudaMalloc(&slots, sizeof(uint64_t) * 16 * n_slots); cudaMemset(slots, 0, sizeof(uint64_t) * 16 * n_slots);
    cudaMalloc(&t_w, 8 * rounds); cudaMalloc(&t_r, 8 * (size_t)rounds * grid); cudaMalloc(&copied, 8 * grid);
    cudaMemset(t_r, 0, 8 * (size_t)rounds * grid); cudaMemset(copied, 0, 8 * grid);
    cudaMallocManaged(&stop, 4); *stop = 0;
    cudaMemAdvise(stop, 4, cudaMemAdviseSetPreferredLocation, 0);
    const size_t smem = 256 + (size_t)(cap > 0 ? cap : 1) * PIECE;
    cudaFuncSetAttribute(hop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaStream_t s1, s2; cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking); cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    // the streaming warps run until the hop rounds are over: a second tiny kernel cannot run (all SMs full?) -- it can: 1 CTA/SM of 256 threads leaves room
    int * hstop, * dstop; cudaHostAlloc(&hstop, 4, cudaHostAllocMapped); *hstop = 0; cudaHostGetDevicePointer(&dstop, hstop, 0);   // the host stops the streamers directly
    cudaEventRecord(e0, s1);
    hop_kernel<<<grid, THREADS, smem, s1>>>(w, wbytes, slots, n_slots, cap, mode, rounds, t_w, t_r, copied, dstop);
    // wait until the last round's readers are done, then stop the streamers
    std::vector<unsigned long long> last(grid);
    for (;;) {
        cudaMemcpyAsync(last.data(), t_r + (size_t)(rounds - 1) * grid, 8 * grid, cudaMemcpyDeviceToHost, s2);
        cudaStreamSynchronize(s2);
        int done = 0;
        for (int i = 0; i < grid; i++) done += last[i] != 0;
        if (done >= grid - 1) break;
        if (cudaStreamQuery(s1) != cudaErrorNotReady) break;
    }
    *(volatile int *)hstop = 1;
    cudaEventRecord(e1, s1);
    cudaError_t e = cudaStreamSynchronize(s1);
    if (e != cudaSuccess) { fprintf(stderr, "kernel failed: %s\n", cudaGetErrorString(e)); return 1; }
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    std::vector<unsigned long long> tw(rounds), tr((size_t)rounds * grid), cp(grid);
    cudaMemcpy(tw.data(), t_w, 8 * rounds, cudaMemcpyDeviceToHost);
    cudaMemcpy(tr.data(), t_r, 8 * (size_t)rounds * grid, cudaMemcpyDeviceToHost);
    cudaMemcpy(cp.data(), copied, 8 * grid, cudaMemcpyDeviceToHost);
    double sum = 0, sum_max = 0; long n = 0; double mn = 1e30, mx = 0;
    for (int r = 20; r < rounds; r++) {
        double rmax = 0;
        for (int c = 0; c < grid; c++) {
            if (c == r % grid) continue;
            const double d = (double)tr[(size_t)r * grid + c] - (double)tw[r];
            sum += d; n++; if (d < mn) mn = d; if (d > mx) mx = d; if (d > rmax) rmax = d;
        }
        sum_max += rmax;
    }
    unsigned long long tot = 0; for (int c = 0; c < grid; c++) tot += cp[c];
    printf("cap %2d (%6.1f KB/SM in flight)  poll_mode %d  slots %5d: latency mean %.2f us, mean of per-round max %.2f us, min %.2f, max %.2f;  stream %.0f GB/s over %.1f ms\n",
           cap, cap * PIECE / 1024.0, mode, n_slots, sum / n / 1e3, sum_max / (rounds - 20) / 1e3, mn / 1e3, mx / 1e3, tot / (ms * 1e6), ms);
    return 0;
}
