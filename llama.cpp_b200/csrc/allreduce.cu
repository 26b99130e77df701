// allreduce.cu -- one-shot NVLink all-reduce for the tensor-parallel decode path (messages of tens of KB).
//
// Every GPU owns a symmetric buffer, peer-mapped by all others (cudaDeviceEnablePeerAccess; on an HGX H100 every pair
// is one NVSwitch hop).  For call number `seq` (kept in device memory, so the launch is CUDA-graph capturable):
//   1. rank r copies its vector into slot r of EVERY rank's buffer set (seq & 1)   -- peer stores over NVLink
//   2. __threadfence_system(), then rank r writes seq into flag[r] of every rank    -- release
//   3. rank r spins until all n flags in its own memory equal seq                    -- acquire
//   4. rank r sums the n slots of its own buffer in rank order into its tensor       -- same order everywhere =>
//                                                                                       bit-identical on all ranks
// Two buffer sets alternate by seq parity: a rank can only be one call ahead of the slowest rank (it needs that
// rank's flag to finish), so the set it overwrites is never still being read.  Bytes over NVLink per rank: n * bytes
// out, n * bytes in; latency = one peer store + one flag round trip (~2-3 us), vs tens of us for a host-driven NCCL
// call at this size.  Roofline: NVLink latency, not bandwidth.
#include "qmm_kernels.cuh"

namespace qmm {

__global__ void __launch_bounds__(1024) oneshot_allreduce_kernel(OneShotDev self, OneShotPeers peers, float * data, int count) {
    __shared__ unsigned seq_s;
    if (threadIdx.x == 0) seq_s = *self.seq + 1;
    __syncthreads();
    const unsigned seq = seq_s;
    const int n = self.n, r = self.rank;
    const size_t set_off = (size_t)(seq & 1) * self.set_floats;
    // 1. push (vectorised when aligned)
    const int nthreads = blockDim.x * gridDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
    if ((count & 3) == 0 && (reinterpret_cast<uintptr_t>(data) & 15) == 0) {
        const float4 * src = reinterpret_cast<const float4 *>(data);
        for (int i = tid; i < count / 4; i += nthreads) {
            const float4 v = src[i];
#pragma unroll 1
            for (int p = 0; p < n; p++) reinterpret_cast<float4 *>(peers.buf[p] + set_off + (size_t)r * self.slot_floats)[i] = v;
        }
    } else {
        for (int i = tid; i < count; i += nthreads) {
            const float v = data[i];
            for (int p = 0; p < n; p++) (peers.buf[p] + set_off + (size_t)r * self.slot_floats)[i] = v;
        }
    }
    // 2. release: all blocks of this rank must have pushed before the flag goes up -> per-rank block counter
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned done = atomicAdd(self.block_counter, 1u) + 1;
        if (done == gridDim.x * seq) {                         // last block of this call
            __threadfence_system();
            for (int p = 0; p < n; p++) *reinterpret_cast<volatile unsigned *>(peers.flags[p] + r) = seq;
        }
    }
    // 3. acquire
    if (threadIdx.x < n) {
        volatile unsigned * f = reinterpret_cast<volatile unsigned *>(self.flags + threadIdx.x);
        long long spins = 0;
        while (*f < seq) { if (++spins > (1ll << 31)) __trap(); }
    }
    __syncthreads();
    __threadfence_system();
    // 4. reduce in rank order
    const float * base = self.buf + set_off;
    for (int i = tid; i < count; i += nthreads) {
        float s = 0.0f;
        for (int p = 0; p < n; p++) s += __ldcv(base + (size_t)p * self.slot_floats + i);
        data[i] = s;
    }
    // bump the call counter once per call (last block to get here)
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned fin = atomicAdd(self.finish_counter, 1u) + 1;
        if (fin == gridDim.x * seq) *self.seq = seq;
    }
}

cudaError_t oneshot_init(OneShotComm & c, const int * devs, int n, size_t max_bytes) {
    if (n < 2 || n > ONESHOT_MAX_DEV) return cudaErrorInvalidValue;
    c.n = n;
    c.slot_floats = (max_bytes / 4 + 63) / 64 * 64;
    c.set_floats = c.slot_floats * n;
    for (int i = 0; i < n; i++) {
        c.devs[i] = devs[i];
        for (int j = 0; j < n; j++) {
            if (i == j) continue;
            int can = 0;
            cudaError_t e = cudaDeviceCanAccessPeer(&can, devs[i], devs[j]);
            if (e != cudaSuccess || !can) return cudaErrorPeerAccessUnsupported;
        }
    }
    for (int i = 0; i < n; i++) {
        cudaError_t e = cudaSetDevice(devs[i]);
        if (e != cudaSuccess) return e;
        for (int j = 0; j < n; j++) {
            if (i == j) continue;
            e = cudaDeviceEnablePeerAccess(devs[j], 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
            if (e != cudaSuccess) return e;
        }
        e = cudaMalloc(&c.buf[i], 2 * c.set_floats * sizeof(float));
        if (e != cudaSuccess) return e;
        e = cudaMalloc(&c.ctl[i], 256);
        if (e != cudaSuccess) return e;
        e = cudaMemset(c.ctl[i], 0, 256);
        if (e != cudaSuccess) return e;
    }
    for (int i = 0; i < n; i++) { cudaSetDevice(devs[i]); cudaDeviceSynchronize(); }
    return cudaSuccess;
}

void oneshot_free(OneShotComm & c) {
    for (int i = 0; i < c.n; i++) {
        cudaSetDevice(c.devs[i]);
        cudaDeviceSynchronize();
        if (c.buf[i]) cudaFree(c.buf[i]);
        if (c.ctl[i]) cudaFree(c.ctl[i]);
        c.buf[i] = nullptr; c.ctl[i] = nullptr;
    }
}

cudaError_t oneshot_allreduce(OneShotComm & c, float * const * data, size_t count, const cudaStream_t * streams) {
    if (count > c.slot_floats) return cudaErrorInvalidValue;
    OneShotPeers peers{};
    for (int p = 0; p < c.n; p++) { peers.buf[p] = c.buf[p]; peers.flags[p] = c.ctl[p]; }
    // small fixed grid: the message is tiny, latency is what matters; every launch of a communicator uses the same grid
    const int blocks = 4, threads = 512;
    for (int r = 0; r < c.n; r++) {
        cudaError_t e = cudaSetDevice(c.devs[r]);
        if (e != cudaSuccess) return e;
        OneShotDev self{};
        self.n = c.n; self.rank = r; self.slot_floats = c.slot_floats; self.set_floats = c.set_floats;
        self.buf = c.buf[r]; self.flags = c.ctl[r];
        self.seq = c.ctl[r] + 32; self.block_counter = c.ctl[r] + 33; self.finish_counter = c.ctl[r] + 34;
        note_launch();
        oneshot_allreduce_kernel<<<blocks, threads, 0, streams[r]>>>(self, peers, data[r], (int)count);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace qmm
