// gemm_layout.cuh -- operand images of the prefill GEMM (gemm_tcgen05.cu), shared by the activation pre-pass, the
// weight de-quantiser and the host-side layout test (tests/host_gemm_layout.cpp).
//
// wgmma.mma_async (fp16) consumes K-major operands from shared memory in the canonical SWIZZLE_128B layout:
// an "atom" is ROWS x 64 fp16 (128 bytes per row); rows are stored in groups of 8 (1024 bytes); inside a group the
// 16-byte chunk index is XORed with the row index (Swizzle<3,4,3>).  One 256-weight K block = 4 atoms.
//
// The dot product does not care about the order of k inside a block, so both operands use the SAME permutation
// of k that makes nibble extraction cheap on the weight side (two nibbles that sit 16 bits apart in a 32-bit word of
// qs become one half2 without a byte shuffle):
//     Q4_K / Q5_K :  k' = k with bits 0 and 1 swapped
//     Q6_K        :  same (its words are unpacked two bytes apart as well)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define GL_HD __host__ __device__ __forceinline__
#else
#define GL_HD inline
#endif

namespace qmm {
namespace gl {

constexpr int ATOM_K     = 64;                 // fp16 elements per atom row (128 bytes)
constexpr int ATOMS_PER_BLOCK = 4;             // 256 / 64

GL_HD int kperm(int k) { return (k & ~3) | ((k & 1) << 1) | ((k >> 1) & 1); }          // swap bits 0 and 1

// byte offset of element (row, kk) inside an atom of `rows` rows; kk in [0, 64)
GL_HD int atom_off(int row, int kk) {
    const int chunk = kk >> 3, slot = kk & 7;
    return (row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4) + slot * 2;
}
GL_HD int atom_bytes(int rows) { return rows * 128; }

// Image of one (n-tile, k-block) of the activation operand, NT token rows:
//   4 main atoms (q_a as fp16 integers, permuted k)  |  1 "mins" atom: row n, kk 0..7 = even part of the 8 sub-block
//   sums bs32_j (bs32_j & ~1), kk 8..15 = their low bits (bs32_j & 1); the split keeps both exactly representable in
//   fp16 (|bs32| <= 4064: even integers are exact up to 4096).  The weight side pairs them with kk 0..7 = kk 8..15 =
//   the 6-bit mins m_j, so  sum_kk A'[m,kk] B'[n,kk] = sum_j m_j bs32_j  exactly.
GL_HD int64_t bimg_block_bytes(int nt) { return (int64_t)(ATOMS_PER_BLOCK + 1) * atom_bytes(nt); }

}  // namespace gl
}  // namespace qmm
