// qmm_attn.cuh -- launchers of the attention kernels that only the C ABI's test entry points call (include/b200_attn.h).
// The backend reaches the same kernels through ops::flash_attn (qmm_ops.cuh); this header is kept apart from the ones the
// plugin's C++ objects compile against.
#pragma once
#include "qmm_ops.cuh"

namespace qmm {
namespace ops {

// The scalar kernel alone (any row count; D a multiple of 32 up to 256): what flash_attn() runs below FA_MIN_ROWS_MMA rows.
cudaError_t flash_attn_scalar(const TensorView & q, const TensorView & k, const TensorView & v, const TensorView * mask, const TensorView & dst,
                              float scale, float logit_softcap, cudaStream_t st);

}  // namespace ops
}  // namespace qmm
