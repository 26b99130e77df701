/*
 * b200_flow.h -- host-only checks of the persistent decode kernel's program plan (csrc/decode_flow.cu); conventions, B200_API and
 * the B200_E_* codes: b200_qmm.h.  No device memory is touched: the programs are recorded with the builder the ggml backend uses
 * and inspected, never launched.
 *
 * They live in a header of their own for the reason b200_attn.h does: the plugin's C++ objects compile against b200_qmm.h, and a
 * checkout without the reference sources links objects built elsewhere only when the headers they were compiled against are
 * unchanged.
 */
#ifndef B200_FLOW_H
#define B200_FLOW_H

#include "b200_qmm.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Records a producer phase over an input of K_in elements -- producer_mode 2: a norm + gate|up SwiGLU pair of M rows each (Q4_K),
 * 0: a norm + single Q4_K matrix of M rows -- and then a Q4_K mat-vec of 4096 rows that reads the producer's M-element output (with
 * a fused RMS_NORM of its own if consumer_norm), on `grid` CTAs.
 * Returns 1 when the consumer reads that output as Q8_K blocks the producer phase quantised once, 0 when the consumer quantises the
 * f32 vector itself, B200_E_UNSUPPORTED when a phase is not representable.
 * block_of_cta[0..grid) receives, per CTA of the producer phase, the Q8_K block it quantises (-1: none; all -1 on the f32 route). */
B200_API int b200_flow_q8k_plan(int producer_mode, int64_t M, int64_t K_in, int consumer_norm, int grid, int * block_of_cta);

/* Records n_layers Llama decoder layers (norm + q|k|v with GQA 32/8 heads of 128, attention, attn_output + residual, norm + gate|up
 * SwiGLU of n_ff rows, ffn_down + residual; Q4_K weights, n_embd = 4096) into a program whose tagged-slot pool holds pool_elems slots,
 * on `grid` CTAs.  *n_q8k: phases that read a Q8_K vector.  *min_phases: fewest phases between the phase that writes a slot and the next
 * phase that writes it again (n_phases when no slot is written twice).  Returns 0, or B200_E_UNSUPPORTED when a phase is not
 * representable. */
B200_API int b200_flow_q8k_reuse(int n_layers, int64_t n_ff, int64_t pool_elems, int grid, int * n_q8k, int * min_phases);

#ifdef __cplusplus
}
#endif

#endif /* B200_FLOW_H */
