/*
 * ggml-b200.h -- the reference-facing drop-in boundary of libggml-b200.so.
 *
 * The library is a ggml *backend plugin*: it exports exactly the two dl entry points the reference's loader looks up
 * (ggml/src/ggml-backend-impl.h:232-271, resolved by load_backend(), ggml/src/ggml-backend-reg.cpp:220-264) and
 * reaches everything else through the five vtables declared in ggml-backend-impl.h:17-230, which it implements in
 * llama.cpp_b200/backend/ggml_b200.cpp.  No other symbol is needed by llama.cpp.
 *
 *   export GGML_BACKEND_PATH=/path/to/libggml-b200.so      # ggml_backend_load_all() dlopens it (reg.cpp:566-593)
 *   llama-bench -m model.gguf -ngl 99 -fa 1 [-sm tensor]   # unmodified reference binaries
 *
 * Registry "B200"; devices "B2000".."B200<n-1>" (one per sm_90 GPU, type GPU, caps async + events); buffer type per
 * device (cudaMalloc, 128-byte tensor alignment, native GGUF block layout); backend = one CUDA stream.
 * get_proc_address() answers: ggml_backend_comm_init / ggml_backend_comm_free / ggml_backend_comm_allreduce_tensor
 * (ggml/include/ggml-backend.h:208-210, used by the meta backend for -sm tensor) and ggml_backend_get_features.
 * supports_op: MUL_MAT / MUL_MAT_ID on Q4_0, Q8_0, Q4_K, Q5_K, Q6_K weights with f32 activations (2-D), and the
 * supporting Llama ops RMS_NORM, MUL, ADD, SCALE, ROPE (normal / neox), SET_ROWS, GET_ROWS, GLU(SWIGLU), CPY/CONT/DUP,
 * FLASH_ATTN_EXT (f16 K/V); everything else is declined and scheduled elsewhere by ggml.
 */
#ifndef GGML_B200_H
#define GGML_B200_H

#ifdef __cplusplus
extern "C" {
#endif

struct ggml_backend_reg;

/* required dl entry point (ggml_backend_init_t): returns the registry object, api_version = GGML_BACKEND_API_VERSION (2) */
struct ggml_backend_reg * ggml_backend_init(void);
/* optional dl entry point (ggml_backend_score_t): 0 when no sm_90 device is usable (the loader then skips the plugin) */
int ggml_backend_score(void);

/* ---- measurement hooks used by bench.py; not part of the ggml interface ---- */
/* journal + snapshot graph inputs on the device so that a captured graph can be replayed */
void ggml_b200_enable_replay(int on);
/* replay the last captured decode graph `reps` times between two CUDA events; 0 on success */
int  ggml_b200_replay_last_graph(int reps, float * ms_out, unsigned long long * kernels_per_replay);
/* re-read the device region of the most recent sizeable device->host tensor read (the logits): after a replay it holds what the
 * replay computed; returns the bytes copied (0 = nothing recorded / buffer too small) */
unsigned long long ggml_b200_reread_last_output(void * dst, unsigned long long cap);
/* bytes through set/get_tensor(_async) and kernels launched (direct + inside graph replays) since load */
void ggml_b200_stats(unsigned long long * h2d_bytes, unsigned long long * d2h_bytes, unsigned long long * kernel_launches);

#ifdef __cplusplus
}
#endif
#endif /* GGML_B200_H */
