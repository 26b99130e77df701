// decode_flow.cuh -- batch-1 decode as ONE persistent dataflow kernel per token (decode_flow.cu).
//
// One CTA per SM stays resident for the whole token and walks a program of phases built from the one-token ggml graph.
// There is NO grid barrier: every vector a phase produces is written as 64-bit (tag, value) slots, and a consumer simply
// polls the slots it needs until they carry the tag of this launch and producer phase (the NCCL "LL" protocol applied to
// on-chip producer/consumer SMs).  A dedicated producer warp per CTA streams the weights of ALL phases through one
// shared-memory ring with cp.async.bulk, so the HBM stream continues across phase boundaries while the consumers wait
// for activations.  See decode_flow.cu for the details and DESIGN.md section 5.3.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <unordered_map>
#include <vector>

namespace qmm {

constexpr int FLOW_MAX_K      = 16384;   // activation length a mat-vec phase can hold (64 blocks of 256)
constexpr int FLOW_MAX_NORM_K = 8192;    // ... with a fused RMS_NORM
constexpr int FLOW_MAX_H      = 8192;    // hidden-state copy kept in shared memory for the residual adds
constexpr int FLOW_PART_ROWS  = 256;     // rows per CTA and phase when a row is split over two warps (K > 8192)

enum { FLOW_MATVEC = 0, FLOW_ATTN = 1, FLOW_COPY = 2, FLOW_ADD = 3, FLOW_SUM = 4 };
constexpr int      FLOW_MAX_PHASES = 2048; // phases per launch (the sync area holds one arrival counter per phase)
constexpr int      FLOW_CNT_BASE  = 64;   // sync words: 0 phase epoch, 1 exit ticket, 2 collective epoch, FLOW_CNT_BASE + q: CTAs that have passed phase q
constexpr int      FLOW_MAX_PEERS = 8;   // GPUs of one tensor-parallel group
constexpr int      FLOW_TRACE_N   = 12;  // trace words per phase and CTA (see FlowProgram::trace)
constexpr uint32_t FLOW_VEC_COLL  = 1;   // FlowVec::flags: the slots were written by the GPUs of the group (see FlowMatvec::peer)

// An f32 vector read by a phase: complete before the launch (plain), or produced by an earlier phase of this launch (ll).
struct FlowVec {
    const float *    plain;
    const uint64_t * ll;
    uint32_t         tag;        // producer phase index + 1; a slot is valid when its high word equals epoch + tag
    uint32_t         flags;      // FLOW_VEC_COLL: tag = index of the collective + 1, valid at collective-epoch + tag (the collective
                                 // epoch advances in lockstep on all GPUs of the group: every launch runs the same collectives)
};
// An f32 vector written by a phase: the ggml tensor's memory (visible after the launch) and/or tagged slots for consumers
// inside the launch.
struct FlowOut {
    float *    plain;
    uint64_t * ll;
};

// dst_m = W_m . q8_K(rms_norm(x) * norm_w)   for up to 3 weight matrices that share x (attn q|k|v, ffn gate|up)
struct FlowMatvec {
    const uint8_t * w[3];
    int64_t         row_stride[3];
    int             M[3];
    int             type[3];         // T_Q4_K | T_Q5_K | T_Q6_K, may differ per matrix
    int             R[3];            // rows per ring piece (host plan)
    FlowOut         out[3];
    FlowVec         x;               // f32 [K]
    FlowVec         residual;        // mode 1
    const float *   norm_w;          // f32 [K] or nullptr
    float *         norm_out;        // optional: the normalised vector itself is a graph output
    float           eps;
    int             K, nmat;
    int             mode;            // 0 store | 1 + residual | 2 SwiGLU pair (out[0] = silu(W0 x) * (W1 x))
    int             keep_h;          // the raw x of this phase is the hidden state: keep it in shared memory
    int             resid_h;         // the residual of this phase is that hidden state
    int             S, seg, RP;      // plan: k-segments per row (1|2), blocks per segment, rows per warp step
    int             plan_pad_[2];
    int             rq[3], rr[3];    // plan: rows per CTA = M / grid and M % grid (CTA c owns rows [c rq + min(c, rr), ...): no division on the device)
    // tensor parallelism (-sm tensor): this GPU's partial result out[0] is ALSO pushed, as tagged slots, into every GPU's exchange
    // region (NVLink peer stores from the epilogue); a FLOW_SUM phase on every GPU then adds the partials in rank order.  This is the
    // all-reduce of ggml_backend_comm_allreduce_tensor fused into the producing and the consuming kernels.
    uint64_t *      peer[FLOW_MAX_PEERS];
    int             npeer;
    uint32_t        coll;            // index of the collective inside the launch
};

// one token: ROPE(q), ROPE(k), K/V cache store, attention over the cache; dst f32 [D, H]
struct FlowAttn {
    FlowVec  q, k, v;                // f32 [D*H], [D*Hkv], [D*Hkv]: the mat-mul outputs, before ROPE
    FlowOut  out;                    // f32 [D*H]
    void *   k_cache; int64_t k_row_bytes;      // cache rows (f16) the new token is stored to: row = idx[0]
    void *   v_cache; int64_t v_row_bytes;
    const int64_t * k_idx; const int64_t * v_idx;
    const int32_t * pos; const float * freq_factors;
    const void * kview; int64_t k_nb1, k_nb2;   // K view [D, n_kv, Hkv] f16: byte strides of a key and of a kv head
    const void * vview; int64_t v_nb1, v_nb2;
    const void * mask;                          // f16 [n_kv] or nullptr
    uint64_t *   part_ll;                       // [n_head * nsplit][D + 2] tagged partials (nsplit > 1)
    int   n_head, n_head_kv, head_dim, n_dims, rope_mode, n_kv, nsplit;
    float freq_scale, ext_factor, attn_factor, theta_scale, corr0, corr1;
    float scale, softcap;
};

struct FlowCopy { FlowVec src; FlowOut out; int n; };             // out = src          (one-row GET_ROWS)
struct FlowAdd  { FlowVec a, b; FlowOut out; int n; };            // out = a + b
// out = src[0] + ... + src[n_first - 1] (the all-reduce: partial sums in rank order), out2 = out + src[n_first] + ... (the residual ADD
// that follows it, folded in by FlowBuilder::add_add; out2.plain == nullptr and n_first == nsrc: no second output).  Spread over all CTAs.
struct FlowSum  { FlowVec src[FLOW_MAX_PEERS + 1]; FlowOut out, out2; int nsrc, n, n_first; };

struct FlowPhase {
    int kind;
    int pad_;
    union {
        FlowMatvec mv;
        FlowAttn   at;
        FlowCopy   cp;
        FlowAdd    ad;
        FlowSum    sm;
    };
};

struct FlowProgram {
    const FlowPhase *    phases;     // device memory
    int                  n_phases;
    unsigned *           sync;       // device, zeroed once: [0] epoch, [1] exit counter, [2] collective epoch
    int                  n_coll;     // collectives (fused all-reduces) in this launch
    // optional [n_phases][FLOW_TRACE_N][160] per phase and CTA (nullptr: off).  globaltimer stamps (ns) of thread 0: 0 phase entered, 1 first
    // prologue pass resolved, 2 activation in registers, 3 warp 0's rows done; 4 / 5 warp 0's cycles waiting for weights / computing;
    // 6 thread 0's first input chunk valid, 7 after the norm reduction, 8 prologue quantised (before the CTA barrier), 9 warp 0's first
    // piece requested; 10 latest moment any warp of the CTA finished its rows (atomicMax), 11 unused
    unsigned long long * trace;
};

size_t      flow_sync_bytes();
size_t      flow_slot_bytes();                                       // bytes of one ring slot (a piece of weight rows must fit)
cudaError_t launch_decode_flow(const FlowProgram & prog, cudaStream_t st);
int         flow_grid(int device);                                   // CTAs of a launch (= SMs)

// Host side: turns a sequence of ops on f32 vectors (named by their device pointers) into a program.  Keeps track of which
// vectors were produced inside the current program (they are read through their tagged slots) and carves those slots out
// of a pool that is reused round-robin -- far enough apart (several layers) that a slot is never rewritten while an
// earlier consumer may still read it (see the reuse argument in decode_flow.cu).
class FlowBuilder {
public:
    void reset(uint64_t * ll_pool, size_t ll_elems, int grid);       // start a new program (pool cursor back to 0)
    void cut();                                                      // everything recorded so far is launched: later reads are plain
    size_t size() const { return phases_.size(); }
    const std::vector<FlowPhase> & phases() const { return phases_; }

    // true if `p` was produced in the current segment WITHOUT slots (too large): the caller has to cut() before reading it
    bool needs_cut(const void * p) const;
    FlowVec vec(const float * p) const;
    FlowOut out(float * p, int n, bool want_ll = true);

    struct MatvecDesc {
        int nmat = 0, K = 0, mode = 0;
        const uint8_t * w[3] = {}; int64_t row_stride[3] = {}; int M[3] = {}; int type[3] = {}; float * dst[3] = {};
        const float * x = nullptr, * residual = nullptr, * norm_w = nullptr; float * norm_out = nullptr; float eps = 0.0f;
    };
    bool matvec_ok(const MatvecDesc & d) const;
    bool add_matvec(const MatvecDesc & d);                           // false: not representable (nothing recorded)
    bool attn_ok(const FlowAttn & a) const;
    // fills q/k/v/out/nsplit/part_ll.  q_vec: the q vector as it was named when its ROPE was postponed (the mat-mul output's buffer may have been
    // handed to another tensor since -- vectors are looked up by address, so a later output at the same address would shadow it)
    bool add_attn(FlowAttn a, const float * q, const float * k, const float * v, float * dst, const FlowVec * q_vec = nullptr);
    bool add_copy(const float * src, float * dst, int n);
    bool add_add(const float * a, const float * b, float * dst, int n);
    int  n_coll() const { return n_coll_; }                          // collectives recorded since the last cut()
    // Fuse an all-reduce over the n builders of a tensor-parallel group: tensors[d] must be the output of the LAST recorded phase of
    // builders[d] (a single-matrix mat-vec); xpool[d] is GPU d's exchange region (slots), xoff the group's cursor into it.
    static bool fuse_allreduce(FlowBuilder * const * builders, int n, float * const * tensors, int nelem, uint64_t * const * xpool, size_t xpool_elems, size_t & xoff);

private:
    struct Produced { uint64_t * ll; uint32_t tag; int n; const float * plain_alias; };
    std::vector<FlowPhase> phases_;
    std::unordered_map<const void *, Produced> produced_;
    const float * h_ptr_ = nullptr;                                  // the vector the CTAs currently hold as hidden state
    const float * h_ptr_copy_ = nullptr;                             // ... and a one-row GET_ROWS copy of it (llama's inp_out_ids in the last layer)
    uint64_t * pool_ = nullptr;
    size_t pool_elems_ = 0, head_ = 0, seg_start_ = 0;
    int n_coll_ = 0;
    int grid_ = 132;
    uint64_t * carve(size_t n);
};

}  // namespace qmm
