// ggml_b200.cpp -- the drop-in boundary: an out-of-tree ggml backend ("B200") implementing the reference's five
// plugin vtables (ggml/src/ggml-backend-impl.h:17-230) and the dl entry points ggml_backend_init / ggml_backend_score
// (:232-271) so that unmodified llama.cpp hosts (llama-bench, llama-cli, test-backend-ops, libllama) load it through
// GGML_BACKEND_PATH (ggml-backend-reg.cpp:566-593) and run GGUF models on sm_90a (H100).
//
// Host-side C++ only: tensors are mapped onto plain views / pointers and handed to the hand-written CUDA in ../csrc
// (the same objects that make up libb200qmm.so).  Built from scratch against the interface; ggml-cuda is not ported.
//
//   reg      B200        get_proc_address: ggml_backend_comm_{init,free,allreduce_tensor} (meta backend, -sm tensor)
//   device   B2000..N    one per sm_90 GPU; GPU type; async + events
//   buft     B200<i>     cudaMalloc'd buffers, 128-byte tensor alignment, 256 bytes of tail slack for 16-byte loads
//   backend  one CUDA stream; graph_compute enqueues every node and returns without blocking; graphs whose
//            cgraph->uid repeats are captured once into a CUDA graph and replayed
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <map>
#include <vector>

#include "ggml-backend-impl.h"
#include "ggml-impl.h"
#include "ggml.h"

#include "../csrc/qmm_kernels.cuh"
#include "../csrc/qmm_ops.cuh"
#include "../csrc/decode_flow.cuh"
#include "comm.h"
#include "../../include/b200_qmm.h"

using qmm::ops::TensorView;

#define B200_CHECK(call)                                                                                         \
    do {                                                                                                         \
        cudaError_t e_ = (call);                                                                                 \
        if (e_ != cudaSuccess) {                                                                                 \
            GGML_ABORT("ggml-b200: %s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__);     \
        }                                                                                                        \
    } while (0)

namespace {

constexpr int MAX_DEVICES = 16;
constexpr int N_COUNTERS = 4096;

struct device_ctx {
    int         index;       // position in our registry
    int         cuda_dev;    // CUDA ordinal
    std::string name;        // "B2000"
    std::string desc;
    std::string pci;
    ggml_backend_buffer_type buft;
    std::string buft_name;
};

struct buffer_ctx {
    int    cuda_dev;
    void * base;
};

// One captured CUDA graph per cgraph->uid.  A split keeps its uid while the scheduler does not re-plan it, and a tensor-parallel
// token is ~65 splits per device (the meta backend cuts at every all-reduce), so the cache is a map, not a single slot (round 1's
// single slot never saw a uid twice in a row under -sm tensor and nothing was ever captured).  Every entry owns the device copy of
// its persistent-kernel program: the captured kernel nodes bake in that pointer, so it must not be shared with other graphs.
struct graph_entry {
    int             seen = 0;          // graph_compute calls with this uid
    cudaGraphExec_t exec = nullptr;
    int             n_nodes = 0;
    uint64_t        n_launches = 0;    // kernels inside the captured graph
    qmm::FlowPhase * d_prog = nullptr; // device program of this graph's persistent-kernel launches
    size_t          prog_cap = 0;      // phases d_prog can hold
    size_t          prog_eager = 0;    // phases the eager run of this uid recorded
    uint64_t        last_use = 0;
    bool            no_capture = false;
};
constexpr size_t GRAPH_CACHE_MAX = 512;

struct backend_ctx;
// Tensor parallelism (-sm tensor through the reference's meta backend): the backends of one group defer their one-token sub-graphs --
// graph_compute only RECORDS phases -- and ggml_backend_comm_allreduce_tensor becomes a recorded collective (peer stores from the
// producing mat-vec's epilogue + a FLOW_SUM phase on every GPU), so a whole token is ONE persistent-kernel launch per GPU instead of
// ~65 host-driven segments with an all-reduce kernel between them.  Everything pending is launched (on all GPUs of the group, they
// wait for each other's slots) at the first call that needs results: synchronize, tensor get / set / copy, events, an op the
// persistent kernel cannot run.
struct tp_group {
    std::vector<backend_ctx *> members;              // rank order
    uint64_t * xpool[qmm::FLOW_MAX_PEERS] = {};      // per GPU: exchange region for the partial vectors (tagged slots), two halves
    size_t     xhalf = 0;                            // slots per half; the halves alternate per token so that a GPU that is one launch
    size_t     xoff = 0;                             //   ahead never overwrites slots a slower peer still reads
    int        flip = 0;
};

struct backend_ctx {
    device_ctx * dev;
    cudaStream_t stream = nullptr;
    void *       ws = nullptr;         // mat-mul workspace (quantised activations / GEMM operands)
    size_t       ws_size = 0;
    std::unordered_map<uint64_t, graph_entry> gcache;
    uint64_t     gc_tick = 0;
    graph_entry * last_entry = nullptr;          // entry most recently launched (bench replay hook)
    tp_group *   tp = nullptr;                   // member of a tensor-parallel group: sub-graphs are deferred (see tp_group)
    bool         tp_open = false;                // phases recorded by earlier graph_compute calls are still pending
    qmm::FlowPhase * prog_target = nullptr;       // where the current enqueue's persistent-kernel launches read their program
    bool         prog_deferred = false;          // capture run: the program is uploaded after the capture, not per flush
    size_t       prog_cap_cur = 0;
    unsigned *   counters = nullptr;   // ticket counters for the fused mat-vec's dynamic row-group distribution
    int          counter_next = 0;
    bool         use_graphs = true;
    bool         fuse = true;
    bool         fuse_decode = true;   // gemv3 / rope_kv fusions (GGML_B200_NO_DECODE_FUSION=1 disables)
    bool         debug_hash = false;   // GGML_B200_NODE_HASH
    // one-token graphs in the meta backend's node order (q mm, ROPE q, v mm, k mm, ROPE k ...: no graph_optimize there):
    int          deferred_rope = -1;   // node index of a ROPE(q) that waits for its ROPE(k) to form the attention phase
    qmm::FlowVec deferred_q{};         // ... and the q vector as the builder knew it at that moment (its buffer may be reused before the attention phase is recorded)
    size_t       deferred_seg = 0;     // ... and the number of programs launched so far (a cut in between invalidates the slots)
    struct {                           // RMS_NORM -> MUL whose consumers are mat-muls that are NOT all adjacent: the normalised vector is
        const ggml_tensor * mul = nullptr, * x = nullptr, * w = nullptr;   // never written; every consumer recomputes it from x
        float eps = 0.0f;
        int   remaining = 0;
    } norm_ctx;
    bool         pdl = false;          // programmatic dependent launch (opt-in: GGML_B200_PDL=1)
    // persistent dataflow decode kernel (csrc/decode_flow.cu): phases recorded while walking a one-token graph, flushed as one launch
    bool         mega = false;
    bool         mega_no_attn = false;  // GGML_B200_MEGA_NO_ATTN=1: attention stays a separate launch (debug)
    qmm::FlowBuilder fb;                          // phases recorded by the current enqueue_graph (all segments, in order)
    std::vector<qmm::FlowPhase> mega_mirror;     // host mirror of what d_mega_phases holds
    size_t       mega_flushed = 0;               // phases of the builder already launched
    qmm::FlowPhase * d_mega_phases = nullptr;
    unsigned *   d_mega_sync = nullptr;          // [0] epoch, [1] exit counter
    uint64_t *   d_mega_ll = nullptr;            // pool of tagged slots (the vectors exchanged between phases)
    unsigned long long * d_mega_trace = nullptr;   // GGML_B200_MEGA_TRACE=<file>: timeline of the last launch, dumped at backend free
    std::string  name;
};

std::vector<tp_group *>   g_tp_groups;          // live tensor-parallel groups (buffer-level transfers flush them all)
std::vector<device_ctx *> g_devices;
ggml_backend_reg          g_reg;
std::vector<ggml_backend_device> g_dev_objs;
std::once_flag            g_once;
backend_ctx *             g_last_graph_backend = nullptr;   // most recent backend that replayed a captured graph (bench hook)
std::atomic<uint64_t>     g_h2d_bytes{0}, g_d2h_bytes{0}, g_graph_launches{0};
const void *              g_last_read_src = nullptr;   // most recent device->host tensor read of >= 4 KB (the logits): bench hook
size_t                    g_last_read_size = 0;
int                       g_last_read_dev = 0;
// bench hook: graph inputs (token id, positions, KV indices, mask ...) live in the same compute buffer as the activations and
// their memory is reused later in the graph, so replaying a captured graph needs them restored.  When enabled, every
// host->device tensor write since the previous graph launch is journalled and snapshotted on the device.
struct input_rec { void * dst; size_t size; size_t snap_off; };
bool                      g_journal_on = false;
std::mutex                g_journal_mu;
std::vector<input_rec>    g_journal;            // writes since the last graph launch
std::vector<input_rec>    g_snap_inputs;        // inputs of the most recent graph launch
void *                    g_snap_buf = nullptr;
size_t                    g_snap_cap = 0;
void journal_write(void * dst, size_t size) {
    if (!g_journal_on) return;
    std::lock_guard<std::mutex> lk(g_journal_mu);
    g_journal.push_back({dst, size, 0});
}

inline void set_device(int cuda_dev) { B200_CHECK(cudaSetDevice(cuda_dev)); }

inline TensorView view_of(const ggml_tensor * t) {
    TensorView v;
    v.data = t->data;
    for (int i = 0; i < 4; i++) { v.ne[i] = t->ne[i]; v.nb[i] = (int64_t)t->nb[i]; }
    v.type = (int)t->type;
    return v;
}

inline bool is_quant(ggml_type t) {
    return t == GGML_TYPE_Q4_0 || t == GGML_TYPE_Q8_0 || t == GGML_TYPE_Q4_K || t == GGML_TYPE_Q5_K || t == GGML_TYPE_Q6_K;
}

// ---------------------------------------------------------------------------------------------- buffer
void tp_flush_all();      // launch whatever tensor-parallel groups have pending (defined with the recorder below)
void buf_free(ggml_backend_buffer_t buffer) {
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    cudaFree(c->base);
    delete c;
}
void * buf_get_base(ggml_backend_buffer_t buffer) { return ((buffer_ctx *)buffer->context)->base; }

void buf_memset_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, uint8_t value, size_t offset, size_t size) {
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemsetAsync((char *)tensor->data + offset, value, size, cudaStreamPerThread));
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
}
void buf_set_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemcpyAsync((char *)tensor->data + offset, data, size, cudaMemcpyHostToDevice, cudaStreamPerThread));
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
    g_h2d_bytes += size;
    journal_write((char *)tensor->data + offset, size);
}
void buf_get_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemcpyAsync(data, (const char *)tensor->data + offset, size, cudaMemcpyDeviceToHost, cudaStreamPerThread));
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
    g_d2h_bytes += size;
    if (size >= 4096) { g_last_read_src = (const char *)tensor->data + offset; g_last_read_size = size; g_last_read_dev = c->cuda_dev; }
}
void buf_set_tensor_2d(ggml_backend_buffer_t buffer, ggml_tensor * tensor, const void * data, size_t offset, size_t size, size_t n_copies,
                       size_t stride_tensor, size_t stride_data) {
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemcpy2DAsync((char *)tensor->data + offset, stride_tensor, data, stride_data, size, n_copies, cudaMemcpyHostToDevice, cudaStreamPerThread));
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
}
void buf_get_tensor_2d(ggml_backend_buffer_t buffer, const ggml_tensor * tensor, void * data, size_t offset, size_t size, size_t n_copies,
                       size_t stride_tensor, size_t stride_data) {
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemcpy2DAsync(data, stride_data, (const char *)tensor->data + offset, stride_tensor, size, n_copies, cudaMemcpyDeviceToHost, cudaStreamPerThread));
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
}
void tp_flush_all();
bool buffer_is_ours(ggml_backend_buffer_t b);
bool buf_cpy_tensor(ggml_backend_buffer_t buffer, const ggml_tensor * src, ggml_tensor * dst) {
    ggml_backend_buffer_t sb = src->view_src ? src->view_src->buffer : src->buffer;
    if (!sb || !buffer_is_ours(sb)) return false;
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(src), cudaMemcpyDeviceToDevice, cudaStreamPerThread));   // UVA: peer copies too
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
    return true;
}
void buf_clear(ggml_backend_buffer_t buffer, uint8_t value) {
    tp_flush_all();
    auto * c = (buffer_ctx *)buffer->context;
    set_device(c->cuda_dev);
    B200_CHECK(cudaMemsetAsync(c->base, value, buffer->size, cudaStreamPerThread));
    B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
}

// Quantised tensors are allocated with their size rounded up to 16 bytes (buft_alloc_size) and the pad is zeroed here: the weight
// streams move whole 16-byte granules, so the last granule of the last row may extend up to 15 bytes past the tensor.  (The reference's
// CUDA backend pads rows to 512 elements for the same reason, ggml-cuda.cu:756-775,909-925; our kernels never read further than that
// one granule, and every buffer also carries 256 bytes of tail slack.)
enum ggml_status buf_init_tensor(ggml_backend_buffer_t buffer, ggml_tensor * tensor) {
    if (tensor->view_src != nullptr || !ggml_is_quantized(tensor->type)) return GGML_STATUS_SUCCESS;
    const size_t real = ggml_nbytes(tensor), padded = (real + 15) & ~size_t(15);
    if (padded > real) {
        auto * c = (buffer_ctx *)buffer->context;
        set_device(c->cuda_dev);
        B200_CHECK(cudaMemsetAsync((char *)tensor->data + real, 0, padded - real, cudaStreamPerThread));
        B200_CHECK(cudaStreamSynchronize(cudaStreamPerThread));
    }
    return GGML_STATUS_SUCCESS;
}

const ggml_backend_buffer_i k_buffer_iface = {
    /* .free_buffer   = */ buf_free,
    /* .get_base      = */ buf_get_base,
    /* .init_tensor   = */ buf_init_tensor,
    /* .memset_tensor = */ buf_memset_tensor,
    /* .set_tensor    = */ buf_set_tensor,
    /* .get_tensor    = */ buf_get_tensor,
    /* .set_tensor_2d = */ buf_set_tensor_2d,
    /* .get_tensor_2d = */ buf_get_tensor_2d,
    /* .cpy_tensor    = */ buf_cpy_tensor,
    /* .clear         = */ buf_clear,
    /* .reset         = */ nullptr,
};
bool buffer_is_ours(ggml_backend_buffer_t b) { return b->iface.free_buffer == buf_free; }

// ---------------------------------------------------------------------------------------------- buffer type
const char * buft_name(ggml_backend_buffer_type_t buft) { return ((device_ctx *)buft->context)->buft_name.c_str(); }
ggml_backend_buffer_t buft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    auto * d = (device_ctx *)buft->context;
    set_device(d->cuda_dev);
    void * p = nullptr;
    if (cudaMalloc(&p, size + 256) != cudaSuccess) {       // + slack: kernels may read up to the next 16-byte boundary
        cudaGetLastError();
        GGML_LOG_ERROR("ggml-b200: failed to allocate %.2f MiB on %s\n", size / 1048576.0, d->name.c_str());
        return nullptr;
    }
    auto * c = new buffer_ctx{d->cuda_dev, p};
    return ggml_backend_buffer_init(buft, k_buffer_iface, c, size);
}
size_t buft_alignment(ggml_backend_buffer_type_t) { return 128; }
bool   buft_is_host(ggml_backend_buffer_type_t) { return false; }
size_t buft_alloc_size(ggml_backend_buffer_type_t, const ggml_tensor * tensor) {
    const size_t n = ggml_nbytes(tensor);
    return ggml_is_quantized(tensor->type) ? (n + 15) & ~size_t(15) : n;      // see buf_init_tensor
}
const ggml_backend_buffer_type_i k_buft_iface = {
    /* .get_name       = */ buft_name,
    /* .alloc_buffer   = */ buft_alloc,
    /* .get_alignment  = */ buft_alignment,
    /* .get_max_size   = */ nullptr,
    /* .get_alloc_size = */ buft_alloc_size,
    /* .is_host        = */ buft_is_host,
};
bool buft_is_ours(ggml_backend_buffer_type_t b) { return b->iface.get_name == buft_name; }

// ---------------------------------------------------------------------------------------------- op support
bool rows_contiguous(const ggml_tensor * t) { return t->nb[0] == ggml_type_size(t->type); }

bool supports_op(ggml_backend_dev_t dev, const ggml_tensor * op) {
    const ggml_tensor * s0 = op->src[0];
    const ggml_tensor * s1 = op->src[1];
    // every source that already lives in one of OUR buffers must live on THIS device (cf. ggml-cuda.cu:4866-4874): the kernels
    // dereference tensor->data directly
    if (dev != nullptr) {
        for (int i = 0; i < GGML_MAX_SRC; i++) {
            const ggml_tensor * s = op->src[i];
            if (s == nullptr) continue;
            const ggml_backend_buffer_t sb = s->view_src ? s->view_src->buffer : s->buffer;
            if (sb != nullptr && buft_is_ours(sb->buft) && sb->buft->context != dev->context) return false;
        }
    }
    switch (op->op) {
        case GGML_OP_NONE: case GGML_OP_RESHAPE: case GGML_OP_VIEW: case GGML_OP_PERMUTE: case GGML_OP_TRANSPOSE:
            return true;
        case GGML_OP_MUL_MAT:
            // small dense weights (the MoE router, [n_embd, n_expert] f32): plain 2-D, one warp per output element
            // batched / broadcast (ne12 = r2 * ne02, ne13 = r3 * ne03): one 2-D mat-mul per slice (run_mul_mat_nd); a slice must be an
            // ordinary row-major matrix view (elements contiguous, row stride >= a row), which also covers the permuted cases whose rows stay whole
            if (s1->ne[2] % s0->ne[2] || s1->ne[3] % s0->ne[3] || s1->ne[2] * s1->ne[3] > 4096) return false;
            if ((s0->type == GGML_TYPE_F32 || s0->type == GGML_TYPE_F16) && s1->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32)
                return rows_contiguous(s0) && rows_contiguous(s1) && ggml_is_contiguous(op) &&
                       s0->ne[1] <= 4096 && s0->nb[1] >= ggml_row_size(s0->type, s0->ne[0]) && s1->nb[1] % 4 == 0;
            // the hot path: quantised weight [K, M] x f32 activations [K, N] (ggml.h:1425-1431)
            return is_quant(s0->type) && s1->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 &&
                   rows_contiguous(s0) && rows_contiguous(s1) && ggml_is_contiguous(op) &&
                   s0->nb[1] >= ggml_row_size(s0->type, s0->ne[0]) && s0->nb[1] % 2 == 0 && s0->nb[2] % 2 == 0 && s0->nb[3] % 2 == 0 &&
                   s1->nb[1] % 4 == 0 && s1->nb[2] % 4 == 0 && s1->nb[3] % 4 == 0 &&
                   (s0->ne[0] % 256 == 0 || s0->ne[0] % 32 == 0);
        case GGML_OP_MUL_MAT_ID: {
            const ggml_tensor * ids = op->src[2];
            return is_quant(s0->type) && s1->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && s0->ne[3] == 1 && s1->ne[3] == 1 &&
                   ggml_is_contiguous(s0) && ggml_is_contiguous(s1) && ggml_is_contiguous(op) && ids->type == GGML_TYPE_I32 &&
                   ids->nb[0] == 4 && ids->nb[1] % 4 == 0 && (s1->ne[1] == 1 || s1->ne[1] == ids->ne[0]);
        }
        case GGML_OP_SOFT_MAX: {
            float max_bias = 0.0f;
            memcpy(&max_bias, (const float *)op->op_params + 1, sizeof(float));
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && max_bias == 0.0f && op->src[2] == nullptr && rows_contiguous(s0) && ggml_is_contiguous(op) &&
                   (!s1 || ((s1->type == GGML_TYPE_F16 || s1->type == GGML_TYPE_F32) && rows_contiguous(s1) && s1->ne[0] >= s0->ne[0] && s1->ne[1] >= s0->ne[1]));
        }
        case GGML_OP_ARGSORT:
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_I32 && s0->ne[0] <= 1024 && rows_contiguous(s0) && ggml_is_contiguous(op);
        case GGML_OP_SUM_ROWS:
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && rows_contiguous(s0) && ggml_is_contiguous(op);
        case GGML_OP_CLAMP:
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32;
        case GGML_OP_ADD: case GGML_OP_MUL: case GGML_OP_DIV:
            return s0->type == GGML_TYPE_F32 && s1->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && ggml_can_repeat(s1, s0);
        case GGML_OP_SCALE:
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32;
        case GGML_OP_RMS_NORM:
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && rows_contiguous(s0) && rows_contiguous(op);
        case GGML_OP_ROPE: {
            const int mode = ((const int32_t *)op->op_params)[2];
            const int n_offs = ((const int32_t *)op->op_params)[15];
            return s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && (mode == 0 || mode == 2) && n_offs == 0 && rows_contiguous(s0) &&
                   rows_contiguous(op) && s1->type == GGML_TYPE_I32;
        }
        case GGML_OP_SET_ROWS:
            return s0->type == GGML_TYPE_F32 && s1->type == GGML_TYPE_I64 && (op->type == GGML_TYPE_F32 || op->type == GGML_TYPE_F16) && rows_contiguous(s0);
        case GGML_OP_GET_ROWS:
            return (s0->type == GGML_TYPE_F32 || s0->type == GGML_TYPE_F16 || is_quant(s0->type)) && s1->type == GGML_TYPE_I32 &&
                   op->type == GGML_TYPE_F32 && rows_contiguous(s0) && rows_contiguous(op) && s0->ne[3] == 1;
        case GGML_OP_GLU:
            return ggml_get_glu_op(op) == GGML_GLU_OP_SWIGLU && s0->type == GGML_TYPE_F32 && op->type == GGML_TYPE_F32 && rows_contiguous(s0) &&
                   rows_contiguous(op) && (!s1 || (s1->type == GGML_TYPE_F32 && rows_contiguous(s1)));
        case GGML_OP_CPY: case GGML_OP_CONT: case GGML_OP_DUP:
            return (s0->type == GGML_TYPE_F32 || s0->type == GGML_TYPE_F16) && (op->type == GGML_TYPE_F32 || op->type == GGML_TYPE_F16);
        case GGML_OP_FLASH_ATTN_EXT: {
            const ggml_tensor * k = op->src[1], * v = op->src[2], * mask = op->src[3];
            float max_bias = 0.0f;
            memcpy(&max_bias, (const float *)op->op_params + 1, sizeof(float));
            return s0->type == GGML_TYPE_F32 && k->type == GGML_TYPE_F16 && v->type == GGML_TYPE_F16 && op->src[4] == nullptr && max_bias == 0.0f &&
                   s0->ne[0] == v->ne[0] && s0->ne[0] % 32 == 0 && s0->ne[0] <= 256 && rows_contiguous(s0) && rows_contiguous(k) && rows_contiguous(v) &&
                   (!mask || mask->type == GGML_TYPE_F16) && ggml_is_contiguous(op);
        }
        default:
            return false;
    }
}

// ---------------------------------------------------------------------------------------------- compute
size_t node_workspace(const ggml_tensor * node) {
    if (node->op == GGML_OP_MUL_MAT) {
        const ggml_tensor * w = node->src[0], * x = node->src[1];
        if (!is_quant(w->type)) return 0;
        const size_t a = qmm::act_workspace_bytes((int)w->type, x->ne[1], w->ne[0]);
        const size_t g = qmm::gemm_workspace_bytes((int)w->type, w->ne[1], x->ne[1], w->ne[0]);
        return (a > g ? a : g) + 512;
    }
    if (node->op == GGML_OP_MUL_MAT_ID) {
        const ggml_tensor * w = node->src[0], * b = node->src[1], * ids = node->src[2];
        const size_t a = qmm::act_workspace_bytes((int)w->type, b->ne[1] * b->ne[2], w->ne[0]);
        const size_t g = qmm::gemm_grouped_workspace_bytes((int)w->type, w->ne[1], ids->ne[0] * b->ne[2], w->ne[2], w->ne[0]);
        return (a > g ? a : g) + 512;
    }
    if (node->op == GGML_OP_FLASH_ATTN_EXT) {
        if (node->src[3]) { const TensorView m = view_of(node->src[3]); return qmm::ops::flash_attn_workspace_bytes(view_of(node->src[0]), view_of(node->src[1]), &m); }
        return qmm::ops::flash_attn_workspace_bytes(view_of(node->src[0]), view_of(node->src[1]), nullptr);
    }
    return 0;
}

struct act_cache_t {                  // quantised activations of the previous mat-mul, reusable while src1 is unchanged
    const void * src = nullptr;
    int64_t      n = 0, k = 0;
    int          act_k8 = -1;
};

cudaError_t run_mul_mat(backend_ctx * b, const ggml_tensor * node, act_cache_t & ac, const ggml_tensor * residual) {
    const ggml_tensor * w = node->src[0], * x = node->src[1];
    if (w->type == GGML_TYPE_F32 || w->type == GGML_TYPE_F16) {
        if (residual != nullptr) return cudaErrorNotSupported;
        return qmm::ops::mul_mat_f(view_of(w), view_of(x), view_of(node), b->stream);
    }
    const int type = (int)w->type;
    const int64_t M = w->ne[1], K = w->ne[0], N = x->ne[1];
    const int64_t ldx = (int64_t)(x->nb[1] / sizeof(float)), ldd = (int64_t)(node->nb[1] / sizeof(float));
    if (N > 8 && qmm::gemm_workspace_bytes(type, M, N, K) != 0) {
        qmm::GemmArgs g{};
        g.w = (const uint8_t *)w->data; g.row_stride = (int64_t)w->nb[1]; g.M = (int)M; g.K = (int)K; g.N = (int)N;
        g.x = (const float *)x->data; g.ldx = ldx; g.dst = (float *)node->data; g.ldd = ldd; g.workspace = b->ws; g.workspace_bytes = b->ws_size;
        // consecutive mat-muls on one activation (attn_q|k|v, ffn_gate|up) share the fp16-integer operand images in the workspace
        g.reuse_operands = b->fuse && ac.src == x->data && ac.n == N && ac.k == K && ac.act_k8 == 2;
        const cudaError_t ge = qmm::launch_gemm(type, g, b->stream);
        if (ge != cudaErrorMisalignedAddress) {           // (a batch slice / permuted view the GEMM's 16-byte loads cannot take: column chunks below)
            ac.src = x->data; ac.n = N; ac.k = K; ac.act_k8 = 2;
            return ge;
        }
    }
    const qmm::ActQ8 act = qmm::act_carve(type, b->ws, N, K);
    const int k8 = (w->type == GGML_TYPE_Q4_K || w->type == GGML_TYPE_Q5_K || w->type == GGML_TYPE_Q6_K) ? 1 : 0;
    if (!(b->fuse && ac.src == x->data && ac.n == N && ac.k == K && ac.act_k8 == k8)) {
        cudaError_t e = qmm::launch_quantize_act(type, (const float *)x->data, ldx, N, K, act, b->stream);
        if (e != cudaSuccess) return e;
        ac.src = x->data; ac.n = N; ac.k = K; ac.act_k8 = k8;
    }
    for (int64_t n0 = 0; n0 < N; n0 += 8) {
        qmm::GemvArgs a{};
        a.w = (const uint8_t *)w->data; a.row_stride = (int64_t)w->nb[1]; a.expert_stride = 0; a.M = (int)M; a.K = (int)K;
        a.ncols = (int)(N - n0 < 8 ? N - n0 : 8); a.nz = 1;
        a.act = act; a.act.qs += n0 * act.qs_stride; a.act.d += n0 * act.d_stride; a.act.bsums += n0 * act.bs_stride;
        a.dst = (float *)node->data + n0 * ldd; a.ldd = ldd;
        a.residual = residual ? (const float *)residual->data + n0 * ldd : nullptr;
        a.ids = nullptr;
        cudaError_t e = qmm::launch_gemv(type, a, b->stream);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// Batched / broadcast mat-mul (ggml_compute_forward_mul_mat's i12/i13 loop with r2 = ne12/ne02, r3 = ne13/ne03, ggml-cpu.c:1254-1452):
// dst[:, :, i12, i13] = w[:, :, i12 / r2, i13 / r3] . x[:, :, i12, i13] -- one 2-D mat-mul per (i12, i13) slice on the same kernels.
cudaError_t run_mul_mat_nd(backend_ctx * b, const ggml_tensor * node, act_cache_t & ac, const ggml_tensor * residual) {
    const ggml_tensor * w = node->src[0], * x = node->src[1];
    if (x->ne[2] == 1 && x->ne[3] == 1) return run_mul_mat(b, node, ac, residual);
    if (residual != nullptr) return cudaErrorNotSupported;
    const int64_t r2 = x->ne[2] / w->ne[2], r3 = x->ne[3] / w->ne[3];
    for (int64_t i13 = 0; i13 < x->ne[3]; i13++) {
        for (int64_t i12 = 0; i12 < x->ne[2]; i12++) {
            ggml_tensor ws = *w, xs = *x, ds = *node;
            ws.data = (char *)w->data + (i12 / r2) * w->nb[2] + (i13 / r3) * w->nb[3];
            xs.data = (char *)x->data + i12 * x->nb[2] + i13 * x->nb[3];
            ds.data = (char *)node->data + i12 * node->nb[2] + i13 * node->nb[3];
            for (ggml_tensor * t : {&ws, &xs, &ds}) { t->ne[2] = 1; t->ne[3] = 1; }
            ds.src[0] = &ws; ds.src[1] = &xs;
            const cudaError_t e = run_mul_mat(b, &ds, ac, nullptr);
            if (e != cudaSuccess) return e;
        }
    }
    ac.src = nullptr;                                     // (the cache keys on the slice pointer only: do not let a later node match a slice)
    return cudaSuccess;
}

cudaError_t run_mul_mat_id(backend_ctx * b, const ggml_tensor * node) {
    const ggml_tensor * w = node->src[0], * x = node->src[1], * ids = node->src[2];
    const int type = (int)w->type;
    const int64_t K = w->ne[0], M = w->ne[1], n_expert = w->ne[2], nb1 = x->ne[1], T = x->ne[2], n_used = ids->ne[0];
    // many (token, slot) rows: group them by expert and run the wgmma GEMM once per expert tile (the per-row GEMV below would stream
    // an expert's weights once per row)
    static const bool no_grouped = getenv("GGML_B200_NO_GROUPED_GEMM") != nullptr;
    if (!no_grouped && T * n_used >= 32 && qmm::gemm_grouped_workspace_bytes(type, M, T * n_used, n_expert, K) != 0) {
        qmm::GemmGroupedArgs ga{};
        ga.w = (const uint8_t *)w->data; ga.row_stride = (int64_t)w->nb[1]; ga.expert_stride = (int64_t)w->nb[2]; ga.M = (int)M; ga.K = (int)K; ga.n_expert = (int)n_expert;
        ga.x = (const float *)x->data; ga.ldx = (int64_t)(x->nb[1] / 4); ga.nb1 = (int)nb1;
        ga.ids = (const int32_t *)ids->data; ga.ids_stride = (int64_t)(ids->nb[1] / 4); ga.T = (int)T; ga.n_used = (int)n_used;
        ga.dst = (float *)node->data; ga.ldd = M; ga.workspace = b->ws; ga.workspace_bytes = b->ws_size;
        const cudaError_t ge = qmm::launch_gemm_grouped(type, ga, b->stream);
        if (ge != cudaErrorNotSupported && ge != cudaErrorMisalignedAddress) return ge;
        cudaGetLastError();
    }
    const qmm::ActQ8 act = qmm::act_carve(type, b->ws, nb1 * T, K);
    cudaError_t e = qmm::launch_quantize_act(type, (const float *)x->data, K, nb1 * T, K, act, b->stream);
    if (e != cudaSuccess) return e;
    const int64_t t_chunk = 65535 / n_used;
    for (int64_t t0 = 0; t0 < T; t0 += t_chunk) {
        const int64_t nt = T - t0 < t_chunk ? T - t0 : t_chunk;
        qmm::GemvArgs a{};
        a.w = (const uint8_t *)w->data; a.row_stride = (int64_t)w->nb[1]; a.expert_stride = (int64_t)w->nb[2]; a.M = (int)M; a.K = (int)K;
        a.ncols = 1; a.nz = (int)(nt * n_used);
        a.act = act; a.act.qs += t0 * nb1 * act.qs_stride; a.act.d += t0 * nb1 * act.d_stride; a.act.bsums += t0 * nb1 * act.bs_stride;
        a.dst = (float *)node->data + t0 * n_used * M; a.ldd = M; a.residual = nullptr;
        a.ids = (const int32_t *)ids->data + t0 * (int64_t)(ids->nb[1] / 4); a.ids_stride = (int64_t)(ids->nb[1] / 4);
        a.n_used = (int)n_used; a.nb1 = (int)nb1; a.n_expert = (int)n_expert;
        e = qmm::launch_gemv(type, a, b->stream);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

inline bool is_noop(const ggml_tensor * n) {
    return ggml_is_empty(n) || n->op == GGML_OP_NONE || n->op == GGML_OP_RESHAPE || n->op == GGML_OP_VIEW || n->op == GGML_OP_PERMUTE ||
           n->op == GGML_OP_TRANSPOSE || (n->flags & GGML_TENSOR_FLAG_COMPUTE) == 0;
}


// ---------------------------------------------------------------------------------------------- decode fusions (N = 1)
inline bool is_kquant(ggml_type t) { return t == GGML_TYPE_Q4_K || t == GGML_TYPE_Q5_K || t == GGML_TYPE_Q6_K; }

inline int next_compute(const ggml_cgraph * g, int i) {           // index of the next node that launches work, or n_nodes
    while (i < g->n_nodes && is_noop(g->nodes[i])) i++;
    return i;
}

// a mat-mul the fused mat-vec can take: K-quant weight [K, M], one f32 activation column, contiguous
inline bool decode_mm_ok(const ggml_tensor * n) {
    if (n->op != GGML_OP_MUL_MAT) return false;
    const ggml_tensor * w = n->src[0], * x = n->src[1];
    return is_kquant(w->type) && x->type == GGML_TYPE_F32 && x->ne[1] == 1 && x->ne[2] == 1 && x->ne[3] == 1 && w->ne[2] == 1 && w->ne[3] == 1 &&
           w->ne[0] % 256 == 0 && ggml_is_contiguous(x) && ((uintptr_t)x->data & 15) == 0 && ggml_is_contiguous(n);
}

// Look ahead for the weights of the next decode mat-vec launch (for the L2 prefetch issued by the current one).
void find_next_weights(const ggml_cgraph * g, int from, qmm::FusedGemvArgs & a) {
    static const bool enabled = getenv("GGML_B200_L2_PREFETCH") != nullptr;   // opt-in: measured slightly negative (it queues ahead of demand loads)
    if (!enabled) return;
    int64_t budget = 32ll << 20;                                   // leave room in the 50 MB L2 for the current stream
    for (int j = from; j < g->n_nodes; j++) {
        const ggml_tensor * n = g->nodes[j];
        if (is_noop(n) || !decode_mm_ok(n)) continue;
        int k = 0;
        for (int jj = j; jj < g->n_nodes && k < 3; jj++) {
            const ggml_tensor * m = g->nodes[jj];
            if (is_noop(m)) continue;
            if (!decode_mm_ok(m) || m->src[1] != n->src[1]) break;
            int64_t bytes = (int64_t)ggml_nbytes(m->src[0]);
            if (bytes > budget) bytes = budget;
            bytes &= ~int64_t(15);
            if (bytes <= 0) break;
            a.next_w[k] = (const uint8_t *)m->src[0]->data; a.next_bytes[k] = bytes; budget -= bytes; k++;
        }
        return;
    }
}


// ---------------------------------------------------------------------------------------------- persistent decode kernel: recorder
constexpr size_t MEGA_MAX_PHASES = 2048;
constexpr size_t MEGA_LL_ELEMS = 512 * 1024;            // tagged slots: 4 MB, ~16 Llama-8B layers of phase outputs between reuses

bool mega_alloc(backend_ctx * b) {
    if (b->d_mega_phases) return true;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(b->stream, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) return false;
    if (cudaMalloc(&b->d_mega_phases, MEGA_MAX_PHASES * sizeof(qmm::FlowPhase)) != cudaSuccess) { cudaGetLastError(); b->d_mega_phases = nullptr; b->mega = false; return false; }
    if (cudaMalloc(&b->d_mega_sync, qmm::flow_sync_bytes()) != cudaSuccess || cudaMalloc(&b->d_mega_ll, MEGA_LL_ELEMS * sizeof(uint64_t)) != cudaSuccess) {
        cudaGetLastError(); b->mega = false; return false;
    }
    // zeroed ON THE BACKEND'S STREAM: it is a non-blocking stream, so a legacy-stream cudaMemset is not ordered before the first launch
    cudaMemsetAsync(b->d_mega_sync, 0, qmm::flow_sync_bytes(), b->stream);
    cudaMemsetAsync(b->d_mega_ll, 0, MEGA_LL_ELEMS * sizeof(uint64_t), b->stream);   // tag 0 is never valid (tags start at epoch + 1)
    const size_t trace_words = MEGA_MAX_PHASES * qmm::FLOW_TRACE_N * 160;
    if (getenv("GGML_B200_MEGA_TRACE") && cudaMalloc(&b->d_mega_trace, trace_words * sizeof(unsigned long long)) == cudaSuccess)
        cudaMemsetAsync(b->d_mega_trace, 0, trace_words * sizeof(unsigned long long), b->stream);
    else b->d_mega_trace = nullptr;
    b->mega_mirror.clear();
    return true;
}

// Launch the phases recorded since the previous flush.  The program lives in device memory; it is (re)uploaded only when it
// differs from what is there.  While a CUDA graph is being captured nothing is uploaded: the launches read the graph entry's own
// program buffer, which graph_compute fills right after the capture.
// GGML_B200_FLOW_DEBUG: why programs were cut short -- (reason -> launches, phases) printed when a backend is freed
static std::map<std::string, std::pair<long, long>> g_flush_stats;
static const char * g_flush_why = "end of graph";
struct flush_why { const char * prev; explicit flush_why(const char * w) : prev(g_flush_why) { g_flush_why = w; } ~flush_why() { g_flush_why = prev; } };
void flush_stats_dump() {
    static const bool on = getenv("GGML_B200_FLOW_DEBUG") != nullptr;
    if (!on || g_flush_stats.empty()) return;
    for (auto & kv : g_flush_stats) fprintf(stderr, "ggml-b200: flow launches because \"%s\": %ld (%ld phases)\n", kv.first.c_str(), kv.second.first, kv.second.second);
    g_flush_stats.clear();
}

cudaError_t mega_flush_one(backend_ctx * b) {
    const size_t n0 = b->mega_flushed, n1 = b->fb.size();
    if (b->deferred_rope >= 0 && n1 > n0) {
        GGML_LOG_ERROR("ggml-b200: program cut (%s) while a ROPE(q) is postponed\n", g_flush_why);
        return cudaErrorUnknown;
    }
    if (n1 > n0) { auto & st = g_flush_stats[g_flush_why]; st.first++; st.second += (long)(n1 - n0); }
    b->tp_open = false;
    if (n1 == n0) return cudaSuccess;
    if (n1 > MEGA_MAX_PHASES || !b->d_mega_phases) return cudaErrorMemoryAllocation;
    const size_t bytes = (n1 - n0) * sizeof(qmm::FlowPhase);
    const qmm::FlowPhase * rec = b->fb.phases().data();
    qmm::FlowPhase * target = b->d_mega_phases;
    if (b->prog_deferred) {
        if (n1 > b->prog_cap_cur) return cudaErrorStreamCaptureUnsupported;                     // aborts the capture; the graph stays eager
        target = b->prog_target;
    } else {
        const bool same = b->mega_mirror.size() >= n1 && memcmp(b->mega_mirror.data() + n0, rec + n0, bytes) == 0;
        if (!same) {
            cudaError_t e = cudaMemcpyAsync(b->d_mega_phases + n0, rec + n0, bytes, cudaMemcpyHostToDevice, b->stream);
            if (e != cudaSuccess) return e;
            if (b->mega_mirror.size() < n1) b->mega_mirror.resize(n1);
            memcpy(b->mega_mirror.data() + n0, rec + n0, bytes);
        }
    }
    qmm::FlowProgram prog{target + n0, (int)(n1 - n0), b->d_mega_sync, b->fb.n_coll(), b->d_mega_trace ? b->d_mega_trace + n0 * qmm::FLOW_TRACE_N * 160 : nullptr};
    b->mega_flushed = n1;
    b->fb.cut();                                        // what was recorded so far is complete memory for everything that follows
    return qmm::launch_decode_flow(prog, b->stream);
}

// Launch what is pending.  In a tensor-parallel group that means on EVERY GPU of the group: their kernels exchange partial results and
// wait for each other.
cudaError_t mega_flush(backend_ctx * b) {
    if (b->tp == nullptr) return mega_flush_one(b);
    cudaError_t err = cudaSuccess;
    bool any = false;
    for (backend_ctx * m : b->tp->members) {
        if (m->fb.size() == m->mega_flushed) { m->tp_open = false; continue; }
        any = true;
        set_device(m->dev->cuda_dev);
        const cudaError_t e = mega_flush_one(m);
        if (e != cudaSuccess && err == cudaSuccess) err = e;
    }
    if (any) { b->tp->xoff = 0; b->tp->flip ^= 1; }
    set_device(b->dev->cuda_dev);
    return err;
}
void tp_flush_all() {
    flush_why w("buffer-level tensor access");
    for (tp_group * g : g_tp_groups) if (!g->members.empty()) mega_flush(g->members[0]);
}

double flow_max_mb() { static const double v = [] { const char * e = getenv("GGML_B200_FLOW_MAX_MB"); return e ? atof(e) : 0.0; }(); return v; }
// a fused mat-vec either becomes a phase of the persistent kernel or its own launch
cudaError_t emit_fused_gemv(backend_ctx * b, const int * types, const qmm::FusedGemvArgs & a, float * norm_out = nullptr) {
    // experiment switch: mat-vecs whose weights exceed GGML_B200_FLOW_MAX_MB (the output head: 431 MB of Q6_K) leave the persistent kernel
    // and run as their own launch on the per-op mat-vec kernel
    bool too_big = false;
    if (flow_max_mb() > 0.0) {
        double mb = 0.0;
        for (int i = 0; i < a.nmat && i < 3; i++) mb += (double)a.M[i] * (double)a.row_stride[i] / 1048576.0;
        too_big = mb > flow_max_mb();
    }
    if (b->mega && !too_big && a.x != nullptr && b->d_mega_phases && b->fb.size() < MEGA_MAX_PHASES) {
        qmm::FlowBuilder::MatvecDesc d;
        d.nmat = a.nmat; d.K = a.K; d.mode = a.mode;
        for (int i = 0; i < a.nmat && i < 3; i++) { d.w[i] = a.w[i]; d.row_stride[i] = a.row_stride[i]; d.M[i] = a.M[i]; d.type[i] = types[i]; d.dst[i] = a.dst[i]; }
        d.x = a.x; d.residual = a.residual[0]; d.norm_w = a.has_norm ? a.norm_w : nullptr; d.norm_out = norm_out; d.eps = a.eps;
        if (b->fb.needs_cut(d.x) || (d.residual && b->fb.needs_cut(d.residual))) { flush_why w("mat-vec input is plain memory written by a pending phase"); const cudaError_t e = mega_flush(b); if (e != cudaSuccess) return e; }
        if (b->fb.add_matvec(d)) return cudaSuccess;
    }
    if (b->mega) { flush_why w("mat-vec not accepted by the builder"); const cudaError_t e = mega_flush(b); if (e != cudaSuccess) return e; }
    if (norm_out != nullptr) return cudaErrorNotSupported;                 // the stand-alone kernel does not materialise the normalised vector
    for (int i = 1; i < a.nmat; i++) if (types[i] != types[0]) return cudaErrorNotSupported;
    return qmm::launch_fused_gemv(types[0], a, b->stream);
}

// Pattern A: RMS_NORM -> MUL(w) -> k mat-muls on that vector [-> GLU(swiglu) for a gate/up pair].
// Pattern B: a lone mat-mul [-> ADD residual].  Returns the number of graph nodes handled (0 = no match).
int try_fuse_matvec_impl(backend_ctx * b, ggml_cgraph * g, int i, cudaError_t & err) {
    err = cudaSuccess;
    static const int fuse_mask = [] { const char * e = getenv("GGML_B200_FUSE_MASK"); return e ? atoi(e) : 15; }();   // bisection: 1 norm+group, 2 swiglu, 4 residual, 8 lone
    ggml_tensor * n0 = g->nodes[i];
    const ggml_tensor * x = nullptr, * norm_w = nullptr;
    float eps = 0.0f;
    float * norm_out = nullptr;
    int first_mm = i;
    int64_t expected_uses = -1;
    const ggml_tensor * cont_mul = nullptr;
    if (n0->op == GGML_OP_RMS_NORM) {
        const int i1 = next_compute(g, i + 1);
        if (i1 >= g->n_nodes) return 0;
        ggml_tensor * mul = g->nodes[i1];
        if (mul->op != GGML_OP_MUL || mul->src[0] != n0 || !ggml_node_has_n_uses(g, i, 1)) return 0;
        const ggml_tensor * w = mul->src[1];
        if (w->type != GGML_TYPE_F32 || !ggml_is_contiguous(w) || w->ne[0] != n0->ne[0] || ggml_nelements(w) != w->ne[0] || ((uintptr_t)w->data & 15)) return 0;
        if (n0->ne[1] != 1 || n0->ne[2] != 1 || n0->ne[3] != 1 || n0->ne[0] > 8192 || n0->ne[0] % 256) return 0;
        const ggml_tensor * src = n0->src[0];
        if (src->type != GGML_TYPE_F32 || !ggml_is_contiguous(src) || ((uintptr_t)src->data & 15)) return 0;
        // the normalised vector itself is a graph output (result_norm): only the persistent kernel can also materialise it
        if ((mul->flags & GGML_TENSOR_FLAG_OUTPUT) && !(b->mega && b->d_mega_phases)) return 0;
        norm_out = (mul->flags & GGML_TENSOR_FLAG_OUTPUT) ? (float *)mul->data : nullptr;
        memcpy(&eps, n0->op_params, sizeof(float));
        x = src; norm_w = w;
        first_mm = next_compute(g, i1 + 1);
        expected_uses = ggml_node_get_use_count(g, i1);
        // every consumer of the normalised vector must be one of the mat-muls we fuse (the vector itself is never written)
        int found = 0, j = first_mm;
        while (j < g->n_nodes && found < 3) {
            ggml_tensor * mm = g->nodes[j];
            if (!decode_mm_ok(mm) || mm->src[1] != mul) break;
            if (flow_max_mb() > 0.0 && (double)ggml_nbytes(mm->src[0]) / 1048576.0 > flow_max_mb()) return 0;   // (experiment switch: see emit_fused_gemv)
            found++;
            j = next_compute(g, j + 1);
        }
        if (found == 0) return 0;
        b->norm_ctx.mul = nullptr;
        if (found != expected_uses) {
            // The meta backend's node order (no graph_optimize there): q mm, ROPE q, v mm, k mm.  The remaining consumers must be decode
            // mat-muls further down and nothing else may read the normalised vector, which is then never written: each group of
            // consumers recomputes it from x in its own prologue (persistent kernel only).
            int later = 0;
            for (int jj = j; jj < g->n_nodes; jj++) {
                const ggml_tensor * t = g->nodes[jj];
                bool uses = false;
                for (int si = 0; si < GGML_MAX_SRC; si++) uses = uses || t->src[si] == mul;
                if (!uses) continue;
                if (!decode_mm_ok(t) || t->src[1] != mul) return 0;
                later++;
            }
            if (!(b->mega && b->d_mega_phases) || found + later != expected_uses || norm_out != nullptr) return 0;
            b->norm_ctx.mul = mul; b->norm_ctx.x = src; b->norm_ctx.w = w; b->norm_ctx.eps = eps; b->norm_ctx.remaining = later;
        }
    } else if (n0->op == GGML_OP_MUL_MAT) {
        if (!decode_mm_ok(n0)) return 0;
        x = n0->src[1];
        if (!(fuse_mask & 12)) return 0;
        if (b->norm_ctx.mul != nullptr && b->norm_ctx.remaining > 0 && n0->src[1] == b->norm_ctx.mul) {   // a later consumer of an unwritten normalised vector
            cont_mul = b->norm_ctx.mul;
            x = b->norm_ctx.x; norm_w = b->norm_ctx.w; eps = b->norm_ctx.eps;
        }
    } else {
        return 0;
    }

    // collect the consecutive mat-muls on x
    ggml_tensor * mms[3];
    int idx[3];
    int nmm = 0, j = first_mm;
    const ggml_tensor * xin = cont_mul ? cont_mul : (norm_w ? g->nodes[next_compute(g, i + 1)] : x);      // the tensor the mat-muls name as src1
    while (j < g->n_nodes && nmm < 3) {
        ggml_tensor * mm = g->nodes[j];
        if (!decode_mm_ok(mm) || mm->src[1] != xin) break;
        if (nmm > 0 && !norm_w) break;                                             // pattern B fuses one mat-mul (its activation is quantised in-kernel)
        mms[nmm] = mm; idx[nmm] = j; nmm++;
        j = next_compute(g, j + 1);
    }
    if (nmm == 0) return 0;
    if (cont_mul) b->norm_ctx.remaining -= nmm;
    int end = j;                                                                   // first node not yet handled

    // large K (ffn_down): quantising 14336 activations inside each of ~300 CTAs costs more than one extra small launch
    const int Kdim = (int)mms[0]->src[0]->ne[0];
    const bool external_q = !norm_w && Kdim > 8192 && !(b->mega && Kdim <= qmm::FLOW_MAX_K);
    qmm::ActQ8 ext_act{};
    if (external_q) {
        if (b->mega) { flush_why w("K too large: external activation quantisation"); err = mega_flush(b); if (err != cudaSuccess) return 0; }
        ext_act = qmm::act_carve((int)mms[0]->src[0]->type, b->ws, 1, Kdim);
        err = qmm::launch_quantize_act((int)mms[0]->src[0]->type, (const float *)x->data, Kdim, 1, Kdim, ext_act, b->stream);
        if (err != cudaSuccess) return 0;
    }
    auto fill = [&](qmm::FusedGemvArgs & a) {
        a = qmm::FusedGemvArgs{};
        a.K = Kdim;
        a.x = external_q ? nullptr : (const float *)x->data;
        a.act = ext_act;
        a.norm_w = norm_w ? (const float *)norm_w->data : nullptr;
        a.eps = eps; a.has_norm = norm_w ? 1 : 0; a.pdl = b->pdl ? 1 : 0;
        a.counter = (b->counters && b->counter_next < N_COUNTERS) ? b->counters + b->counter_next++ : nullptr;
    };
    auto set_mat = [&](qmm::FusedGemvArgs & a, int slot, const ggml_tensor * mm, float * dst) {
        a.w[slot] = (const uint8_t *)mm->src[0]->data; a.row_stride[slot] = (int64_t)mm->src[0]->nb[1]; a.M[slot] = (int)mm->src[0]->ne[1]; a.dst[slot] = dst;
    };

    // SwiGLU pair: exactly [gate, up] of one type, both used only by the GLU that follows
    if ((fuse_mask & 2) && nmm == 2 && mms[0]->src[0]->type == mms[1]->src[0]->type && mms[0]->ne[0] == mms[1]->ne[0] && end < g->n_nodes) {
        ggml_tensor * glu = g->nodes[end];
        if (glu->op == GGML_OP_GLU && ggml_get_glu_op(glu) == GGML_GLU_OP_SWIGLU && glu->src[0] == mms[0] && glu->src[1] == mms[1] &&
            ((const int32_t *)glu->op_params)[1] == 0 && ggml_node_has_n_uses(g, idx[0], 1) && ggml_node_has_n_uses(g, idx[1], 1) && ggml_is_contiguous(glu)) {
            qmm::FusedGemvArgs a;
            fill(a);
            a.nmat = 2; a.mode = 2;
            set_mat(a, 0, mms[0], (float *)glu->data);
            set_mat(a, 1, mms[1], (float *)glu->data);
            find_next_weights(g, end + 1, a);
            const int ty[3] = {(int)mms[0]->src[0]->type, (int)mms[1]->src[0]->type, 0};
            err = emit_fused_gemv(b, ty, a, norm_out);
            if (err == cudaErrorNotSupported) { err = cudaSuccess; return 0; }
            return next_compute(g, end + 1) - i;
        }
    }
    // residual: a single mat-mul followed by ADD(mm, r)
    if ((fuse_mask & 4) && nmm == 1 && end < g->n_nodes) {
        ggml_tensor * add = g->nodes[end];
        if (add->op == GGML_OP_ADD && (add->src[0] == mms[0] || add->src[1] == mms[0]) && ggml_node_has_n_uses(g, idx[0], 1)) {
            const ggml_tensor * other = add->src[0] == mms[0] ? add->src[1] : add->src[0];
            if (other->type == GGML_TYPE_F32 && ggml_are_same_shape(other, mms[0]) && ggml_is_contiguous(other) && ggml_is_contiguous(add)) {
                qmm::FusedGemvArgs a;
                fill(a);
                a.nmat = 1; a.mode = 1;
                set_mat(a, 0, mms[0], (float *)add->data);
                a.residual[0] = (const float *)other->data;
                find_next_weights(g, end + 1, a);
                const int ty[3] = {(int)mms[0]->src[0]->type, 0, 0};
                err = emit_fused_gemv(b, ty, a, norm_out);
                if (err == cudaErrorNotSupported) { err = cudaSuccess; return 0; }
                return next_compute(g, end + 1) - i;
            }
        }
    }
    // plain: group consecutive mat-muls into one launch each -- same type for the stand-alone kernel, any K-quant mix (attn_q|k Q4_K +
    // attn_v Q6_K) for the persistent kernel
    if (norm_w ? !(fuse_mask & 1) : !(fuse_mask & 8)) return 0;
    const bool mix = b->mega && b->d_mega_phases != nullptr && !external_q;
    int k = 0;
    while (k < nmm) {
        int k2 = k + 1;
        while (k2 < nmm && (mix || mms[k2]->src[0]->type == mms[k]->src[0]->type)) k2++;
        qmm::FusedGemvArgs a;
        fill(a);
        a.nmat = k2 - k; a.mode = 0;
        for (int m = k; m < k2; m++) set_mat(a, m - k, mms[m], (float *)mms[m]->data);
        find_next_weights(g, k2 < nmm ? idx[k2] : end, a);
        int ty[3] = {0, 0, 0};
        for (int m = k; m < k2; m++) ty[m - k] = (int)mms[m]->src[0]->type;
        if (norm_out != nullptr && (k != 0 || k2 != nmm)) { err = cudaSuccess; return 0; }   // (only a single group can carry the norm output)
        err = emit_fused_gemv(b, ty, a, norm_out);
        if (err == cudaErrorNotSupported) {
            err = cudaSuccess;
            if (k == 0) return 0;                                                  // nothing launched yet: generic path
            return 0;                                                              // (a later group can only differ by type, which decode_mm_ok already vetted)
        }
        if (err != cudaSuccess) return 0;
        k = k2;
    }
    return end - i;
}

// Pattern C (one token): ROPE(Q), ROPE(K), SET_ROWS(K cache <- roped K), SET_ROWS(V cache <- V) -> one launch.
int try_fuse_matvec(backend_ctx * b, ggml_cgraph * g, int i, cudaError_t & err) {
    const int used = try_fuse_matvec_impl(b, g, i, err);
    if (used == 0 && g->nodes[i]->op == GGML_OP_RMS_NORM) b->norm_ctx.mul = nullptr;    // the generic path writes the normalised vector
    return used;
}

// GGML_B200_FLOW_DEBUG: which condition made the ROPE + KV-store pattern decline (first few times per condition)
int rope_decline(const ggml_cgraph * g, int i, int which) {
    static const bool on = getenv("GGML_B200_FLOW_DEBUG") != nullptr;
    static int said[32] = {};
    if (on && which < 32 && said[which]++ < 2) {
        fprintf(stderr, "ggml-b200: ROPE/KV pattern declined at condition %d, node %d of %d:", which, i, g->n_nodes);
        for (int j = i; j < g->n_nodes && j < i + 8; j++) {
            const ggml_tensor * t = g->nodes[j];
            fprintf(stderr, " [%s %s ne=%lldx%lldx%lld%s src0=%s]", ggml_op_name(t->op), t->name, (long long)t->ne[0], (long long)t->ne[1], (long long)t->ne[2],
                    (t->flags & GGML_TENSOR_FLAG_COMPUTE) ? "" : " NOCOMPUTE", t->src[0] ? t->src[0]->name : "-");
        }
        fprintf(stderr, "\n");
    }
    return 0;
}
// ROPE(q) at node i, ROPE(k) at node ik (adjacent, or separated by mat-muls that have been recorded in between).  Returns the index of
// the first node NOT handled, or -1 (nothing done).
// dry: only answer whether the pair WOULD become an attention phase of the persistent kernel; must: it has to (ROPE(q) was postponed past
// mat-muls whose outputs reuse its source buffer, so the stand-alone kernels can no longer run it).
int fuse_rope_pair(backend_ctx * b, ggml_cgraph * g, int i, int ik, cudaError_t & err, bool dry = false, bool must = false) {
    err = cudaSuccess;
    ggml_tensor * rq = g->nodes[i];
    if (rq->op != GGML_OP_ROPE) return -1 + rope_decline(g, i, 1);
    if (ik >= g->n_nodes) return -1 + rope_decline(g, i, 2);
    ggml_tensor * rk = g->nodes[ik];
    if (rk->op != GGML_OP_ROPE || rk->src[1] != rq->src[1] || rk->src[2] != rq->src[2]) return -1 + rope_decline(g, i, 3);
    if (memcmp(rq->op_params, rk->op_params, sizeof(int32_t) * 16) != 0) return -1 + rope_decline(g, i, 4);
    const int isk = next_compute(g, ik + 1);
    if (isk >= g->n_nodes) return -1 + rope_decline(g, i, 5);
    const int isv = next_compute(g, isk + 1);
    if (isv >= g->n_nodes) return -1 + rope_decline(g, i, 6);
    ggml_tensor * sk = g->nodes[isk], * sv = g->nodes[isv];
    if (sk->op != GGML_OP_SET_ROWS || sv->op != GGML_OP_SET_ROWS) return -1 + rope_decline(g, i, 7);
    const ggml_tensor * q_in = rq->src[0], * k_in = rk->src[0];
    if (rq->type != GGML_TYPE_F32 || rk->type != GGML_TYPE_F32 || rq->ne[2] != 1 || rq->ne[3] != 1 || rk->ne[2] != 1 || rk->ne[3] != 1) return -1 + rope_decline(g, i, 8);
    if (!ggml_is_contiguous(rq) || !ggml_is_contiguous(rk) || !ggml_is_contiguous(q_in) || !ggml_is_contiguous(k_in) || rq->ne[0] != rk->ne[0]) return -1 + rope_decline(g, i, 9);
    const int32_t * p = (const int32_t *)rq->op_params;
    if ((p[2] != 0 && p[2] != 2) || p[15] != 0) return -1 + rope_decline(g, i, 10);
    // SET_ROWS(K): source must be exactly the roped K (a view of it), one row, f16 cache, i64 index
    const ggml_tensor * ks = sk->src[0], * vs = sv->src[0];
    if (ks->data != rk->data || ggml_nelements(ks) != ggml_nelements(rk) || !ggml_is_contiguous(ks) || ks->ne[1] != 1) return -1 + rope_decline(g, i, 11);
    if (vs->type != GGML_TYPE_F32 || !ggml_is_contiguous(vs) || vs->ne[1] != 1 || ggml_nelements(vs) != ggml_nelements(ks)) return -1 + rope_decline(g, i, 12);
    if (sk->type != GGML_TYPE_F16 || sv->type != GGML_TYPE_F16 || sk->src[1]->type != GGML_TYPE_I64 || sv->src[1]->type != GGML_TYPE_I64) return -1 + rope_decline(g, i, 13);
    if (ggml_nelements(sk->src[1]) != 1 || ggml_nelements(sv->src[1]) != 1 || sk->nb[0] != 2 || sv->nb[0] != 2) return -1 + rope_decline(g, i, 14);
    if (sk->ne[0] != ks->ne[0] || sv->ne[0] != vs->ne[0]) return -1 + rope_decline(g, i, 15);
    qmm::ops::RopeKVArgs a{};
    a.q_src = (const float *)q_in->data; a.q_dst = (float *)rq->data; a.n_head = (int)rq->ne[1];
    a.k_src = (const float *)k_in->data; a.k_dst = (float *)rk->data; a.n_head_kv = (int)rk->ne[1];
    a.v_src = (const float *)vs->data;
    a.k_cache = sk->data; a.k_row_bytes = (int64_t)sk->nb[1];
    a.v_cache = sv->data; a.v_row_bytes = (int64_t)sv->nb[1];
    a.k_idx = (const int64_t *)sk->src[1]->data; a.v_idx = (const int64_t *)sv->src[1]->data;
    a.pos = (const int32_t *)rq->src[1]->data; a.freq_factors = rq->src[2] ? (const float *)rq->src[2]->data : nullptr;
    a.head_dim = (int)rq->ne[0]; a.n_dims = p[1]; a.mode = p[2]; a.n_ctx_orig = p[4];
    memcpy(&a.freq_base, p + 5, 4); memcpy(&a.freq_scale, p + 6, 4); memcpy(&a.ext_factor, p + 7, 4);
    memcpy(&a.attn_factor, p + 8, 4); memcpy(&a.beta_fast, p + 9, 4); memcpy(&a.beta_slow, p + 10, 4);
    if ((int64_t)a.head_dim * a.n_head_kv != vs->ne[0]) return 0;
    if (b->mega && !b->mega_no_attn && b->d_mega_phases && b->fb.size() < MEGA_MAX_PHASES) {
        // persistent kernel: ROPE + cache store + the FLASH_ATTN_EXT that follows become one phase.  The ROPE nodes' own outputs are
        // not materialised (ggml-alloc makes them in-place on the mat-mul outputs, which other CTAs are still reading -- the round-1
        // race), so they must have no consumer outside the phase.
        const int ifa = next_compute(g, isv + 1);
        ggml_tensor * fa = ifa < g->n_nodes ? g->nodes[ifa] : nullptr;
        const bool q_only_here = ggml_node_get_use_count(g, i) == 1, k_only_here = ggml_node_get_use_count(g, ik) == 1;
        if (fa && fa->op == GGML_OP_FLASH_ATTN_EXT && supports_op(nullptr, fa) && q_only_here && k_only_here) {
            const ggml_tensor * fq = fa->src[0], * fk = fa->src[1], * fv = fa->src[2], * fm = fa->src[3];
            float scale, softcap;
            memcpy(&scale, fa->op_params, 4);
            memcpy(&softcap, (const float *)fa->op_params + 2, 4);
            const bool shapes = fq->data == rq->data && fq->ne[0] == a.head_dim && fq->ne[1] == 1 && fq->ne[2] == a.n_head && fq->ne[3] == 1 &&
                                fq->nb[2] == (size_t)a.head_dim * 4 &&
                                fk->data == sk->data && fv->data == sv->data && fk->nb[1] == sk->nb[1] && fv->nb[1] == sv->nb[1] &&
                                fk->ne[0] == a.head_dim && fv->ne[0] == a.head_dim && fk->ne[2] == a.n_head_kv && fv->ne[2] == a.n_head_kv &&
                                fk->ne[3] == 1 && fv->ne[3] == 1 && fk->ne[1] == fv->ne[1] &&
                                (!fm || (fm->ne[0] >= fk->ne[1] && fm->ne[2] == 1 && fm->ne[3] == 1)) &&
                                fa->nb[1] == (size_t)a.head_dim * 4 && ggml_is_contiguous(fa);
            if (shapes) {
                qmm::FlowAttn m;
                memset(&m, 0, sizeof(m));
                m.k_cache = a.k_cache; m.k_row_bytes = a.k_row_bytes; m.v_cache = a.v_cache; m.v_row_bytes = a.v_row_bytes;
                m.k_idx = a.k_idx; m.v_idx = a.v_idx; m.pos = a.pos; m.freq_factors = a.freq_factors;
                m.kview = fk->data; m.k_nb1 = (int64_t)fk->nb[1]; m.k_nb2 = (int64_t)fk->nb[2];
                m.vview = fv->data; m.v_nb1 = (int64_t)fv->nb[1]; m.v_nb2 = (int64_t)fv->nb[2];
                m.mask = fm ? fm->data : nullptr;
                m.n_head = a.n_head; m.n_head_kv = a.n_head_kv; m.head_dim = a.head_dim; m.n_dims = a.n_dims; m.rope_mode = a.mode; m.n_kv = (int)fk->ne[1];
                m.freq_scale = a.freq_scale; m.ext_factor = a.ext_factor; m.attn_factor = a.attn_factor;
                qmm::ops::rope_derived(a, m.theta_scale, m.corr0, m.corr1);
                m.softcap = softcap; m.scale = softcap != 0.0f ? scale / softcap : scale;
                if (dry) return b->fb.attn_ok(m) ? 1 : -1;
                const qmm::FlowVec * qv = must ? &b->deferred_q : nullptr;
                if (must && (b->deferred_q.ll == nullptr || b->deferred_seg != b->mega_flushed || b->fb.needs_cut(a.k_src) || b->fb.needs_cut(a.v_src))) {
                    GGML_LOG_ERROR("ggml-b200: a postponed ROPE(q) lost its tagged slots (a program cut between its mat-mul and the attention phase)\n");
                    err = cudaErrorUnknown; return -1;
                }
                if (!must && (b->fb.needs_cut(a.q_src) || b->fb.needs_cut(a.k_src) || b->fb.needs_cut(a.v_src))) { flush_why w("attention input is plain memory written by a pending phase"); err = mega_flush(b); if (err != cudaSuccess) return -1; }
                if (b->fb.add_attn(m, a.q_src, a.k_src, a.v_src, (float *)fa->data, qv)) return next_compute(g, ifa + 1);
            }
        }
    }
    if (dry) return -1;
    if (must) { GGML_LOG_ERROR("ggml-b200: a postponed ROPE(q) cannot join an attention phase\n"); err = cudaErrorUnknown; return -1; }
    if (b->mega) {
        flush_why w("ROPE/KV/attention group not accepted by the builder");
        err = mega_flush(b);
        if (err != cudaSuccess) return -1;
    }
    err = qmm::ops::rope_kv_store(a, b->stream);
    if (err == cudaErrorNotSupported) { err = cudaSuccess; return -1; }
    return next_compute(g, isv + 1);
}

inline bool regions_overlap(const ggml_tensor * a, const ggml_tensor * c) {
    const char * a0 = (const char *)a->data, * c0 = (const char *)c->data;
    return a0 != nullptr && c0 != nullptr && a0 < c0 + ggml_nbytes(c) && c0 < a0 + ggml_nbytes(a);
}

cudaError_t run_rope_node(backend_ctx * b, const ggml_tensor * node) {
    const int32_t * p = (const int32_t *)node->op_params;
    float fb, fs, ef, af, bf, bs;
    memcpy(&fb, p + 5, 4); memcpy(&fs, p + 6, 4); memcpy(&ef, p + 7, 4); memcpy(&af, p + 8, 4); memcpy(&bf, p + 9, 4); memcpy(&bs, p + 10, 4);
    return qmm::ops::rope(view_of(node->src[0]), (const int32_t *)node->src[1]->data, node->src[2] ? (const float *)node->src[2]->data : nullptr,
                          view_of(node), p[1], p[2], p[4], fb, fs, ef, af, bf, bs, b->stream);
}

// Pattern C at a ROPE node.  Returns the number of graph nodes handled starting at i (0 = no match: the caller runs the node itself).
int try_fuse_rope_kv(backend_ctx * b, ggml_cgraph * g, int i, cudaError_t & err) {
    err = cudaSuccess;
    if (b->deferred_rope >= 0) {                                   // this is the ROPE(k) a deferred ROPE(q) has been waiting for
        const int iq = b->deferred_rope;
        b->deferred_rope = -1;
        const int nxt = fuse_rope_pair(b, g, iq, i, err, false, true);
        if (err != cudaSuccess || nxt < 0) { if (err == cudaSuccess) err = cudaErrorUnknown; return 0; }
        return nxt - i;
    }
    const int ik = next_compute(g, i + 1);
    if (ik < g->n_nodes && g->nodes[ik]->op == GGML_OP_ROPE) {
        const int nxt = fuse_rope_pair(b, g, i, ik, err);
        return nxt >= 0 ? nxt - i : 0;
    }
    // the meta backend's order: ROPE(q), then the k / v mat-muls, then ROPE(k).  Only the persistent kernel can use that (q stays in
    // tagged slots); ROPE(q) is postponed, which is safe only if nothing recorded in between writes over what it reads or writes
    if (!(b->mega && !b->mega_no_attn && b->d_mega_phases)) return rope_decline(g, i, 16);
    // Leases W / Y / Z (-sm tensor on two GPUs; one GPU with GGML_B200_NO_GRAPH_OPTIMIZE=1): with the postponed ROPE(q) the attention phase produced
    // wrong logits (NMSE 0.4 - 0.6) and, on the 8B model, a trapped launch.  Cause: ROPE(q) is not in place in this node order, so ggml-alloc
    // hands the q mat-mul's buffer to the v / k mat-mul output, and the builder -- which names vectors by address -- then found THAT vector when
    // the attention phase asked for q.  The q vector is now remembered when the ROPE is postponed (deferred_q); lease Z3: bit-identical to the
    // default order on the small model, 397 tok/s on the 8B model in this order.  GGML_B200_NO_DEFER_ROPE=1 keeps ROPE / KV store / attention
    // as their own launches in this node order.
    static const bool defer_off = getenv("GGML_B200_NO_DEFER_ROPE") != nullptr;
    if (defer_off) return rope_decline(g, i, 20);
    ggml_tensor * rq = g->nodes[i];
    int j = ik;
    while (j < g->n_nodes && (is_noop(g->nodes[j]) || decode_mm_ok(g->nodes[j]))) {
        // (an output that reuses ROPE(q)'s SOURCE buffer is fine: the attention phase reads q from its tagged slots, not from memory)
        if (!is_noop(g->nodes[j]) && regions_overlap(g->nodes[j], rq)) return rope_decline(g, i, 17);
        j++;
    }
    if (j >= g->n_nodes || g->nodes[j]->op != GGML_OP_ROPE || g->nodes[j]->src[1] != rq->src[1] || g->nodes[j]->src[2] != rq->src[2]) return rope_decline(g, i, 18);
    { cudaError_t e2 = cudaSuccess; if (fuse_rope_pair(b, g, i, j, e2, true) < 0) return rope_decline(g, i, 19); }
    b->deferred_rope = i;
    b->deferred_q = b->fb.vec((const float *)rq->src[0]->data);
    b->deferred_seg = b->mega_flushed;
    return ik - i;                                                 // the ROPE(q) node (and the views behind it) are "done" for now
}


// Debug aid (GGML_B200_NODE_HASH=<file>): after every launch group, synchronise and append "graph# node# op name fnv1a(output)" --
// two runs of the same inputs must produce the same file; the first differing line names the op whose launch is not reproducible.
void debug_hash_nodes(backend_ctx * b, ggml_cgraph * g, int i0, int i1) {
    static FILE * f = [] { const char * p = getenv("GGML_B200_NODE_HASH"); return p ? fopen(p, "a") : nullptr; }();
    static const char * dump_dir = getenv("GGML_B200_NODE_DUMP");                 // + raw outputs of the graphs listed in ..._GRAPHS ("1,8")
    static const std::string dump_graphs = [] { const char * p = getenv("GGML_B200_NODE_DUMP_GRAPHS"); return std::string(",") + (p ? p : "") + ","; }();
    static int graph_no = -1;
    if (f == nullptr) return;
    if (i0 == 0) graph_no++;
    cudaStreamSynchronize(b->stream);
    std::vector<uint8_t> host;
    bool epilogue_fused = false;                                                   // a GLU / ADD in the group: its mat-mul outputs are not materialised
    for (int j = i0; j <= i1; j++) epilogue_fused = epilogue_fused || g->nodes[j]->op == GGML_OP_GLU || g->nodes[j]->op == GGML_OP_ADD;
    const bool dump = dump_dir != nullptr && dump_graphs.find("," + std::to_string(graph_no) + ",") != std::string::npos;
    for (int j = i0; j <= i1; j++) {
        const ggml_tensor * t = g->nodes[j];
        const bool want = j == i1 || t->op == GGML_OP_ROPE || (t->op == GGML_OP_MUL_MAT && !epilogue_fused);
        if (!want || is_noop(t) || t->data == nullptr || t->op == GGML_OP_SET_ROWS || !ggml_is_contiguous(t)) continue;
        host.resize(ggml_nbytes(t));
        if (cudaMemcpy(host.data(), t->data, host.size(), cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); continue; }
        uint64_t h = 1469598103934665603ull;
        for (uint8_t c : host) { h ^= c; h *= 1099511628211ull; }
        fprintf(f, "%d %d %s %s %016llx\n", graph_no, j, ggml_op_name(t->op), t->name, (unsigned long long)h);
        if (dump && t->op == GGML_OP_ROPE) {                                       // who else lives in this output's bytes?
            const char * lo = (const char *)t->data, * hi = lo + ggml_nbytes(t);
            fprintf(f, "# %d %d %s data %p..%p src0 %s %p\n", graph_no, j, t->name, (void *)lo, (void *)hi, t->src[0]->name, t->src[0]->data);
            for (int k = 0; k < g->n_nodes; k++) {
                const ggml_tensor * o = g->nodes[k];
                for (int si = -1; si < GGML_MAX_SRC; si++) {
                    const ggml_tensor * q = si < 0 ? o : o->src[si];
                    if (q == nullptr || q->data == nullptr || q == t) continue;
                    const char * ql = (const char *)q->data, * qh = ql + ggml_nbytes(q);
                    if (ql < hi && lo < qh) fprintf(f, "#    overlaps node %d %s%s %s (%s) %p..%p\n", k, si < 0 ? "" : "src of ", ggml_op_name(o->op), q->name, ggml_op_name(q->op), (void *)ql, (void *)qh);
                }
            }
        }
        if (dump) {
            const std::string path = std::string(dump_dir) + "/g" + std::to_string(graph_no) + "_n" + std::to_string(j) + ".bin";
            if (FILE * df = fopen(path.c_str(), "wb")) { fwrite(host.data(), 1, host.size(), df); fclose(df); }
        }
    }
    fflush(f);
}

cudaError_t enqueue_graph(backend_ctx * b, ggml_cgraph * g) {
    act_cache_t ac;
    cudaStream_t st = b->stream;
    b->deferred_rope = -1;
    b->norm_ctx.mul = nullptr; b->norm_ctx.remaining = 0;
    if (b->mega && !mega_alloc(b) && !b->d_mega_phases) b->mega = false;
    const bool deferred = b->tp != nullptr && b->mega;
    if (!(deferred && b->tp_open)) {                       // (tensor-parallel group: keep recording into the pending program)
        b->fb.reset(b->d_mega_ll, MEGA_LL_ELEMS, qmm::flow_grid(b->dev->cuda_dev));
        b->mega_flushed = 0;
    }
    if (b->counters) {                                      // one memset node per graph: every fused launch gets its own zeroed ticket
        cudaError_t e0 = cudaMemsetAsync(b->counters, 0, sizeof(unsigned) * N_COUNTERS, st);
        if (e0 != cudaSuccess) return e0;
        b->counter_next = 0;
    }
    for (int i = 0; i < g->n_nodes; i++) {
        ggml_tensor * node = g->nodes[i];
        if (is_noop(node)) continue;
        cudaError_t e = cudaSuccess;
        const int i_first = i;
        if (b->fuse_decode && (node->op == GGML_OP_RMS_NORM || node->op == GGML_OP_MUL_MAT || node->op == GGML_OP_ROPE)) {
            static const bool no_rope_f = getenv("GGML_B200_NO_ROPE_KV_FUSION") != nullptr, no_mv_f = getenv("GGML_B200_NO_MATVEC_FUSION") != nullptr;   // (bisection switches)
            const int used = node->op == GGML_OP_ROPE ? (no_rope_f ? 0 : try_fuse_rope_kv(b, g, i, e)) : (no_mv_f ? 0 : try_fuse_matvec(b, g, i, e));
            if (e != cudaSuccess) {
                GGML_LOG_ERROR("ggml-b200: fused %s (%s) failed: %s\n", ggml_op_name(node->op), node->name, cudaGetErrorString(e));
                return e;
            }
            if (used > 0) { i += used - 1; ac.src = nullptr; if (b->debug_hash) debug_hash_nodes(b, g, i_first, i); continue; }
        }
        if (b->mega) {
            // tiny one-row ops between mat-vec phases stay inside the persistent kernel (each is a phase of its own, run by one CTA)
            if (b->d_mega_phases && b->fb.size() > b->mega_flushed && b->fb.size() < MEGA_MAX_PHASES) {
                if (node->op == GGML_OP_GET_ROWS && node->src[0]->type == GGML_TYPE_F32 && node->src[1]->type == GGML_TYPE_I32 && ggml_nelements(node->src[1]) == 1 &&
                    node->type == GGML_TYPE_F32 && ggml_is_contiguous(node->src[0]) && ggml_is_contiguous(node) && node->src[0]->ne[1] == 1 && node->src[0]->ne[2] == 1 &&
                    node->src[0]->ne[3] == 1 && node->ne[0] < (1 << 16) && !b->fb.needs_cut(node->src[0]->data)) {
                    // one row out of a one-row matrix (llama's inp_out_ids on a one-token batch): the only valid index is 0
                    if (b->fb.add_copy((const float *)node->src[0]->data, (float *)node->data, (int)node->ne[0])) continue;
                }
                if (node->op == GGML_OP_ADD && node->type == GGML_TYPE_F32 && node->src[0]->type == GGML_TYPE_F32 && node->src[1]->type == GGML_TYPE_F32 &&
                    ggml_are_same_shape(node->src[0], node->src[1]) && ggml_is_contiguous(node) && ggml_is_contiguous(node->src[0]) && ggml_is_contiguous(node->src[1]) &&
                    ggml_nelements(node) == node->ne[0] && ggml_nelements(node) < (1 << 16) && !b->fb.needs_cut(node->src[0]->data) && !b->fb.needs_cut(node->src[1]->data)) {
                    if (b->fb.add_add((const float *)node->src[0]->data, (const float *)node->src[1]->data, (float *)node->data, (int)ggml_nelements(node))) continue;
                }
            }
            { flush_why w(ggml_op_name(node->op)); e = mega_flush(b); }   // anything else runs as its own launch, after what has been recorded
            if (e != cudaSuccess) { GGML_LOG_ERROR("ggml-b200: persistent decode kernel launch failed: %s\n", cudaGetErrorString(e)); return e; }
        }
        switch (node->op) {
            case GGML_OP_MUL_MAT: {
                if (b->norm_ctx.mul != nullptr && node->src[1] == b->norm_ctx.mul) {
                    // this consumer could not be recorded: write the normalised vector now (x is still live), everything after reads memory
                    const TensorView w = view_of(b->norm_ctx.w);
                    e = qmm::ops::rms_norm(view_of(b->norm_ctx.x), &w, view_of(b->norm_ctx.mul), b->norm_ctx.eps, st);
                    b->norm_ctx.mul = nullptr;
                    if (e != cudaSuccess) break;
                }
                // fusion: MUL_MAT (N <= 8) followed by ADD(mm, r) with the mat-mul output used only there -> residual in the epilogue
                const ggml_tensor * residual = nullptr;
                if (b->fuse && i + 1 < g->n_nodes && node->src[1]->ne[1] <= 8 && is_quant(node->src[0]->type)) {
                    ggml_tensor * nx = g->nodes[i + 1];
                    if (nx->op == GGML_OP_ADD && !is_noop(nx) && (nx->src[0] == node || nx->src[1] == node) && ggml_node_has_n_uses(g, i, 1)) {
                        const ggml_tensor * other = nx->src[0] == node ? nx->src[1] : nx->src[0];
                        if (other->type == GGML_TYPE_F32 && ggml_are_same_shape(other, node) && ggml_is_contiguous(other) && ggml_is_contiguous(nx)) {
                            // compute straight into the ADD's output
                            ggml_tensor tmp = *node;
                            tmp.data = nx->data;
                            e = run_mul_mat(b, &tmp, ac, other);
                            i++;                       // the ADD is done
                            break;
                        }
                    }
                }
                (void)residual;
                e = run_mul_mat_nd(b, node, ac, nullptr);
            } break;
            case GGML_OP_MUL_MAT_ID:
                e = run_mul_mat_id(b, node); ac.src = nullptr;
                break;
            case GGML_OP_RMS_NORM: {
                float eps;
                memcpy(&eps, node->op_params, sizeof(float));
                // fusion: RMS_NORM followed by MUL(norm, w) with the norm used only there (the CPU backend fuses the same pair, ops.cpp:3760-3768)
                if (b->fuse && i + 1 < g->n_nodes) {
                    ggml_tensor * nx = g->nodes[i + 1];
                    if (nx->op == GGML_OP_MUL && !is_noop(nx) && nx->src[0] == node && nx->src[1]->type == GGML_TYPE_F32 && rows_contiguous(nx->src[1]) &&
                        nx->src[1]->ne[0] == node->ne[0] && ggml_are_same_shape(nx, node) && rows_contiguous(nx) && ggml_node_has_n_uses(g, i, 1)) {
                        const TensorView w = view_of(nx->src[1]);
                        e = qmm::ops::rms_norm(view_of(node->src[0]), &w, view_of(nx), eps, st);
                        i++;
                        break;
                    }
                }
                e = qmm::ops::rms_norm(view_of(node->src[0]), nullptr, view_of(node), eps, st);
            } break;
            case GGML_OP_SOFT_MAX: {
                float sc;
                memcpy(&sc, node->op_params, sizeof(float));
                if (node->src[1]) { const TensorView m = view_of(node->src[1]); e = qmm::ops::soft_max(view_of(node->src[0]), &m, view_of(node), sc, st); }
                else e = qmm::ops::soft_max(view_of(node->src[0]), nullptr, view_of(node), sc, st);
            } break;
            case GGML_OP_ARGSORT: e = qmm::ops::argsort(view_of(node->src[0]), view_of(node), ((const int32_t *)node->op_params)[0] == GGML_SORT_ORDER_DESC, st); break;
            case GGML_OP_SUM_ROWS: e = qmm::ops::sum_rows(view_of(node->src[0]), view_of(node), st); break;
            case GGML_OP_CLAMP: {
                float lo, hi;
                memcpy(&lo, node->op_params, sizeof(float));
                memcpy(&hi, (const float *)node->op_params + 1, sizeof(float));
                e = qmm::ops::clamp(view_of(node->src[0]), view_of(node), lo, hi, st);
            } break;
            case GGML_OP_DIV: e = qmm::ops::binary(2, view_of(node->src[0]), view_of(node->src[1]), view_of(node), st); break;
            case GGML_OP_ADD: e = qmm::ops::binary(0, view_of(node->src[0]), view_of(node->src[1]), view_of(node), st); break;
            case GGML_OP_MUL: e = qmm::ops::binary(1, view_of(node->src[0]), view_of(node->src[1]), view_of(node), st); break;
            case GGML_OP_SCALE: {
                float s, bias;
                memcpy(&s, node->op_params, sizeof(float));
                memcpy(&bias, (const float *)node->op_params + 1, sizeof(float));
                e = qmm::ops::scale(view_of(node->src[0]), view_of(node), s, bias, st);
            } break;
            case GGML_OP_ROPE: {
                const int32_t * p = (const int32_t *)node->op_params;
                float fb, fs, ef, af, bf, bs;
                memcpy(&fb, p + 5, 4); memcpy(&fs, p + 6, 4); memcpy(&ef, p + 7, 4); memcpy(&af, p + 8, 4); memcpy(&bf, p + 9, 4); memcpy(&bs, p + 10, 4);
                e = qmm::ops::rope(view_of(node->src[0]), (const int32_t *)node->src[1]->data, node->src[2] ? (const float *)node->src[2]->data : nullptr,
                                   view_of(node), p[1], p[2], p[4], fb, fs, ef, af, bf, bs, st);
            } break;
            case GGML_OP_SET_ROWS: e = qmm::ops::set_rows(view_of(node->src[0]), view_of(node->src[1]), view_of(node), st); break;
            case GGML_OP_GET_ROWS: e = qmm::ops::get_rows(view_of(node->src[0]), view_of(node->src[1]), view_of(node), st); break;
            case GGML_OP_GLU: {
                const bool swapped = ((const int32_t *)node->op_params)[1] != 0;
                if (node->src[1]) { const TensorView bv = view_of(node->src[1]); e = qmm::ops::swiglu(view_of(node->src[0]), &bv, view_of(node), swapped, st); }
                else e = qmm::ops::swiglu(view_of(node->src[0]), nullptr, view_of(node), swapped, st);
            } break;
            case GGML_OP_CPY: e = qmm::ops::copy(view_of(node->src[0]), view_of(node->src[1]), st); break;
            case GGML_OP_CONT: case GGML_OP_DUP: e = qmm::ops::copy(view_of(node->src[0]), view_of(node), st); break;
            case GGML_OP_FLASH_ATTN_EXT: {
                float scale, softcap;
                memcpy(&scale, node->op_params, 4);
                memcpy(&softcap, (const float *)node->op_params + 2, 4);
                if (node->src[3]) { const TensorView m = view_of(node->src[3]); e = qmm::ops::flash_attn(view_of(node->src[0]), view_of(node->src[1]), view_of(node->src[2]), &m, view_of(node), scale, softcap, st, b->ws, b->ws_size); }
                else e = qmm::ops::flash_attn(view_of(node->src[0]), view_of(node->src[1]), view_of(node->src[2]), nullptr, view_of(node), scale, softcap, st, b->ws, b->ws_size);
            } break;
            default:
                GGML_LOG_ERROR("ggml-b200: op %s reached graph_compute but is not supported\n", ggml_op_name(node->op));
                return cudaErrorNotSupported;
        }
        if (e != cudaSuccess) {
            GGML_LOG_ERROR("ggml-b200: %s (%s) failed: %s\n", ggml_op_name(node->op), node->name, cudaGetErrorString(e));
            return e;
        }
        // anything that may write the activation a later mat-mul would re-use invalidates the quantised copy
        if (node->op != GGML_OP_MUL_MAT) ac.src = nullptr;
        if (b->debug_hash) debug_hash_nodes(b, g, i_first, i);
    }
    if (deferred) {
        b->tp_open = b->fb.size() > b->mega_flushed;       // launched later, together with the peers' programs (mega_flush)
    } else if (b->mega) {
        const cudaError_t e = mega_flush(b);
        if (e != cudaSuccess) { GGML_LOG_ERROR("ggml-b200: persistent decode kernel launch failed: %s\n", cudaGetErrorString(e)); return e; }
    }
    return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------- backend (stream)
inline void tp_sync_point(backend_ctx * b) { if (b->tp != nullptr && b->tp_open) { flush_why w("host sync point (tensor get/set/copy, synchronize, event)"); mega_flush(b); } }

void graph_entry_release(graph_entry & e) {
    if (e.exec) cudaGraphExecDestroy(e.exec);
    if (e.d_prog) cudaFree(e.d_prog);
    e.exec = nullptr; e.d_prog = nullptr; e.prog_cap = 0;
}
void graph_cache_clear(backend_ctx * b) {
    for (auto & kv : b->gcache) graph_entry_release(kv.second);
    b->gcache.clear();
    b->last_entry = nullptr;
    if (g_last_graph_backend == b) g_last_graph_backend = nullptr;
}

const char * backend_name(ggml_backend_t backend) { return ((backend_ctx *)backend->context)->name.c_str(); }

void backend_free(ggml_backend_t backend) {
    auto * b = (backend_ctx *)backend->context;
    flush_stats_dump();
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    if (b->tp != nullptr) { for (auto & m : b->tp->members) if (m == b) m = nullptr; b->tp->members.erase(std::remove(b->tp->members.begin(), b->tp->members.end(), nullptr), b->tp->members.end()); b->tp = nullptr; }
    cudaStreamSynchronize(b->stream);
    if (b->d_mega_trace && !b->mega_mirror.empty()) {       // timeline of the last eager token: [n][kind, K, sum M, type] then [n][FLOW_TRACE_N][160], see FlowProgram::trace
        const char * path = getenv("GGML_B200_MEGA_TRACE");
        const int grid = qmm::flow_grid(b->dev->cuda_dev);
        const int n = (int)b->mega_mirror.size();
        std::vector<unsigned long long> raw((size_t)n * qmm::FLOW_TRACE_N * 160);
        if (path && cudaMemcpy(raw.data(), b->d_mega_trace, raw.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost) == cudaSuccess) {
            if (FILE * f = fopen(path, "wb")) {
                fwrite(&n, 4, 1, f); fwrite(&grid, 4, 1, f);
                for (int i = 0; i < n; i++) {
                    const qmm::FlowPhase & ph = b->mega_mirror[i];
                    int rec[4] = {ph.kind, 0, 0, 0};
                    if (ph.kind == qmm::FLOW_MATVEC) { rec[1] = ph.mv.K; rec[2] = ph.mv.M[0] + (ph.mv.nmat > 1 ? ph.mv.M[1] : 0) + (ph.mv.nmat > 2 ? ph.mv.M[2] : 0); rec[3] = ph.mv.type[0] + 100 * ph.mv.type[ph.mv.nmat - 1]; }
                    if (ph.kind == qmm::FLOW_ATTN) { rec[1] = ph.at.n_kv; rec[2] = ph.at.n_head; rec[3] = ph.at.nsplit; }
                    fwrite(rec, 4, 4, f);
                }
                fwrite(raw.data(), sizeof(unsigned long long), raw.size(), f);
                fclose(f);
            }
        }
    }
    graph_cache_clear(b);
    if (b->d_mega_phases) cudaFree(b->d_mega_phases);
    if (b->d_mega_sync) cudaFree(b->d_mega_sync);
    if (b->d_mega_ll) cudaFree(b->d_mega_ll);
    if (b->d_mega_trace) cudaFree(b->d_mega_trace);
    if (b->ws) cudaFree(b->ws);
    if (b->counters) cudaFree(b->counters);
    cudaStreamDestroy(b->stream);
    delete b;
    delete backend;
}
void backend_set_tensor_async(ggml_backend_t backend, ggml_tensor * tensor, const void * data, size_t offset, size_t size) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    B200_CHECK(cudaMemcpyAsync((char *)tensor->data + offset, data, size, cudaMemcpyHostToDevice, b->stream));
    g_h2d_bytes += size;
    journal_write((char *)tensor->data + offset, size);
}
void backend_get_tensor_async(ggml_backend_t backend, const ggml_tensor * tensor, void * data, size_t offset, size_t size) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    B200_CHECK(cudaMemcpyAsync(data, (const char *)tensor->data + offset, size, cudaMemcpyDeviceToHost, b->stream));
    g_d2h_bytes += size;
    if (size >= 4096) { g_last_read_src = (const char *)tensor->data + offset; g_last_read_size = size; g_last_read_dev = b->dev->cuda_dev; }
}
void backend_set_tensor_2d_async(ggml_backend_t backend, ggml_tensor * tensor, const void * data, size_t offset, size_t size, size_t n_copies,
                                 size_t stride_tensor, size_t stride_data) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    B200_CHECK(cudaMemcpy2DAsync((char *)tensor->data + offset, stride_tensor, data, stride_data, size, n_copies, cudaMemcpyHostToDevice, b->stream));
}
void backend_get_tensor_2d_async(ggml_backend_t backend, const ggml_tensor * tensor, void * data, size_t offset, size_t size, size_t n_copies,
                                 size_t stride_tensor, size_t stride_data) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    B200_CHECK(cudaMemcpy2DAsync(data, stride_data, (const char *)tensor->data + offset, stride_tensor, size, n_copies, cudaMemcpyDeviceToHost, b->stream));
}
bool backend_is_ours(ggml_backend_t be);
bool backend_cpy_tensor_async(ggml_backend_t backend_src, ggml_backend_t backend_dst, const ggml_tensor * src, ggml_tensor * dst) {
    if (!backend_is_ours(backend_src) || !backend_is_ours(backend_dst)) return false;
    ggml_backend_buffer_t sb = src->view_src ? src->view_src->buffer : src->buffer;
    ggml_backend_buffer_t db = dst->view_src ? dst->view_src->buffer : dst->buffer;
    if (!sb || !db || !buffer_is_ours(sb) || !buffer_is_ours(db)) return false;
    auto * bs = (backend_ctx *)backend_src->context;
    auto * bd = (backend_ctx *)backend_dst->context;
    tp_sync_point(bs);
    tp_sync_point(bd);
    if (bs == bd) {
        set_device(bd->dev->cuda_dev);
        B200_CHECK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, bd->stream));
        return true;
    }
    if (bs->dev == bd->dev) {                 // two streams of the same GPU
        set_device(bs->dev->cuda_dev);
        cudaEvent_t ev0;
        B200_CHECK(cudaMemcpyAsync(dst->data, src->data, ggml_nbytes(dst), cudaMemcpyDeviceToDevice, bs->stream));
        B200_CHECK(cudaEventCreateWithFlags(&ev0, cudaEventDisableTiming));
        B200_CHECK(cudaEventRecord(ev0, bs->stream));
        B200_CHECK(cudaStreamWaitEvent(bd->stream, ev0, 0));
        B200_CHECK(cudaEventDestroy(ev0));
        return true;
    }
    // The copy runs on the PRODUCER's stream (so later writes to src on that stream cannot overtake it) and the consumer's
    // stream waits for it -- the ordering the scheduler and the meta backend's butterfly fallback rely on
    // (same contract as ggml-cuda.cu's cpy_tensor_async).  NVLink peer copy through UVA.
    cudaEvent_t ev;
    set_device(bs->dev->cuda_dev);
    B200_CHECK(cudaMemcpyPeerAsync(dst->data, bd->dev->cuda_dev, src->data, bs->dev->cuda_dev, ggml_nbytes(dst), bs->stream));
    B200_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    B200_CHECK(cudaEventRecord(ev, bs->stream));
    set_device(bd->dev->cuda_dev);
    B200_CHECK(cudaStreamWaitEvent(bd->stream, ev, 0));
    B200_CHECK(cudaEventDestroy(ev));
    return true;
}
void backend_synchronize(ggml_backend_t backend) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    B200_CHECK(cudaStreamSynchronize(b->stream));
}

ggml_status backend_graph_compute(ggml_backend_t backend, ggml_cgraph * g) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    // workspace: sized before anything is enqueued (no allocation during capture)
    size_t need = 0;
    for (int i = 0; i < g->n_nodes; i++) {
        if (is_noop(g->nodes[i])) continue;
        const size_t n = node_workspace(g->nodes[i]);
        if (n > need) need = n;
    }
    if (need > b->ws_size) {
        B200_CHECK(cudaStreamSynchronize(b->stream));
        if (b->ws) B200_CHECK(cudaFree(b->ws));
        need = (need + (size_t(1) << 20)) & ~((size_t(1) << 20) - 1);
        B200_CHECK(cudaMalloc(&b->ws, need));
        b->ws_size = need;
        graph_cache_clear(b);                              // captured graphs bake in the old workspace pointer
    }

    // CUDA graph replay keyed on cgraph->uid (ggml-impl.h:344-346): the scheduler gives a split a new uid whenever it
    // is re-planned, so an unchanged uid means unchanged topology AND tensor addresses.
    if (b->use_graphs && g->uid != 0 && g->n_nodes >= 8 && !(b->tp != nullptr && b->mega)) {
        auto it = b->gcache.find(g->uid);
        if (it == b->gcache.end()) {
            if (b->gcache.size() >= GRAPH_CACHE_MAX) {         // evict the least recently used entry
                auto victim = b->gcache.begin();
                for (auto jt = b->gcache.begin(); jt != b->gcache.end(); ++jt) if (jt->second.last_use < victim->second.last_use) victim = jt;
                if (b->last_entry == &victim->second) b->last_entry = nullptr;
                B200_CHECK(cudaStreamSynchronize(b->stream));
                graph_entry_release(victim->second);
                b->gcache.erase(victim);
            }
            it = b->gcache.emplace(g->uid, graph_entry{}).first;
        }
        graph_entry & ge = it->second;
        ge.last_use = ++b->gc_tick;
        if (ge.exec && ge.n_nodes == g->n_nodes) {
            if (g_journal_on) {                            // snapshot this launch's inputs on the device (bench hook only)
                std::lock_guard<std::mutex> lk(g_journal_mu);
                size_t need = 0;
                for (auto & r : g_journal) { r.snap_off = need; need += (r.size + 255) & ~size_t(255); }
                if (need > g_snap_cap) { if (g_snap_buf) cudaFree(g_snap_buf); B200_CHECK(cudaMalloc(&g_snap_buf, need + 4096)); g_snap_cap = need + 4096; }
                for (auto & r : g_journal) B200_CHECK(cudaMemcpyAsync((char *)g_snap_buf + r.snap_off, r.dst, r.size, cudaMemcpyDeviceToDevice, b->stream));
                g_snap_inputs = g_journal;
                g_journal.clear();
            }
            B200_CHECK(cudaGraphLaunch(ge.exec, b->stream));
            g_graph_launches += ge.n_launches;
            g_last_graph_backend = b;
            b->last_entry = &ge;
            return GGML_STATUS_SUCCESS;
        }
        ge.seen++;
        if (ge.seen >= 2 && !ge.no_capture) {              // second sighting: capture once, replay from now on
            if (ge.exec) { cudaGraphExecDestroy(ge.exec); ge.exec = nullptr; }
            // the entry's own program buffer, sized from what the eager run of this uid recorded (allocated before the capture starts)
            const size_t want = ge.prog_eager + 8;
            if (b->mega && ge.prog_cap < want) {
                if (ge.d_prog) { B200_CHECK(cudaStreamSynchronize(b->stream)); cudaFree(ge.d_prog); ge.d_prog = nullptr; ge.prog_cap = 0; }
                if (cudaMalloc(&ge.d_prog, want * sizeof(qmm::FlowPhase)) == cudaSuccess) ge.prog_cap = want; else cudaGetLastError();
            }
            if (b->mega) mega_alloc(b);                    // sync words / scratch exist before the capture starts
            cudaGraph_t graph = nullptr;
            B200_CHECK(cudaStreamBeginCapture(b->stream, cudaStreamCaptureModeRelaxed));
            b->prog_deferred = true; b->prog_target = ge.d_prog; b->prog_cap_cur = ge.prog_cap;
            const uint64_t l0 = b200_qmm_launch_count();
            const cudaError_t e = enqueue_graph(b, g);
            b->prog_deferred = false;
            ge.n_launches = b200_qmm_launch_count() - l0;
            const cudaError_t e2 = cudaStreamEndCapture(b->stream, &graph);
            if (e == cudaSuccess && e2 == cudaSuccess && graph) {
                if (cudaGraphInstantiate(&ge.exec, graph, 0) == cudaSuccess) {
                    ge.n_nodes = g->n_nodes;
                    cudaGraphDestroy(graph);
                    if (b->fb.size() > 0)                  // the program the captured launches read (stream-ordered before the first replay)
                        B200_CHECK(cudaMemcpyAsync(ge.d_prog, b->fb.phases().data(), b->fb.size() * sizeof(qmm::FlowPhase), cudaMemcpyHostToDevice, b->stream));
                    B200_CHECK(cudaGraphLaunch(ge.exec, b->stream));
                    g_last_graph_backend = b;
                    b->last_entry = &ge;
                    return GGML_STATUS_SUCCESS;
                }
            }
            if (graph) cudaGraphDestroy(graph);
            cudaGetLastError();
            ge.exec = nullptr;
            ge.no_capture = true;                          // capture failed for this graph: it stays eager (still correct)
            GGML_LOG_WARN("ggml-b200: CUDA graph capture failed for one graph, it stays eager\n");
        }
        const bool ok = enqueue_graph(b, g) == cudaSuccess;
        ge.prog_eager = b->fb.size();
        return ok ? GGML_STATUS_SUCCESS : GGML_STATUS_FAILED;
    }
    return enqueue_graph(b, g) == cudaSuccess ? GGML_STATUS_SUCCESS : GGML_STATUS_FAILED;
}


// graph_optimize (called by the scheduler BEFORE buffers are planned, ggml-backend.cpp:1468-1470): make mat-muls that
// share an activation adjacent (attn_q, attn_v, attn_k all read attn_norm but llama.cpp interleaves ROPE / RESHAPE nodes),
// so that graph_compute can hand them to one fused launch.  A mat-mul only depends on its weight (a leaf) and the
// shared activation, so moving it up to sit right behind its first sibling never violates a dependency.
void backend_graph_optimize(ggml_backend_t backend, ggml_cgraph * g) {
    auto * b = (backend_ctx *)backend->context;
    if (!b->fuse_decode) return;
    // GGML_B200_NO_GRAPH_OPTIMIZE=1: keep llama.cpp's own node order -- the order the meta backend hands to its sub-backends under
    // -sm tensor (it does not call graph_optimize) -- so that the code paths of that order can be exercised on ONE GPU
    static const bool no_opt = getenv("GGML_B200_NO_GRAPH_OPTIMIZE") != nullptr;
    if (no_opt) return;
    for (int i = 0; i < g->n_nodes; i++) {
        ggml_tensor * a = g->nodes[i];
        if (a->op != GGML_OP_MUL_MAT) continue;
        int insert = i + 1;
        for (int j = i + 1; j < g->n_nodes && j < i + 24; j++) {
            ggml_tensor * c = g->nodes[j];
            if (c->op != GGML_OP_MUL_MAT || c->src[1] != a->src[1]) continue;
            bool weight_is_leaf = true;                       // src0 must not be produced inside (i, j)
            for (int k = i + 1; k < j; k++) if (g->nodes[k] == c->src[0] || (c->src[0]->view_src && g->nodes[k] == c->src[0]->view_src)) weight_is_leaf = false;
            if (!weight_is_leaf) continue;
            if (j != insert) {
                for (int k = j; k > insert; k--) g->nodes[k] = g->nodes[k - 1];
                g->nodes[insert] = c;
            }
            insert++;
        }
        i = insert - 1;
    }
}

void backend_event_record(ggml_backend_t backend, ggml_backend_event_t event) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    tp_sync_point(b);
    B200_CHECK(cudaEventRecord((cudaEvent_t)event->context, b->stream));
}
void backend_event_wait(ggml_backend_t backend, ggml_backend_event_t event) {
    auto * b = (backend_ctx *)backend->context;
    set_device(b->dev->cuda_dev);
    B200_CHECK(cudaStreamWaitEvent(b->stream, (cudaEvent_t)event->context, 0));
}

const ggml_backend_i k_backend_iface = {
    /* .get_name            = */ backend_name,
    /* .free                = */ backend_free,
    /* .set_tensor_async    = */ backend_set_tensor_async,
    /* .get_tensor_async    = */ backend_get_tensor_async,
    /* .set_tensor_2d_async = */ backend_set_tensor_2d_async,
    /* .get_tensor_2d_async = */ backend_get_tensor_2d_async,
    /* .cpy_tensor_async    = */ backend_cpy_tensor_async,
    /* .synchronize         = */ backend_synchronize,
    /* .graph_plan_create   = */ nullptr,
    /* .graph_plan_free     = */ nullptr,
    /* .graph_plan_update   = */ nullptr,
    /* .graph_plan_compute  = */ nullptr,
    /* .graph_compute       = */ backend_graph_compute,
    /* .event_record        = */ backend_event_record,
    /* .event_wait          = */ backend_event_wait,
    /* .graph_optimize      = */ backend_graph_optimize,
};
bool backend_is_ours(ggml_backend_t be) { return be && be->iface.get_name == backend_name; }

ggml_guid_t backend_guid() {
    static ggml_guid guid = {0xb2, 0x00, 0x5a, 0x10, 0x0a, 0x71, 0x4c, 0x9e, 0x8f, 0x21, 0x67, 0x67, 0x6d, 0x6c, 0xb2, 0x00};
    return &guid;
}

// ---------------------------------------------------------------------------------------------- device
const char * dev_name(ggml_backend_dev_t dev) { return ((device_ctx *)dev->context)->name.c_str(); }
const char * dev_desc(ggml_backend_dev_t dev) { return ((device_ctx *)dev->context)->desc.c_str(); }
void dev_memory(ggml_backend_dev_t dev, size_t * free, size_t * total) {
    set_device(((device_ctx *)dev->context)->cuda_dev);
    B200_CHECK(cudaMemGetInfo(free, total));
}
enum ggml_backend_dev_type dev_type(ggml_backend_dev_t) { return GGML_BACKEND_DEVICE_TYPE_GPU; }
void dev_props(ggml_backend_dev_t dev, ggml_backend_dev_props * props) {
    auto * d = (device_ctx *)dev->context;
    props->name = d->name.c_str();
    props->description = d->desc.c_str();
    props->type = GGML_BACKEND_DEVICE_TYPE_GPU;
    props->device_id = d->pci.empty() ? nullptr : d->pci.c_str();
    dev_memory(dev, &props->memory_free, &props->memory_total);
    props->caps = {/* async */ true, /* host_buffer */ true, /* buffer_from_host_ptr */ false, /* events */ true};
}
ggml_backend_t dev_init_backend(ggml_backend_dev_t dev, const char *) {
    auto * d = (device_ctx *)dev->context;
    set_device(d->cuda_dev);
    auto * b = new backend_ctx();
    b->dev = d;
    b->name = d->name;
    if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) { delete b; return nullptr; }
    if (getenv("GGML_B200_DYNAMIC_SPLIT") != nullptr && cudaMalloc(&b->counters, sizeof(unsigned) * N_COUNTERS) != cudaSuccess) { cudaGetLastError(); b->counters = nullptr; }
    b->debug_hash = getenv("GGML_B200_NODE_HASH") != nullptr;
    b->use_graphs = getenv("GGML_B200_NO_GRAPHS") == nullptr && !b->debug_hash;
    b->fuse = getenv("GGML_B200_NO_FUSION") == nullptr;
    b->fuse_decode = b->fuse && getenv("GGML_B200_NO_DECODE_FUSION") == nullptr;
    // Programmatic dependent launch is OPT-IN (GGML_B200_PDL=1): it buys ~5-8 % on decode, but run-to-run bit-identity of the
    // logits is not yet established with it on every model shape (see DESIGN.md "PDL"), so the default keeps plain launches.
    b->mega_no_attn = getenv("GGML_B200_MEGA_NO_ATTN") != nullptr;
    { const char * me = getenv("GGML_B200_MEGA"); b->mega = b->fuse_decode && !(me != nullptr && me[0] == '0'); }   // persistent decode kernel: on unless GGML_B200_MEGA=0
    b->pdl = getenv("GGML_B200_PDL") != nullptr && getenv("GGML_B200_NO_PDL") == nullptr;
    qmm::set_pdl(b->pdl);
    // Q8_0 activations (Q4_0 / Q8_0 weights): reproduce the from_float the x86 CPU backend really runs (AVX2: id = 127/amax,
    // round-half-even, arch/x86/quants.c:302-345) rather than quantize_row_q8_0_ref; they differ on (near-)ties only
    qmm::set_q8_0_mode(getenv("GGML_B200_Q8_0_REF") ? 0 : 1);
    return new ggml_backend{backend_guid(), k_backend_iface, dev, b};
}
ggml_backend_buffer_type_t dev_buffer_type(ggml_backend_dev_t dev) { return &((device_ctx *)dev->context)->buft; }

// Pinned host memory for what the host reads and writes every step (llama.cpp puts the logits / embeddings output buffer and the
// graph inputs there when the device offers it): the 513 KB logits copy of a decode step then runs at PCIe speed instead of through a
// pageable staging copy.  Same construction as the reference (ggml-cuda.cu:1262-1320): a CPU buffer around cudaMallocHost memory.
const char * host_buft_name(ggml_backend_buffer_type_t) { return "B200_Host"; }
void host_buf_free(ggml_backend_buffer_t buffer) { cudaFreeHost(buffer->context); }
ggml_backend_buffer_t host_buft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    void * ptr = nullptr;
    if (getenv("GGML_B200_NO_PINNED") != nullptr || cudaMallocHost(&ptr, size) != cudaSuccess) {
        cudaGetLastError();
        return ggml_backend_buft_alloc_buffer(ggml_backend_cpu_buffer_type(), size);      // pageable, still correct
    }
    ggml_backend_buffer_t buffer = ggml_backend_cpu_buffer_from_ptr(ptr, size);
    buffer->buft = buft;
    buffer->iface.free_buffer = host_buf_free;
    return buffer;
}
ggml_backend_buffer_type_t dev_host_buffer_type(ggml_backend_dev_t dev) {
    static ggml_backend_buffer_type host_buft = {
        /* .iface   = */ {host_buft_name, host_buft_alloc, ggml_backend_cpu_buffer_type()->iface.get_alignment, nullptr,
                          ggml_backend_cpu_buffer_type()->iface.get_alloc_size, ggml_backend_cpu_buffer_type()->iface.is_host},
        /* .device  = */ nullptr,
        /* .context = */ nullptr,
    };
    if (host_buft.device == nullptr) host_buft.device = &g_dev_objs[0];
    (void)dev;
    return &host_buft;
}
// Weights that stayed in host memory (partial offload): worth copying over for a big batch only (ggml-cuda.cu:5321-5340).
bool dev_offload_op(ggml_backend_dev_t, const ggml_tensor * op) {
    int64_t batch;
    switch (op->op) {
        case GGML_OP_GET_ROWS: batch = 0; break;
        case GGML_OP_MUL_MAT: batch = op->ne[1]; break;
        case GGML_OP_MUL_MAT_ID: case GGML_OP_ROPE: batch = op->ne[2]; break;
        default: batch = ggml_nrows(op); break;
    }
    return batch >= 32;
}
bool dev_supports_buft(ggml_backend_dev_t dev, ggml_backend_buffer_type_t buft) {
    return buft_is_ours(buft) && buft->context == dev->context;
}
ggml_backend_event_t dev_event_new(ggml_backend_dev_t dev) {
    set_device(((device_ctx *)dev->context)->cuda_dev);
    cudaEvent_t ev;
    B200_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    return new ggml_backend_event{dev, ev};
}
void dev_event_free(ggml_backend_dev_t, ggml_backend_event_t event) {
    cudaEventDestroy((cudaEvent_t)event->context);
    delete event;
}
void dev_event_synchronize(ggml_backend_dev_t, ggml_backend_event_t event) { B200_CHECK(cudaEventSynchronize((cudaEvent_t)event->context)); }

const ggml_backend_device_i k_device_iface = {
    /* .get_name             = */ dev_name,
    /* .get_description      = */ dev_desc,
    /* .get_memory           = */ dev_memory,
    /* .get_type             = */ dev_type,
    /* .get_props            = */ dev_props,
    /* .init_backend         = */ dev_init_backend,
    /* .get_buffer_type      = */ dev_buffer_type,
    /* .get_host_buffer_type = */ dev_host_buffer_type,
    /* .buffer_from_host_ptr = */ nullptr,
    /* .supports_op          = */ supports_op,
    /* .supports_buft        = */ dev_supports_buft,
    /* .offload_op           = */ dev_offload_op,
    /* .event_new            = */ dev_event_new,
    /* .event_free           = */ dev_event_free,
    /* .event_synchronize    = */ dev_event_synchronize,
};

// ---------------------------------------------------------------------------------------------- reg
const char * reg_name(ggml_backend_reg_t) { return "B200"; }
size_t reg_dev_count(ggml_backend_reg_t) { return g_devices.size(); }
ggml_backend_dev_t reg_get_device(ggml_backend_reg_t, size_t i) { return i < g_dev_objs.size() ? &g_dev_objs[i] : nullptr; }

ggml_backend_feature * reg_features(ggml_backend_reg_t) {
    static ggml_backend_feature f[] = {{"ARCH", "sm_90a"}, {"WGMMA", "1"}, {"CPU_FALLBACK", "0"}, {nullptr, nullptr}};
    return f;
}

void * reg_proc_address(ggml_backend_reg_t, const char * name) {
    if (!strcmp(name, "ggml_backend_comm_init")) return (void *)b200_comm_init;
    if (!strcmp(name, "ggml_backend_comm_free")) return (void *)b200_comm_free;
    if (!strcmp(name, "ggml_backend_comm_allreduce_tensor")) return (void *)b200_comm_allreduce_tensor;
    if (!strcmp(name, "ggml_backend_get_features")) return (void *)reg_features;
    return nullptr;   // split buffer type (-sm row, legacy), set_n_threads, extra bufts: not provided
}

const ggml_backend_reg_i k_reg_iface = {reg_name, reg_dev_count, reg_get_device, reg_proc_address};

void init_registry() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    for (int i = 0; i < n && (int)g_devices.size() < MAX_DEVICES; i++) {
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, i) != cudaSuccess) { cudaGetLastError(); continue; }
        if (p.major != 9) continue;                        // sm_90a code only: no other architecture, no fallback
        auto * d = new device_ctx();
        d->index = (int)g_devices.size();
        d->cuda_dev = i;
        d->name = "B200" + std::to_string(d->index);
        d->desc = p.name;
        char pci[32];
        snprintf(pci, sizeof(pci), "%04x:%02x:%02x.0", p.pciDomainID, p.pciBusID, p.pciDeviceID);
        d->pci = pci;
        d->buft_name = d->name;
        g_devices.push_back(d);
    }
    g_reg = ggml_backend_reg{GGML_BACKEND_API_VERSION, k_reg_iface, nullptr};
    g_dev_objs.resize(g_devices.size());
    for (size_t i = 0; i < g_devices.size(); i++) {
        g_dev_objs[i] = ggml_backend_device{k_device_iface, &g_reg, g_devices[i]};
        g_devices[i]->buft = ggml_backend_buffer_type{k_buft_iface, &g_dev_objs[i], g_devices[i]};
    }
}

}  // namespace

// ---- tensor-parallel group API used by comm.cpp
bool b200_tp_join(ggml_backend_t * backends, int n) {
    // The all-reduce fused into the decode kernel is opt-in (GGML_B200_TP_FUSION=1) at the end of round 2: on two GPUs (lease W2) it is correct
    // when ROPE / attention run as their own launches (GGML_B200_NO_DEFER_ROPE=1: 206 tok/s, most collectives "not fusable") but a launch traps
    // when the whole token is one program per GPU; the host-driven path below it (one-shot NVLink all-reduce between per-GPU programs) is
    // correct and faster today (271 tok/s).
    if (n < 2 || n > qmm::FLOW_MAX_PEERS || getenv("GGML_B200_NO_TP_FUSION") || !getenv("GGML_B200_TP_FUSION")) return false;
    auto * g = new tp_group();
    g->xhalf = (size_t)2 << 20;                                   // 2 M slots per half = 32 MB per GPU in total
    for (int i = 0; i < n; i++) {
        if (!backend_is_ours(backends[i])) { delete g; return false; }
        auto * b = (backend_ctx *)backends[i]->context;
        if (!b->mega || b->tp != nullptr) { delete g; return false; }
        g->members.push_back(b);
    }
    for (int i = 0; i < n; i++) {
        set_device(g->members[i]->dev->cuda_dev);
        if (cudaMalloc(&g->xpool[i], 2 * g->xhalf * sizeof(uint64_t)) != cudaSuccess || cudaMemset(g->xpool[i], 0, 2 * g->xhalf * sizeof(uint64_t)) != cudaSuccess) {
            cudaGetLastError();
            for (int j = 0; j <= i; j++) if (g->xpool[j]) { set_device(g->members[j]->dev->cuda_dev); cudaFree(g->xpool[j]); }
            delete g;
            return false;
        }
        cudaDeviceSynchronize();
    }
    for (backend_ctx * b : g->members) b->tp = g;
    g_tp_groups.push_back(g);
    return true;
}
void b200_tp_leave(ggml_backend_t * backends, int n) {
    if (n <= 0 || !backend_is_ours(backends[0])) return;
    tp_group * g = ((backend_ctx *)backends[0]->context)->tp;
    if (g == nullptr) return;
    if (!g->members.empty()) mega_flush(g->members[0]);
    for (size_t i = 0; i < g->members.size(); i++) {
        set_device(g->members[i]->dev->cuda_dev);
        cudaStreamSynchronize(g->members[i]->stream);
        g->members[i]->tp = nullptr;
    }
    for (int i = 0; i < qmm::FLOW_MAX_PEERS; i++) if (g->xpool[i]) cudaFree(g->xpool[i]);     // (UVA: any current device may free it)
    g_tp_groups.erase(std::remove(g_tp_groups.begin(), g_tp_groups.end(), g), g_tp_groups.end());
    delete g;
}
// Record the all-reduce of tensors[i] (one per backend of the group, in group order) into the pending programs.  false: nothing was
// recorded (the caller runs the stand-alone all-reduce; everything pending has been launched first).
bool b200_tp_fused_allreduce(ggml_backend_t * backends, int n, struct ggml_tensor ** tensors) {
    if (n < 2 || !backend_is_ours(backends[0])) return false;
    tp_group * g = ((backend_ctx *)backends[0]->context)->tp;
    if (g == nullptr || (int)g->members.size() != n) return false;
    qmm::FlowBuilder * fbs[qmm::FLOW_MAX_PEERS];
    float * ptrs[qmm::FLOW_MAX_PEERS];
    uint64_t * pools[qmm::FLOW_MAX_PEERS];
    bool ok = true;
    const int64_t ne = ggml_nelements(tensors[0]);
    for (int i = 0; i < n; i++) {
        auto * b = (backend_ctx *)backends[i]->context;
        if (b != g->members[i] || !b->tp_open || tensors[i]->type != GGML_TYPE_F32 || !ggml_is_contiguous(tensors[i]) || ggml_nelements(tensors[i]) != ne ||
            (tensors[i]->flags & GGML_TENSOR_FLAG_COMPUTE) == 0) {
            static int said = 0;
            if (getenv("GGML_B200_FLOW_DEBUG") && said++ < 8)
                fprintf(stderr, "ggml-b200: all-reduce of %s not fused on GPU %d: member %d open %d type %d contiguous %d ne %lld/%lld compute %d pending %zu flushed %zu\n", tensors[i]->name, i,
                        (int)(b == g->members[i]), (int)b->tp_open, (int)tensors[i]->type, (int)ggml_is_contiguous(tensors[i]), (long long)ggml_nelements(tensors[i]), (long long)ne,
                        (int)((tensors[i]->flags & GGML_TENSOR_FLAG_COMPUTE) != 0), b->fb.size(), b->mega_flushed);
            ok = false;
        }
        fbs[i] = &b->fb; ptrs[i] = (float *)tensors[i]->data; pools[i] = g->xpool[i] + (size_t)g->flip * g->xhalf;
    }
    if (ok && ne > 0 && ne <= 65536) {
        ok = qmm::FlowBuilder::fuse_allreduce(fbs, n, ptrs, (int)ne, pools, g->xhalf, g->xoff);
        static int said2 = 0;
        if (!ok && getenv("GGML_B200_FLOW_DEBUG") && said2++ < 8) fprintf(stderr, "ggml-b200: all-reduce of %s (%lld elements): the builder declined (last phase is not a single mat-vec writing this tensor, or the exchange pool is full)\n", tensors[0]->name, (long long)ne);
    } else ok = false;
    if (!ok) { flush_why w("all-reduce not fusable"); mega_flush(g->members[0]); }
    return ok;
}

// accessors used by comm.cpp
int b200_backend_cuda_device(ggml_backend_t backend) { return backend_is_ours(backend) ? ((backend_ctx *)backend->context)->dev->cuda_dev : -1; }
cudaStream_t b200_backend_stream(ggml_backend_t backend) { return backend_is_ours(backend) ? ((backend_ctx *)backend->context)->stream : nullptr; }

extern "C" {
// ---- measurement hooks for bench.py (not part of the ggml interface) ----
// Replays the most recently replayed captured graph (one decode token) `reps` times on its stream between two CUDA
// events: the device-resident throughput, no host copies.  Returns 0 and the elapsed milliseconds, or -1 if no graph.
__attribute__((visibility("default"))) int ggml_b200_replay_last_graph(int reps, float * ms_out, unsigned long long * launches_per_replay) {
    backend_ctx * b = g_last_graph_backend;
    if (!b || !b->last_entry || !b->last_entry->exec || g_snap_inputs.empty()) return -1;
    set_device(b->dev->cuda_dev);
    cudaEvent_t e0, e1;
    B200_CHECK(cudaEventCreate(&e0));
    B200_CHECK(cudaEventCreate(&e1));
    B200_CHECK(cudaStreamSynchronize(b->stream));
    B200_CHECK(cudaEventRecord(e0, b->stream));
    for (int i = 0; i < reps; i++) {
        if (g_snap_inputs.size() <= 16) {                  // inputs stay on the device: one small kernel restores them
            qmm::ops::MultiCopyArgs mc{};
            mc.n = (int)g_snap_inputs.size();
            for (int k = 0; k < mc.n; k++) { mc.dst[k] = g_snap_inputs[k].dst; mc.src[k] = (char *)g_snap_buf + g_snap_inputs[k].snap_off; mc.bytes[k] = (unsigned)g_snap_inputs[k].size; }
            B200_CHECK(qmm::ops::multi_copy(mc, b->stream));
        } else {
            for (auto & r : g_snap_inputs) B200_CHECK(cudaMemcpyAsync(r.dst, (char *)g_snap_buf + r.snap_off, r.size, cudaMemcpyDeviceToDevice, b->stream));
        }
        B200_CHECK(cudaGraphLaunch(b->last_entry->exec, b->stream));
    }
    B200_CHECK(cudaEventRecord(e1, b->stream));
    B200_CHECK(cudaEventSynchronize(e1));
    B200_CHECK(cudaEventElapsedTime(ms_out, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (launches_per_replay) *launches_per_replay = b->last_entry->n_launches;
    g_graph_launches += b->last_entry->n_launches * (uint64_t)reps;
    return 0;
}
// Re-read the device region of the most recent sizeable device->host tensor read (the logits of the last decoded token).  After
// ggml_b200_replay_last_graph the region holds what the REPLAY computed, so the bench can check that the timed replays produce
// the same logits as the end-to-end step they repeat.  Returns the number of bytes copied (0: nothing recorded / buffer too small).
__attribute__((visibility("default"))) unsigned long long ggml_b200_reread_last_output(void * dst, unsigned long long cap) {
    if (!g_last_read_src || g_last_read_size > cap) return 0;
    set_device(g_last_read_dev);
    B200_CHECK(cudaDeviceSynchronize());
    B200_CHECK(cudaMemcpy(dst, g_last_read_src, g_last_read_size, cudaMemcpyDeviceToHost));
    return g_last_read_size;
}
// enable journalling + device snapshots of graph inputs so that ggml_b200_replay_last_graph can restore them (see above)
__attribute__((visibility("default"))) void ggml_b200_enable_replay(int on) { g_journal_on = on != 0; }
// bytes moved through set/get_tensor(_async) and kernels launched (direct + inside graph replays) since load
__attribute__((visibility("default"))) void ggml_b200_stats(unsigned long long * h2d, unsigned long long * d2h, unsigned long long * launches) {
    if (h2d) *h2d = g_h2d_bytes.load();
    if (d2h) *d2h = g_d2h_bytes.load();
    if (launches) *launches = b200_qmm_launch_count() + g_graph_launches.load();
}

// dl entry points, ggml-backend-impl.h:232-271
__attribute__((visibility("default"))) ggml_backend_reg_t ggml_backend_init(void) {
    std::call_once(g_once, init_registry);
    return &g_reg;
}
__attribute__((visibility("default"))) int ggml_backend_score(void) {
    std::call_once(g_once, init_registry);
    return g_devices.empty() ? 0 : 100;
}
}
