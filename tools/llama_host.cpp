// llama_host.cpp -- a minimal driver over the REFERENCE's unmodified libllama (built by oracle/host.mk) that exposes
// what llama-bench measures (tools/llama-bench/llama-bench.cpp:2114-2162: test_prompt = llama_decode per n_batch chunk
// + one llama_synchronize; test_gen = llama_decode of 1 token + llama_synchronize per token) as a small C API that
// bench.py and the parity tests call through ctypes, plus a CLI.  (The unmodified llama-bench itself is built by oracle/host.mk too
// and reported beside these numbers; this driver exists for what llama-bench has no hooks for: logits out, cb_eval dumps, device
// replay.)  libllama, ggml and the backend registry it drives are the reference's own code, compiled unmodified by oracle/host.mk.
//
// The backend under test is selected exactly as a user would: GGML_BACKEND_PATH=/path/libggml-b200.so makes
// ggml_backend_load_all() dlopen the plugin (ggml-backend-reg.cpp:566-593); n_gpu_layers > 0 offloads to it.
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "ggml-backend.h"
#include "llama.h"

struct lh_ctx {
    llama_model * model = nullptr;
    llama_context * ctx = nullptr;
    int n_vocab = 0;
    int n_batch = 0;
};

// optional per-node dump (LH_DUMP=<file>): llama's cb_eval hook (ggml_backend_sched_set_eval_callback, ggml-backend.h:309-316)
static FILE * g_dump = nullptr;
// LH_DUMP_MULMAT=<dir>: for every MUL_MAT / MUL_MAT_ID node with a quantised weight, write weight bytes, f32 inputs and
// the backend's f32 output, so a test can replay the SAME mat-mul (same model, same prompt, same activations) elsewhere.
static int g_mm_count = 0;
static void dump_mulmat(struct ggml_tensor * t) {
    const char * dir = getenv("LH_DUMP_MULMAT");
    const struct ggml_tensor * w = t->src[0], * x = t->src[1];
    if (!dir || t->op != GGML_OP_MUL_MAT || !ggml_is_quantized(w->type) || !ggml_is_contiguous(w) || !ggml_is_contiguous(x) || x->type != GGML_TYPE_F32) return;
    if (g_mm_count >= (getenv("LH_DUMP_MULMAT_MAX") ? atoi(getenv("LH_DUMP_MULMAT_MAX")) : 64)) return;
    char path[512];
    snprintf(path, sizeof(path), "%s/mm_%03d.bin", dir, g_mm_count++);
    FILE * f = fopen(path, "wb");
    if (!f) return;
    int64_t hdr[4] = {(int64_t)w->type, w->ne[1], w->ne[0], x->ne[1]};       // type, M, K, N
    fwrite(hdr, sizeof(hdr), 1, f);
    char wname[64] = {0};                                                     // weights are read from the GGUF by name:
    strncpy(wname, w->name, 63);                                              // CPU_REPACK buffers cannot be read back
    fwrite(wname, 64, 1, f);
    std::vector<uint8_t> buf;
    buf.resize(ggml_nbytes(x));
    ggml_backend_tensor_get(x, buf.data(), 0, buf.size()); fwrite(buf.data(), 1, buf.size(), f);
    buf.resize(ggml_nbytes(t));
    ggml_backend_tensor_get(t, buf.data(), 0, buf.size()); fwrite(buf.data(), 1, buf.size(), f);
    fclose(f);
}

// LH_DUMP_TENSORS=<dir> + LH_DUMP_NAMES=<prefix>[,<prefix>...]: write the f32 output of every node whose name starts with one of
// the prefixes ("kqv_out-0", "result_norm", ...) to <dir>/<name>.<n>.f32; the scheduler is asked to stop ONLY at those nodes,
// so everything in between still runs fused, as in a normal decode.
static std::vector<std::string> g_want;
static int g_want_count = 0;
static bool wanted(const struct ggml_tensor * t) {
    for (const auto & w : g_want) if (strncmp(t->name, w.c_str(), w.size()) == 0) return true;
    return false;
}
static void dump_named(struct ggml_tensor * t) {
    const char * dir = getenv("LH_DUMP_TENSORS");
    if (!dir || !wanted(t) || t->type != GGML_TYPE_F32 || !ggml_is_contiguous(t)) return;
    char path[768];
    snprintf(path, sizeof(path), "%s/%s.%03d.f32", dir, t->name, g_want_count++);
    FILE * f = fopen(path, "wb");
    if (!f) return;
    std::vector<uint8_t> buf(ggml_nbytes(t));
    ggml_backend_tensor_get(t, buf.data(), 0, buf.size());
    fwrite(buf.data(), 1, buf.size(), f);
    fclose(f);
}

static bool dump_cb(struct ggml_tensor * t, bool ask, void *) {
    if (ask) return g_want.empty() ? true : wanted(t);
    dump_named(t);
    dump_mulmat(t);
    if (!g_dump || (t->type != GGML_TYPE_F32 && t->type != GGML_TYPE_F16)) return true;
    const size_t n = (size_t)ggml_nelements(t);
    if (!ggml_is_contiguous(t) || n == 0) { fprintf(g_dump, "%s %s noncontig\n", ggml_op_name(t->op), t->name); return true; }
    std::vector<uint8_t> buf(ggml_nbytes(t));
    ggml_backend_tensor_get(t, buf.data(), 0, buf.size());
    double sum = 0, asum = 0;
    std::vector<float> f(n);
    if (t->type == GGML_TYPE_F32) memcpy(f.data(), buf.data(), n * 4);
    else for (size_t i = 0; i < n; i++) f[i] = ggml_fp16_to_fp32(((const ggml_fp16_t *)buf.data())[i]);
    for (size_t i = 0; i < n; i++) { sum += f[i]; asum += fabs(f[i]); }
    fprintf(g_dump, "%s %s [%lld,%lld,%lld,%lld] sum=%.9g asum=%.9g v=", ggml_op_name(t->op), t->name, (long long)t->ne[0], (long long)t->ne[1],
            (long long)t->ne[2], (long long)t->ne[3], sum, asum);
    for (size_t i = 0; i < n && i < 6; i++) fprintf(g_dump, "%.7g,", f[i]);
    fprintf(g_dump, "\n");
    return true;
}

static void quiet_log(ggml_log_level level, const char * text, void *) {
    if (level >= GGML_LOG_LEVEL_WARN || getenv("LH_VERBOSE")) fputs(text, stderr);
}

extern "C" {

// devices: comma separated device names ("B2000,B2001") or NULL/"" = llama.cpp's default choice; split_mode: 0 none, 1 layer, 2 row, 3 tensor
void * lh_open(const char * path, int n_gpu_layers, int n_ctx, int n_batch, int n_ubatch, int flash_attn, int split_mode, int n_threads, const char * devices) {
    static bool inited = false;
    if (!inited) {
        llama_log_set(quiet_log, nullptr);
        ggml_backend_load_all();
        llama_backend_init();
        inited = true;
    }
    auto * h = new lh_ctx();
    llama_model_params mp = llama_model_default_params();
    mp.n_gpu_layers = n_gpu_layers;
    mp.split_mode = (llama_split_mode)split_mode;
    std::vector<ggml_backend_dev_t> devs;
    if (devices && *devices) {
        std::string s(devices);
        size_t pos = 0;
        while (pos <= s.size()) {
            size_t c = s.find(',', pos);
            std::string name = s.substr(pos, c == std::string::npos ? std::string::npos : c - pos);
            ggml_backend_dev_t d = ggml_backend_dev_by_name(name.c_str());
            if (!d) { fprintf(stderr, "lh_open: unknown device %s\n", name.c_str()); delete h; return nullptr; }
            devs.push_back(d);
            if (c == std::string::npos) break;
            pos = c + 1;
        }
        devs.push_back(nullptr);
        mp.devices = devs.data();
    }
    h->model = llama_model_load_from_file(path, mp);
    if (!h->model) { delete h; return nullptr; }
    llama_context_params cp = llama_context_default_params();
    cp.n_ctx = n_ctx;
    cp.n_batch = n_batch;
    cp.n_ubatch = n_ubatch;
    cp.n_threads = n_threads;
    cp.n_threads_batch = n_threads;
    cp.flash_attn_type = flash_attn ? LLAMA_FLASH_ATTN_TYPE_ENABLED : LLAMA_FLASH_ATTN_TYPE_DISABLED;
    cp.no_perf = true;
    if (const char * names = getenv("LH_DUMP_NAMES")) {
        g_want.clear();
        std::string ns(names);
        for (size_t pos = 0; pos <= ns.size();) { const size_t c = ns.find(',', pos); g_want.push_back(ns.substr(pos, c == std::string::npos ? std::string::npos : c - pos)); if (c == std::string::npos) break; pos = c + 1; }
    }
    if (getenv("LH_DUMP") || getenv("LH_DUMP_MULMAT") || getenv("LH_DUMP_TENSORS")) { if (!g_dump && getenv("LH_DUMP")) g_dump = fopen(getenv("LH_DUMP"), "w"); cp.cb_eval = dump_cb; cp.cb_eval_user_data = nullptr; }
    h->ctx = llama_init_from_model(h->model, cp);
    if (!h->ctx) { llama_model_free(h->model); delete h; return nullptr; }
    h->n_vocab = llama_vocab_n_tokens(llama_model_get_vocab(h->model));
    h->n_batch = n_batch;
    return h;
}

void lh_close(void * p) {
    auto * h = (lh_ctx *)p;
    if (!h) return;
    llama_free(h->ctx);
    llama_model_free(h->model);
    delete h;
}

int lh_n_vocab(void * p) { return ((lh_ctx *)p)->n_vocab; }
void lh_clear(void * p) { llama_memory_clear(llama_get_memory(((lh_ctx *)p)->ctx), true); }
void lh_sync(void * p) { llama_synchronize(((lh_ctx *)p)->ctx); }

// Decode n tokens (appended to the current sequence); copy the logits of the LAST token to logits_out (n_vocab floats).
int lh_decode(void * p, const int32_t * tokens, int n, float * logits_out) {
    auto * h = (lh_ctx *)p;
    std::vector<llama_token> t(tokens, tokens + n);
    for (int i = 0; i < n; i += h->n_batch) {
        const int nb = std::min(h->n_batch, n - i);
        const int rc = llama_decode(h->ctx, llama_batch_get_one(t.data() + i, nb));
        if (rc) return rc;
    }
    llama_synchronize(h->ctx);
    if (logits_out) {
        const float * l = llama_get_logits_ith(h->ctx, -1);
        if (!l) return -100;
        memcpy(logits_out, l, sizeof(float) * (size_t)h->n_vocab);
    }
    return 0;
}

// llama-bench's test_gen: n_gen single-token decodes, each followed by llama_synchronize. Returns seconds.
double lh_test_gen(void * p, int n_gen, unsigned seed) {
    auto * h = (lh_ctx *)p;
    std::mt19937 rng(seed);
    llama_token tok = (llama_token)(rng() % h->n_vocab);
    const auto t0 = std::chrono::steady_clock::now();
    for (int i = 0; i < n_gen; i++) {
        if (llama_decode(h->ctx, llama_batch_get_one(&tok, 1))) return -1.0;
        llama_synchronize(h->ctx);
        tok = (llama_token)(rng() % h->n_vocab);
    }
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// llama-bench's test_prompt: n_prompt random tokens in n_batch chunks, one llama_synchronize at the end. Returns seconds.
double lh_test_prompt(void * p, int n_prompt, unsigned seed) {
    auto * h = (lh_ctx *)p;
    std::mt19937 rng(seed);
    std::vector<llama_token> t((size_t)h->n_batch);
    const auto t0 = std::chrono::steady_clock::now();
    for (int done = 0; done < n_prompt;) {
        const int nb = std::min(n_prompt - done, h->n_batch);
        for (int i = 0; i < nb; i++) t[i] = (llama_token)(rng() % h->n_vocab);
        if (llama_decode(h->ctx, llama_batch_get_one(t.data(), nb))) return -1.0;
        done += nb;
    }
    llama_synchronize(h->ctx);
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

}  // extern "C"

#ifdef LH_MAIN
// CLI: llama_host model.gguf [-ngl N] [-p N] [-n N] [-r R] [-b N] [-ub N] [-fa 0|1] [-sm 0..3] [-t N] [-dev names]
int main(int argc, char ** argv) {
    if (argc < 2) { fprintf(stderr, "usage: %s model.gguf [-ngl N] [-p N] [-n N] [-r R] [-b N] [-ub N] [-fa 0|1] [-sm N] [-t N] [-dev a,b]\n", argv[0]); return 2; }
    int ngl = 99, np = 512, ng = 128, reps = 3, nb = 2048, nub = 512, fa = 1, sm = 1, nt = 8;
    const char * dev = nullptr;
    for (int i = 2; i + 1 < argc; i += 2) {
        std::string a = argv[i];
        if (a == "-ngl") ngl = atoi(argv[i + 1]); else if (a == "-p") np = atoi(argv[i + 1]); else if (a == "-n") ng = atoi(argv[i + 1]);
        else if (a == "-r") reps = atoi(argv[i + 1]); else if (a == "-b") nb = atoi(argv[i + 1]); else if (a == "-ub") nub = atoi(argv[i + 1]);
        else if (a == "-fa") fa = atoi(argv[i + 1]); else if (a == "-sm") sm = atoi(argv[i + 1]); else if (a == "-t") nt = atoi(argv[i + 1]);
        else if (a == "-dev") dev = argv[i + 1];
    }
    void * h = lh_open(argv[1], ngl, std::max(np + ng, 512), nb, nub, fa, sm, nt, dev);
    if (!h) { fprintf(stderr, "failed to load %s\n", argv[1]); return 1; }
    if (np > 0) { lh_test_prompt(h, std::min(np, nub), 1); lh_clear(h); }      // warm-up like llama-bench.cpp:2353-2379
    if (ng > 0) { lh_test_gen(h, 1, 1); lh_clear(h); }
    for (int r = 0; r < reps; r++) {
        if (np > 0) { lh_clear(h); double s = lh_test_prompt(h, np, 7 + r); printf("{\"test\": \"pp%d\", \"rep\": %d, \"t_s\": %.6f, \"tok_s\": %.2f}\n", np, r, s, np / s); }
        if (ng > 0) { lh_clear(h); double s = lh_test_gen(h, ng, 9 + r); printf("{\"test\": \"tg%d\", \"rep\": %d, \"t_s\": %.6f, \"tok_s\": %.2f}\n", ng, r, s, ng / s); }
    }
    lh_close(h);
    return 0;
}
#endif
