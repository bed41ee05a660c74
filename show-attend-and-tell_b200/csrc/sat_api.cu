// sat_api.cu — the C ABI of libsat_b200.so (include/sat_b200.h): handle, weight
// ingestion (TF variable names/layouts, base_model.py:242-278), workspace, and the
// kernel sequences of prepare / decode step / decode loop / beam search.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/sat_b200.h"
#include "sat_attention.cuh"
#include "sat_linear.cuh"
#include "sat_rows.cuh"
#include "sat_internal.h"

using namespace sat;

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CK(x)                                                                                   \
    do {                                                                                        \
        cudaError_t e_ = (x);                                                                   \
        if (e_ != cudaSuccess) return fail(SAT_ERR_CUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
    } while (0)
#define RET(x)                 \
    do {                       \
        int r_ = (x);          \
        if (r_ != SAT_OK) return r_; \
    } while (0)

// ------------------------------------------------------------------ handle
struct Layer {
    std::string name;  // TF scope, e.g. "decode/fc_1"
    int K = 0, n_out = 0;
    bool lstm = false, has_bias = true;
    int k_blocks = 0, n_tiles = 0;
    uint8_t* wpack = nullptr;
    float* bias = nullptr;  // packed order, n_tiles*128
    bool w_set = false, b_set = false;
    uint8_t* xpack = nullptr;  // packed activations (x_mode 1)
    size_t xpack_bytes = 0;
    unsigned* xbar = nullptr;  // {count, generation}
    unsigned long long* am_key = nullptr;   // fused-argmax tile candidates
    unsigned* am_ctr = nullptr;
    size_t am_n = 0;
    float* am_sum = nullptr;     // word probabilities: per-tile softmax partials (like am_key), forced-word logits
    float* am_wlogit = nullptr;
    size_t am_sum_n = 0;
    float2* am_smp = nullptr;    // sampling: per-tile {raw maximum, raw logit of the sampled candidate} (like am_key)
    size_t am_smp_n = 0;
};

struct VecParam {  // a kernel of shape [n,1] kept as a plain fp32 vector
    std::string name;
    int n = 0;
    float* dev = nullptr;
    bool set = false;
};

struct GraphEntry {
    std::vector<long long> key;
    int seen = 0;
    cudaGraphExec_t exec = nullptr;
    long long kernels = 0;  // kernel launches one replay stands for
};

struct sat_handle {
    sat_dims d;
    int dev = 0, num_sms = 0, smem_optin = 0;
    int opt_prologue1 = 1;   // mean of the contexts taken by the packing pass of the projection ("prologue1")
    int opt_gemm = 1, opt_layout = 0, opt_graphs = 1, opt_hoist = 1, opt_coop = 1, opt_xpack = 1;
    // dense weights: -1 = per launch (see plan()), else one policy for every weight stream; both attention streams
    // evict_first
    int opt_l2_w = -1, opt_l2_t = 1, opt_l2_ctx = 1;
    bool weights_locked = false;

    Layer init_a1, init_a2, init_b1, init_b2;  // 1-layer mode uses init_a1 / init_b1 as fc_a / fc_b
    Layer att_1a, att_1b;                      // 1-layer mode: att_1b is fc_b [H, L], att_1a unused
    VecParam att_vec;                          // attend/fc_2 [A] or attend/fc_a [D]
    Layer lstm;
    Layer dec_1, dec_2;                        // 1-layer mode uses dec_2 as decode/fc
    float* embedding = nullptr;
    bool emb_set = false;
    std::vector<Layer*> layers;

    // workspace
    int max_rows = 0;
    float *T1 = nullptr, *q = nullptr, *e = nullptr, *alpha = nullptr, *z = nullptr, *mean = nullptr;
    float *tmp_a = nullptr, *tmp_b = nullptr, *t_dec = nullptr, *logits = nullptr;
    float* st_c[2] = {nullptr, nullptr};
    float* st_h[2] = {nullptr, nullptr};
    int32_t *word = nullptr, *zero_word = nullptr;
    unsigned* rowcnt = nullptr;
    // beam
    int32_t *topk_idx = nullptr, *part_n = nullptr, *comp_n = nullptr, *comp_sent = nullptr;
    int32_t* sent[2] = {nullptr, nullptr};
    float* topk_p = nullptr;
    double* part_score = nullptr;
    void* comp_heap = nullptr;
    // beam maps (sat_beam_search_maps), allocated on the first request: back-pointer history, see BeamParams
    float *hist_alpha = nullptr, *hist_p = nullptr, *comp_p = nullptr;
    int32_t *hist_parent = nullptr, *comp_prov = nullptr, *res_src = nullptr;
    // host-form staging
    float* stage_ctx = nullptr;
    void* stage_misc = nullptr;
    size_t stage_misc_bytes = 0;
    // cross-batch overlap of the loop prologue (option "xbatch"): the projection / initialize of batch i+1 run on
    // their own stream into the other of two buffer sets while batch i decodes
    struct XbSlot {
        float *T1 = nullptr, *c0 = nullptr, *h0 = nullptr;
        uint8_t* pa_h0 = nullptr;
        cudaEvent_t ev_prep = nullptr, ev_done = nullptr;
        bool used = false;
    } xb[2];
    cudaStream_t xb_stream = nullptr;
    int xb_next = 0;
    int opt_xbatch = 0;
    int ops_since_xb = 0;   // compute entry points called since the last overlapped loop (they share slot 0's buffers)
    // pipelined host-buffer loop (sat_decode_loop_host_submit / _wait): two staging slots and a copy stream
    float* pipe_ctx[2] = {nullptr, nullptr};
    int32_t* pipe_tok[2] = {nullptr, nullptr};   // [tokens | forced words]
    size_t pipe_tok_elems[2] = {0, 0};
    cudaStream_t pipe_copy = nullptr;
    cudaEvent_t pipe_up[2] = {nullptr, nullptr}, pipe_done[2] = {nullptr, nullptr};
    bool pipe_busy[2] = {false, false};

    // contexts state
    const float* prep_ctx = nullptr;
    int prep_ni = 0;
    float* att_part = nullptr;
    size_t att_part_floats = 0;
    // packed activations (bf16 hi/lo UMMA tiles written by the producer kernels)
    bool pa_ok = false;            // every operand width is a multiple of 64
    int opt_pa = 1;
    uint8_t* pa_h[2] = {nullptr, nullptr};
    uint8_t *pa_z = nullptr, *pa_emb = nullptr, *pa_t = nullptr;
    // valid for the duration of one step_impl call
    bool pa_on = false;
    uint8_t *pa_cur_h_in = nullptr, *pa_cur_h_out = nullptr, *pa_cur_z = nullptr;
    float* z2[2] = {nullptr, nullptr};       // context vectors, double buffered for the overlapped loop
    uint8_t* pa_z2[2] = {nullptr, nullptr};
    cudaStream_t side = nullptr;           // second stream of the decode loop (attention of step t+1)
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int opt_overlap = 2, opt_att_sms = 0, opt_att_occ = 1, opt_att_warps = 8, opt_pdl = 1, opt_warm = 1, opt_att_wpc = 1, opt_att_reuse_q = 0, opt_l2_vocab = -1, opt_l2_prefetch = 0, opt_stages = 0, opt_train_tc = 1, opt_dec1_splits = 0;
    // chained dense launch of the greedy loop (sat_chain.cu): arrival counters, split-K scratch, per-row arg-max keys
    unsigned* chain_ctr = nullptr;         // [kChainMaxPhase + kChainMaxPhase * kChainMaxTiles]
    float* chain_scratch = nullptr;
    unsigned long long* chain_best = nullptr;
    int opt_chain = 0, opt_chain_cluster = 0;   // (opt-in: see fused_loop_available)
    int chain_clusters[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};   // resident clusters of the chained kernel per cluster size
    const unsigned* att_qflag = nullptr;   // set around the attention launch that runs beside a chained launch
    unsigned att_qtarget = 0;
    SampleParams* smp = nullptr;           // sampling loop: {seed, 1 / temperature}, written before each call (not in graphs)
    void* train = nullptr;                 // training state (sat_train.cu)
    void (*train_free)(void*) = nullptr;
    unsigned long long* trace = nullptr;   // [1024][16] timeline stamps of the last traced launch
    int opt_trace = 0;
    int trace_at = 0;      // with trace == 1: index of the dense launch (counted from the option call) to stamp
    bool lin_w_dynamic = false;   // next dense launch: its weight operand comes from the preceding kernel
    int att_loop_grid = 0; // CTAs of the last attention launch that ran beside the vocabulary layer (decode loop)
    int att_loop_beside = 0; // 1: that launch ran beside its predecessor (did not wait for it before streaming)
    int tl_count = 0;      // with trace == 3: launches recorded so far ({min start, max end} per launch)
    std::vector<std::string> tl_names;

    std::vector<GraphEntry> graphs;

    // launch accounting / optional per-kernel-family timing (eager launches only)
    long long launches = 0;
    int opt_profile = 0;
    int cur_tag = 0;
    struct ProfRec { int tag; cudaEvent_t a, b; };
    std::vector<ProfRec> prof;
};

enum ProfTag { kTagAtt = 0, kTagAttState, kTagLstm, kTagDec1, kTagDec2, kTagProj, kTagInit, kTagRows, kTagBeam, kNumTags };
static const char* kTagNames[kNumTags] = {"att", "att_state", "lstm", "dec1", "dec2", "proj", "init", "rows", "beam"};

struct ProfScope {
    sat_handle* h; cudaStream_t st; bool on; cudaEvent_t a = nullptr, b = nullptr; int tag;
    ProfScope(sat_handle* h_, int tag_, cudaStream_t st_) : h(h_), st(st_), tag(tag_) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        cudaStreamIsCapturing(st, &cs);
        on = h->opt_profile && cs == cudaStreamCaptureStatusNone;
        if (on) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, st); }
    }
    ~ProfScope() {
        if (on) { cudaEventRecord(b, st); h->prof.push_back({tag, a, b}); }
    }
};

template <typename T>
static int dmalloc(T** p, size_t n) {
    if (n == 0) n = 1;
    cudaError_t e = cudaMalloc((void**)p, n * sizeof(T));
    if (e != cudaSuccess) return fail(SAT_ERR_NOMEM, "cudaMalloc(%zu bytes): %s", n * sizeof(T), cudaGetErrorString(e));
    return SAT_OK;
}

// Scratch buffers grow (free + larger allocation) when a call needs more than any call before it.  Every captured graph
// may hold the old address, so the graphs go with it and are captured again on their next use.
static void drop_graphs(sat_handle* h) {
    for (auto& g : h->graphs)
        if (g.exec) cudaGraphExecDestroy(g.exec);
    h->graphs.clear();
}

static int layer_setup(sat_handle* h, Layer& ly, const char* name, int K, int n_out, bool lstm, bool has_bias) {
    ly.name = name;
    ly.K = K;
    ly.n_out = n_out;
    ly.lstm = lstm;
    ly.has_bias = has_bias;
    ly.k_blocks = (K + kBK - 1) / kBK;
    ly.n_tiles = (n_out + kTileN - 1) / kTileN;
    if (K % 8) return fail(SAT_ERR_UNSUPPORTED, "%s: input width %d must be a multiple of 8", name, K);
    RET(dmalloc(&ly.wpack, (size_t)ly.n_tiles * ly.k_blocks * kWStageBytes));
    RET(dmalloc(&ly.bias, (size_t)ly.n_tiles * kTileN));
    CK(cudaMemset(ly.bias, 0, (size_t)ly.n_tiles * kTileN * sizeof(float)));
    ly.b_set = !has_bias;
    h->layers.push_back(&ly);
    return SAT_OK;
}

static void layer_free(Layer& ly) {
    cudaFree(ly.wpack);
    cudaFree(ly.bias);
    cudaFree(ly.xpack);
    cudaFree(ly.xbar);
    cudaFree(ly.am_key);
    cudaFree(ly.am_ctr);
    cudaFree(ly.am_sum);
    cudaFree(ly.am_wlogit);
    cudaFree(ly.am_smp);
    ly = Layer();
}

int sat_fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
const sat_dims* sat_handle_dims(sat_handle* h) { return &h->d; }
int sat_handle_device(sat_handle* h) { return h->dev; }
void** sat_handle_train_slot(sat_handle* h) { return &h->train; }
void sat_handle_set_train_free(sat_handle* h, void (*fn)(void*)) { h->train_free = fn; }

extern "C" int sat_version(void) { return 100; }
extern "C" const char* sat_last_error(void) { return g_err; }

extern "C" void sat_destroy(sat_handle* h) {
    if (!h) return;
    cudaDeviceSynchronize();
    if (h->train && h->train_free) h->train_free(h->train);
    if (h->side) cudaStreamDestroy(h->side);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->xb_stream) cudaStreamDestroy(h->xb_stream);
    for (int i = 0; i < 2; ++i) {
        if (h->xb[i].ev_prep) cudaEventDestroy(h->xb[i].ev_prep);
        if (h->xb[i].ev_done) cudaEventDestroy(h->xb[i].ev_done);
        if (i == 1) { cudaFree(h->xb[i].T1); cudaFree(h->xb[i].c0); cudaFree(h->xb[i].h0); cudaFree(h->xb[i].pa_h0); }   // slot 0 aliases the handle's own buffers
    }
    if (h->pipe_copy) cudaStreamDestroy(h->pipe_copy);
    for (int i = 0; i < 2; ++i) {
        if (h->pipe_up[i]) cudaEventDestroy(h->pipe_up[i]);
        if (h->pipe_done[i]) cudaEventDestroy(h->pipe_done[i]);
        cudaFree(h->pipe_ctx[i]);
        cudaFree(h->pipe_tok[i]);
    }
    for (auto& g : h->graphs)
        if (g.exec) cudaGraphExecDestroy(g.exec);
    for (Layer* ly : h->layers) layer_free(*ly);
    void* bufs[] = {h->att_vec.dev, h->embedding, h->T1, h->q, h->e, h->alpha, h->z, h->mean, h->tmp_a, h->tmp_b,
                    h->t_dec, h->logits, h->st_c[0], h->st_c[1], h->st_h[0], h->st_h[1], h->word, h->zero_word,
                    h->rowcnt, h->topk_idx, h->part_n, h->comp_n, h->comp_sent, h->sent[0], h->sent[1], h->topk_p,
                    h->part_score, h->comp_heap, h->stage_ctx, h->stage_misc, h->att_part, h->trace, h->pa_h[0], h->pa_h[1], h->pa_z, h->pa_emb, h->pa_t, h->pa_z2[1], h->z2[1],
                    h->chain_ctr, h->chain_scratch, h->chain_best, h->hist_alpha, h->hist_p, h->comp_p, h->hist_parent,
                    h->comp_prov, h->res_src, h->smp};
    for (void* b : bufs) cudaFree(b);
    delete h;
}

extern "C" int sat_create(const sat_dims* dims, sat_handle** out) {
    if (!dims || !out) return fail(SAT_ERR_INVALID, "sat_create: null argument");
    *out = nullptr;
    const sat_dims& d = *dims;
    if (d.max_batch < 1 || d.num_ctx < 1 || d.dim_ctx < 1 || d.num_lstm_units < 1 || d.vocabulary_size < 2)
        return fail(SAT_ERR_INVALID, "sat_create: non-positive dimension");
    if (d.num_ctx > 256) return fail(SAT_ERR_UNSUPPORTED, "num_ctx %d > 256", d.num_ctx);
    if (d.dim_ctx % 32 || d.num_lstm_units % 32 || d.dim_embedding % 8 || d.dim_attend_layer % 8 ||
        d.dim_decode_layer % 8 || d.dim_initalize_layer % 8)
        return fail(SAT_ERR_UNSUPPORTED, "dim_ctx and num_lstm_units must be multiples of 32, the other widths of 8");
    if (d.max_beam > 4) return fail(SAT_ERR_UNSUPPORTED, "max_beam %d > 4", d.max_beam);
    for (int v : {d.num_attend_layers, d.num_decode_layers, d.num_initalize_layers})
        if (v != 1 && v != 2) return fail(SAT_ERR_INVALID, "num_*_layers must be 1 or 2");
    int ndev = 0;
    cudaError_t ce = cudaGetDeviceCount(&ndev);
    if (ce != cudaSuccess || ndev == 0)
        return fail(SAT_ERR_CUDA, "no CUDA device (%s): sat_b200 has no CPU path", cudaGetErrorString(ce));

    sat_handle* h = new sat_handle();
    h->d = d;
    // SAT_PDL=0: start with programmatic dependent launch off (option "pdl").  For tools that assume one kernel of a
    // stream at a time: compute-sanitizer's synccheck reports warps of an early-started kernel as divergent at their
    // first block barrier.
    if (const char* e = getenv("SAT_PDL")) h->opt_pdl = (e[0] == '0') ? 0 : 1;
    int rc = SAT_OK;
    auto body = [&]() -> int {
        CK(cudaGetDevice(&h->dev));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, h->dev));
        if (prop.major != 9 || prop.minor != 0)   // (the library holds sm_90a code only)
            return fail(SAT_ERR_UNSUPPORTED, "device sm_%d%d is not sm_90", prop.major, prop.minor);
        h->num_sms = prop.multiProcessorCount;
        CK(cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->dev));
        CK(lin_init_attrs());
        const int D = d.dim_ctx, E = d.dim_embedding, H = d.num_lstm_units, A = d.dim_attend_layer,
                  Dd = d.dim_decode_layer, I = d.dim_initalize_layer, V = d.vocabulary_size, L = d.num_ctx;
        if (d.num_initalize_layers == 2) {
            RET(layer_setup(h, h->init_a1, "initialize/fc_a1", D, I, false, true));
            RET(layer_setup(h, h->init_a2, "initialize/fc_a2", I, H, false, true));
            RET(layer_setup(h, h->init_b1, "initialize/fc_b1", D, I, false, true));
            RET(layer_setup(h, h->init_b2, "initialize/fc_b2", I, H, false, true));
        } else {
            RET(layer_setup(h, h->init_a1, "initialize/fc_a", D, H, false, true));
            RET(layer_setup(h, h->init_b1, "initialize/fc_b", D, H, false, true));
        }
        if (d.num_attend_layers == 2) {
            RET(layer_setup(h, h->att_1a, "attend/fc_1a", D, A, false, true));
            RET(layer_setup(h, h->att_1b, "attend/fc_1b", H, A, false, true));
            h->att_vec.name = "attend/fc_2";
            h->att_vec.n = A;
        } else {
            RET(layer_setup(h, h->att_1b, "attend/fc_b", H, L, false, false));
            h->att_vec.name = "attend/fc_a";
            h->att_vec.n = D;
        }
        RET(dmalloc(&h->att_vec.dev, (size_t)h->att_vec.n));
        RET(layer_setup(h, h->lstm, "lstm/lstm_cell", D + E + H, 4 * H, true, true));
        if (d.num_decode_layers == 2) {
            RET(layer_setup(h, h->dec_1, "decode/fc_1", H + D + E, Dd, false, true));
            RET(layer_setup(h, h->dec_2, "decode/fc_2", Dd, V, false, true));
        } else {
            RET(layer_setup(h, h->dec_2, "decode/fc", H + D + E, V, false, true));
        }
        RET(dmalloc(&h->embedding, (size_t)V * E));

        const size_t R = (size_t)d.max_batch;
        h->max_rows = d.max_batch;
        const int RL = d.num_attend_layers == 2 ? A : D;
        if (d.num_attend_layers == 2) RET(dmalloc(&h->T1, R * L * A));
        RET(dmalloc(&h->q, R * (size_t)(d.num_attend_layers == 2 ? A : L)));
        (void)RL;
        RET(dmalloc(&h->e, R * L));
        RET(dmalloc(&h->alpha, R * L));
        RET(dmalloc(&h->z, R * D));
        RET(dmalloc(&h->mean, R * D));
        RET(dmalloc(&h->tmp_a, R * (size_t)(I > H ? I : H)));
        RET(dmalloc(&h->tmp_b, R * (size_t)(I > H ? I : H)));
        RET(dmalloc(&h->t_dec, R * Dd));
        RET(dmalloc(&h->logits, R * V));
        for (int i = 0; i < 2; ++i) {
            RET(dmalloc(&h->st_c[i], R * H));
            RET(dmalloc(&h->st_h[i], R * H));
        }
        RET(dmalloc(&h->word, R));
        RET(dmalloc(&h->zero_word, R));
        CK(cudaMemset(h->zero_word, 0, R * sizeof(int32_t)));
        RET(dmalloc(&h->rowcnt, R));
        CK(cudaMemset(h->rowcnt, 0, R * sizeof(unsigned)));
        h->pa_ok = (D % 64 == 0) && (E % 64 == 0) && (H % 64 == 0) && (d.num_decode_layers == 1 || Dd % 64 == 0);
        if (h->pa_ok) {
            const size_t RP = R + 272;   // rows padded to whole row tiles
            RET(dmalloc(&h->pa_h[0], RP * H * 4));
            RET(dmalloc(&h->pa_h[1], RP * H * 4));
            RET(dmalloc(&h->pa_z, RP * D * 4));
            RET(dmalloc(&h->pa_z2[1], RP * D * 4));
            h->pa_z2[0] = h->pa_z;
            RET(dmalloc(&h->z2[1], R * D));
            h->z2[0] = h->z;
            RET(dmalloc(&h->pa_emb, RP * E * 4));
            RET(dmalloc(&h->pa_t, RP * Dd * 4));
        }
        const int T = d.max_caption_length > 0 ? d.max_caption_length : 1;
        if (d.max_beam >= 1) {
            const size_t K = (size_t)d.max_beam + 1;
            RET(dmalloc(&h->topk_idx, R * K));
            RET(dmalloc(&h->topk_p, R * K));
            RET(dmalloc(&h->part_score, R));
            RET(dmalloc(&h->part_n, R));
            RET(dmalloc(&h->comp_n, R));
            RET(dmalloc(&h->comp_sent, R * T));
            RET(dmalloc(&h->sent[0], R * T));
            RET(dmalloc(&h->sent[1], R * T));
            RET(dmalloc((uint8_t**)&h->comp_heap, R * beam_citem_bytes()));
        }
        return SAT_OK;
    };
    rc = body();
    if (rc != SAT_OK) {
        sat_destroy(h);
        return rc;
    }
    *out = h;
    return SAT_OK;
}

extern "C" int sat_set_option(sat_handle* h, const char* key, int64_t value) {
    if (!h || !key) return fail(SAT_ERR_INVALID, "sat_set_option: null argument");
    std::string k(key);
    if (k == "gemm") h->opt_gemm = (int)value;
    else if (k == "umma_layout") {
        if (h->weights_locked && (int)value != h->opt_layout)
            return fail(SAT_ERR_STATE, "umma_layout must be chosen before the first sat_set_weight");
        if (value != 0 && value != 1) return fail(SAT_ERR_INVALID, "umma_layout must be 0 or 1");
        h->opt_layout = (int)value;
    } else if (k == "graphs") h->opt_graphs = (int)value;
    else if (k == "hoist") { h->opt_hoist = (int)value; h->prep_ctx = nullptr; }
    else if (k == "prologue1") h->opt_prologue1 = (int)value;
    else if (k == "coop") h->opt_coop = (int)value;
    else if (k == "xpack") h->opt_xpack = (int)value;
    else if (k == "pa") h->opt_pa = (int)value;
    else if (k == "overlap") h->opt_overlap = (int)value;
    else if (k == "att_sms") h->opt_att_sms = (int)value;
    else if (k == "att_occ") h->opt_att_occ = (int)value;
    else if (k == "att_warps") h->opt_att_warps = (int)value;
    else if (k == "pdl") h->opt_pdl = (int)value;
    else if (k == "warm") h->opt_warm = (int)value;
    else if (k == "att_wpc") h->opt_att_wpc = (int)value;
    else if (k == "att_reuse_q") h->opt_att_reuse_q = (int)value;
    else if (k == "xbatch") h->opt_xbatch = (int)value;
    else if (k == "chain") h->opt_chain = (int)value;
    else if (k == "chain_cluster") h->opt_chain_cluster = (int)value;
    else if (k == "trace") {
        h->opt_trace = (int)value;
        if (value && !h->trace) RET(dmalloc(&h->trace, (size_t)1024 * 16));
        if (h->trace) CK(cudaMemset(h->trace, value == 3 ? 0xFF : 0, 1024 * 16 * sizeof(unsigned long long)));
        if (value == 3 && h->trace) {   // max cells start at 0, min cells at ~0
            std::vector<unsigned long long> init(1024 * 16);
            for (size_t i = 0; i < init.size(); ++i) init[i] = (i & 1) ? 0ull : ~0ull;   // cells 0,2 are minima, 1,3 maxima
            CK(cudaMemcpy(h->trace, init.data(), init.size() * 8, cudaMemcpyHostToDevice));
        }
        h->tl_count = 0;
        h->tl_names.clear();
        return SAT_OK;
    } else if (k == "trace_at") { h->trace_at = (int)value; return SAT_OK; }
    else if (k == "l2_w") h->opt_l2_w = (int)value;
    else if (k == "l2_vocab") h->opt_l2_vocab = (int)value;
    else if (k == "l2_prefetch") h->opt_l2_prefetch = (int)value;
    else if (k == "stages") h->opt_stages = (int)value;
    else if (k == "train_tc") h->opt_train_tc = (int)value;
    else if (k == "dec1_splits") h->opt_dec1_splits = (int)value;
    else if (k == "l2_t") h->opt_l2_t = (int)value;
    else if (k == "l2_ctx") h->opt_l2_ctx = (int)value;
    else if (k == "profile") {
        h->opt_profile = (int)value;
        for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
        h->prof.clear();
        return SAT_OK;
    } else if (k == "reset_counters") { h->launches = 0; return SAT_OK; }
    else return fail(SAT_ERR_INVALID, "unknown option '%s'", key);
    if (h->xb_stream) cudaStreamSynchronize(h->xb_stream);
    for (auto& g : h->graphs) {  // options change the captured work
        if (g.exec) cudaGraphExecDestroy(g.exec);
    }
    h->graphs.clear();
    return SAT_OK;
}

extern "C" int sat_get_info(sat_handle* h, const char* key, int64_t* value) {
    if (!h || !key || !value) return fail(SAT_ERR_INVALID, "sat_get_info: null argument");
    std::string k(key);
    if (k == "num_sms") *value = h->num_sms;
    else if (k == "smem_optin") *value = h->smem_optin;
    else if (k == "gemm") *value = h->opt_gemm;
    else if (k == "umma_layout") *value = h->opt_layout;
    else if (k == "launches") *value = h->launches;
    else if (k.rfind("prof_ns_", 0) == 0 || k.rfind("prof_n_", 0) == 0) {
        const bool want_n = k.rfind("prof_n_", 0) == 0;
        const std::string t = k.substr(want_n ? 7 : 8);
        int tag = -1;
        for (int i = 0; i < kNumTags; ++i) if (t == kTagNames[i]) tag = i;
        if (tag < 0) return fail(SAT_ERR_INVALID, "unknown profile tag '%s'", t.c_str());
        CK(cudaDeviceSynchronize());
        double ns = 0; long long n = 0;
        for (auto& r : h->prof) if (r.tag == tag) { float ms = 0; cudaEventElapsedTime(&ms, r.a, r.b); ns += ms * 1e6; ++n; }
        *value = want_n ? n : (int64_t)ns;
    }
    else if (k == "trace_ptr") *value = (int64_t)(uintptr_t)h->trace;
    else if (k == "tl_count") *value = h->tl_count;
    else if (k == "att_loop_grid") *value = h->att_loop_grid;
    else if (k == "att_loop_beside") *value = h->att_loop_beside;
    else if (k.rfind("tl_tag_", 0) == 0) {   // family code of timeline entry i: index into the tag list, grid in the high bits
        const int i = atoi(k.c_str() + 7);
        if (i < 0 || i >= (int)h->tl_names.size()) return fail(SAT_ERR_INVALID, "timeline index");
        snprintf(g_err, sizeof(g_err), "%s", h->tl_names[i].c_str());   // name returned through sat_last_error()
        *value = i;
    }
    else if (k == "weight_bytes") {
        size_t b = 0;
        for (Layer* ly : h->layers) b += (size_t)ly->n_tiles * ly->k_blocks * kWStageBytes;
        *value = (int64_t)b;
    } else {
        int rc = SAT_OK;
        if (sat_train_info(h, key, value, &rc)) return rc;
        return fail(SAT_ERR_INVALID, "unknown info key '%s'", key);
    }
    return SAT_OK;
}

// ------------------------------------------------------------------ weights
extern "C" int sat_set_weight(sat_handle* h, const char* tf_var_name, const float* dev, int64_t rows, int64_t cols,
                              void* stream) {
    if (!h || !tf_var_name || !dev) return fail(SAT_ERR_INVALID, "sat_set_weight: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaSetDevice(h->dev));
    std::string name(tf_var_name);
    if (name.size() > 2 && name.compare(name.size() - 2, 2, ":0") == 0) name.resize(name.size() - 2);
    h->weights_locked = true;
    h->prep_ctx = nullptr;
    if (h->xb_stream) CK(cudaStreamSynchronize(h->xb_stream));   // a prologue may still be reading the old weights
    if (name == "word_embedding/weights") {
        if (rows != h->d.vocabulary_size || cols != h->d.dim_embedding)
            return fail(SAT_ERR_INVALID, "%s: expected [%d,%d], got [%lld,%lld]", name.c_str(), h->d.vocabulary_size,
                        h->d.dim_embedding, (long long)rows, (long long)cols);
        CK(cudaMemcpyAsync(h->embedding, dev, (size_t)rows * cols * sizeof(float), cudaMemcpyDeviceToDevice, st));
        h->emb_set = true;
        return SAT_OK;
    }
    if (name == h->att_vec.name + "/kernel") {
        if (rows * cols != h->att_vec.n)
            return fail(SAT_ERR_INVALID, "%s: expected %d elements, got [%lld,%lld]", name.c_str(), h->att_vec.n,
                        (long long)rows, (long long)cols);
        CK(cudaMemcpyAsync(h->att_vec.dev, dev, (size_t)h->att_vec.n * sizeof(float), cudaMemcpyDeviceToDevice, st));
        h->att_vec.set = true;
        return SAT_OK;
    }
    for (Layer* ly : h->layers) {
        if (name == ly->name + "/kernel") {
            if (rows != ly->K || cols != ly->n_out)
                return fail(SAT_ERR_INVALID, "%s: expected [%d,%d], got [%lld,%lld]", name.c_str(), ly->K, ly->n_out,
                            (long long)rows, (long long)cols);
            CK(lin_repack_weight(dev, ly->K, ly->n_out, ly->lstm ? ly->n_out / 4 : 0, ly->wpack, h->opt_layout, st));
            ly->w_set = true;
            return SAT_OK;
        }
        if (name == ly->name + "/bias") {
            if (!ly->has_bias) return fail(SAT_ERR_INVALID, "%s: layer has no bias (use_bias=False)", name.c_str());
            if (rows * cols != ly->n_out)
                return fail(SAT_ERR_INVALID, "%s: expected %d elements, got [%lld,%lld]", name.c_str(), ly->n_out,
                            (long long)rows, (long long)cols);
            CK(lin_repack_bias(dev, ly->n_out, ly->lstm ? ly->n_out / 4 : 0, ly->bias, st));
            ly->b_set = true;
            return SAT_OK;
        }
    }
    return fail(SAT_ERR_INVALID, "unknown variable '%s'", name.c_str());
}

extern "C" int sat_weights_missing(sat_handle* h) {
    if (!h) return fail(SAT_ERR_INVALID, "null handle");
    int missing = 0;
    for (Layer* ly : h->layers) missing += (ly->w_set ? 0 : 1) + (ly->b_set ? 0 : 1);
    missing += h->emb_set ? 0 : 1;
    missing += h->att_vec.set ? 0 : 1;
    return missing;
}

static int require_ready(sat_handle* h) {
    if (!h) return fail(SAT_ERR_INVALID, "null handle");
    CK(cudaSetDevice(h->dev));   // lazily allocated buffers and every launch belong to the handle's device
    ++h->ops_since_xb;
    for (Layer* ly : h->layers) {
        if (!ly->w_set) return fail(SAT_ERR_STATE, "variable %s/kernel was never set", ly->name.c_str());
        if (!ly->b_set) return fail(SAT_ERR_STATE, "variable %s/bias was never set", ly->name.c_str());
    }
    if (!h->emb_set) return fail(SAT_ERR_STATE, "variable word_embedding/weights was never set");
    if (!h->att_vec.set) return fail(SAT_ERR_STATE, "variable %s/kernel was never set", h->att_vec.name.c_str());
    return SAT_OK;
}

// ------------------------------------------------------------ dense planning
static LinSeg seg(const float* p, int ld, int width, const int32_t* gather = nullptr, const uint8_t* pa = nullptr) {
    LinSeg s;
    s.ptr = p;
    s.gather = gather;
    s.ld = ld;
    s.width = width;
    s.row_div = 1;
    s.pa = pa;
    return s;
}

static int row_tile_for(int rows) {
    const int nrt = (rows + kMaxRowTile - 1) / kMaxRowTile;
    const int per = (rows + nrt - 1) / nrt;
    return ((per + 15) / 16) * 16;
}

static bool stream_capturing(cudaStream_t st) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) return false;
    return cs != cudaStreamCaptureStatusNone;
}

static int plan(sat_handle* h, Layer& ly, LinProblem& P, std::initializer_list<LinSeg> segs, int rows, int epi,
                float* out, int ldo, cudaStream_t st, int force_splits = 0, int group = 1) {
    memset(&P, 0, sizeof(P));
    int k = 0, ns = 0;
    for (const LinSeg& s : segs) {
        if (s.width % 8 || s.ld % 4) return fail(SAT_ERR_UNSUPPORTED, "%s: segment width/ld alignment", ly.name.c_str());
        P.seg[ns++] = s;
        k += s.width;
    }
    if (k != ly.K) return fail(SAT_ERR_INVALID, "%s: operand width %d != %d", ly.name.c_str(), k, ly.K);
    P.nseg = ns;
    P.K = ly.K;
    P.k_blocks = ly.k_blocks;
    P.rows = rows;
    P.row_tile = row_tile_for(rows);
    P.n_row_tiles = (rows + P.row_tile - 1) / P.row_tile;
    P.n_out = ly.n_out;
    P.n_tiles = ly.n_tiles;
    P.wpack = ly.wpack;
    P.bias = ly.bias;
    P.epi = epi;
    P.out = out;
    P.ldo = ldo;
    // L2 policy of the weights: evict_first where one CTA row reads each weight tile once per launch (the decode step
    // at batch <= 128).  A step reads ~137 MB at workload 2 through a 50 MB L2, so no weight survives to the next
    // step, and weights marked evict_last only displace other data: on an H100 the workload-2 loop runs 8 % faster with
    // its weights evict_first than evict_last (tools/l2_sweep.py), and an experiment that kept a 16 to 40 MB prefix of
    // the LSTM / fc_1b / fc_1 / vocabulary weights evict_last was slower than keeping none.  With more than one row
    // tile, several CTAs read each weight tile in the same launch and L2 serves all but the first: evict_last.
    P.l2_w = P.n_row_tiles > 1 ? 2 : 1;
    // split-K: fill the SMs; cost model in units of K-blocks (fixed per-CTA overhead ~4)
    const int tiles = P.n_tiles * P.n_row_tiles;
    // split-K: the `splits` CTAs of a tile form one thread-block cluster (partials meet in DSMEM), so the
    // factor is a portable cluster size.  Cost model in units of K blocks: a CTA costs its K range plus a
    // fixed ~4 blocks (pipeline fill + epilogue); a split adds a cluster barrier.
    const int budget = h->num_sms / (group > 0 ? group : 1);
    int best = 1;
    if (force_splits > 0) {
        best = 1;
        while (best * 2 <= force_splits && best * 2 <= 8 && best * 2 <= P.k_blocks) best *= 2;
    } else {
        double bc = 1e30;
        for (int s = 1; s <= 8 && s <= P.k_blocks; s *= 2) {
            const int waves = (tiles * s + budget - 1) / budget;
            const double c = waves * ((P.k_blocks + s - 1) / s + 4.0) + (s > 1 ? 1.0 : 0.0);
            if (c < bc - 1e-9) { bc = c; best = s; }
        }
    }
    P.splits = best;
    P.cta_count = tiles * best;
    // packed-activation scratch for the cooperative pre-pass (used when the launch fits one wave)
    const size_t xneed = (size_t)P.n_row_tiles * P.k_blocks * 2 * P.row_tile * kBK * 2;
    if (xneed > ly.xpack_bytes || !ly.xbar) {
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "%s: scratch growth during graph capture", ly.name.c_str());
        CK(cudaDeviceSynchronize());
        drop_graphs(h);   // captured graphs hold the buffer freed below
        cudaFree(ly.xpack);
        ly.xpack = nullptr;
        ly.xpack_bytes = 0;
        RET(dmalloc(&ly.xpack, xneed));
        ly.xpack_bytes = xneed;
        if (!ly.xbar) {
            RET(dmalloc(&ly.xbar, (size_t)2));
            CK(cudaMemset(ly.xbar, 0, 2 * sizeof(unsigned)));
        }
    }
    P.xpack = ly.xpack;
    P.xbar = ly.xbar;
    return SAT_OK;
}

static int launch(sat_handle* h, LinProblem* probs, int n, cudaStream_t st) {
    LinLaunch L;
    memset(&L, 0, sizeof(L));
    int begin = 0, max_rt = 16;
    int smin = probs[0].splits;
    for (int i = 1; i < n; ++i) smin = probs[i].splits < smin ? probs[i].splits : smin;
    for (int i = 0; i < n; ++i) {   // one cluster shape per launch: grouped problems share the split factor
        probs[i].splits = smin;
        probs[i].cta_count = probs[i].n_tiles * probs[i].n_row_tiles * smin;
    }
    for (int i = 0; i < n; ++i) {
        L.p[i] = probs[i];
        L.p[i].cta_begin = begin;
        begin += probs[i].cta_count;
        if (probs[i].row_tile > max_rt) max_rt = probs[i].row_tile;
    }
    L.nprob = n;
    L.layout_mode = h->opt_layout;
    L.stages = lin_pick_stages(max_rt);
    if (h->opt_stages > 0 && h->opt_stages < L.stages) L.stages = h->opt_stages;   // experiment knob: shallower pipeline
    // options "l2_w" / "l2_vocab" (vocabulary layer), when set, replace the policy chosen by plan() / sat_dense_packed
    const int l2w = (h->cur_tag == kTagDec2 && h->opt_l2_vocab >= 0) ? h->opt_l2_vocab : h->opt_l2_w;
    if (l2w >= 0)
        for (int i = 0; i < n; ++i) L.p[i].l2_w = l2w;
    L.dbg = nullptr;
    L.tl = nullptr;
    L.warm_epilogue = h->opt_warm;
    L.l2_prefetch = h->opt_l2_prefetch;
    L.w_dynamic = h->lin_w_dynamic ? 1 : 0;
    h->lin_w_dynamic = false;
    if (h->opt_trace == 1 && begin <= 1024 && h->trace_at-- == 0) L.dbg = h->trace;
    if (h->opt_trace == 3 && h->tl_count < 4000) {
        L.tl = h->trace + 4 * h->tl_count++;
        h->tl_names.push_back(std::string(kTagNames[h->cur_tag]) + "/" + std::to_string(begin));
    }
    bool all_pa = true;
    for (int i = 0; i < n; ++i)
        for (int sgi = 0; sgi < probs[i].nseg; ++sgi) all_pa = all_pa && probs[i].seg[sgi].pa != nullptr;
    if (all_pa) L.x_mode = 2;   // operands were packed by their producers: nothing to convert, nothing to wait for
    else L.x_mode = (h->opt_xpack && smin == 1 && begin <= h->num_sms) ? 1 : 0;  // pre-pass: grid barrier, no clusters
    L.pdl = (h->opt_pdl && L.x_mode != 1) ? 1 : 0;   // (the cooperative pre-pass launch keeps full serialization)
    if (L.stages < 1) return fail(SAT_ERR_UNSUPPORTED, "row tile %d does not fit in shared memory", max_rt);
    {
        ProfScope ps(h, h->cur_tag, st);
        CK(lin_launch(L, st, h->opt_gemm == 0));
    }
    h->launches += 1;
    return SAT_OK;
}

// Dense product on the wgmma kernel from operands that are ALREADY in the packed layouts (training path,
// sat_train.cu): out[rows, n_out] (+)= X * W with X a packed activation of row tile `row_tile` and W a packed weight.
int sat_handle_layout_mode(sat_handle* h) { return h->opt_layout; }
int sat_handle_train_tc(sat_handle* h) { return h->opt_train_tc && h->opt_gemm != 0; }

int sat_dense_packed(sat_handle* h, const uint8_t* x_pa, int rows, int row_tile, int K, const uint8_t* wpack,
                     const float* bias_packed, int n_out, int epi, float* out, int ldo, int accumulate, int splits,
                     void* stream, int weights_dynamic) {
    if (!h || !x_pa || !wpack || !out) return fail(SAT_ERR_INVALID, "sat_dense_packed: null argument");
    if (K % kBK || row_tile % 16 || row_tile > kMaxRowTile || splits < 1 || splits > 8 || (splits & (splits - 1)))
        return fail(SAT_ERR_INVALID, "sat_dense_packed: K %d / row tile %d / splits %d", K, row_tile, splits);
    LinProblem P;
    memset(&P, 0, sizeof(P));
    P.seg[0].pa = x_pa;
    P.seg[0].width = K;
    P.seg[0].ld = K;
    P.seg[0].row_div = 1;
    P.nseg = 1;
    P.K = K;
    P.k_blocks = K / kBK;
    while (splits > 1 && splits > P.k_blocks) splits >>= 1;   // every CTA of a split needs at least one K block
    P.rows = rows;
    P.row_tile = row_tile;
    P.n_row_tiles = (rows + row_tile - 1) / row_tile;
    P.n_out = n_out;
    P.n_tiles = (n_out + kTileN - 1) / kTileN;
    P.splits = splits;
    P.cta_count = P.n_tiles * P.n_row_tiles * splits;
    P.wpack = wpack;
    P.l2_w = 2;   // (training: every weight stream evict_last)
    P.bias = bias_packed;
    P.epi = epi;
    P.out = out;
    P.ldo = ldo;
    P.accumulate = accumulate;
    h->cur_tag = kTagProj;
    h->lin_w_dynamic = weights_dynamic != 0;
    return launch(h, &P, 1, (cudaStream_t)stream);
}

// --------------------------------------------------------------- contexts
// attend fc_1a over every location (model.py:417-420): T1 = tanh(ctx2d * W1a + b1a)
// mean_done (optional): the caller also wants the mean over the L locations (initialize); set to true if the packing
// pass produced it on the way (one pass over the conv features for both, SURVEY section 8 row f3)
static int project_contexts(sat_handle* h, const float* ctx, int n_img, cudaStream_t st, bool* mean_done = nullptr) {
    if (h->d.num_attend_layers != 2) return SAT_OK;
    h->cur_tag = kTagProj;
    LinProblem P;
    RET(plan(h, h->att_1a, P, {seg(ctx, h->d.dim_ctx, h->d.dim_ctx)}, n_img * h->d.num_ctx, kEpiBiasTanh, h->T1,
             h->d.dim_attend_layer, st));
    if (h->opt_gemm != 0 && h->opt_pa && (h->d.dim_ctx % 64) == 0) {
        // thousands of rows: converting them inside the GEMM's producer warps is latency bound, so the
        // contexts are packed once by a streaming kernel and the GEMM fetches them by TMA
        if (mean_done && h->opt_prologue1 && (h->d.dim_ctx % 128) == 0) {
            CK(ctx_mean_pack_launch(ctx, h->mean, P.xpack, P.row_tile, h->opt_layout, n_img, h->d.num_ctx, h->d.dim_ctx, st));
            *mean_done = true;
        } else {
            PackJob job{ctx, nullptr, h->d.dim_ctx, h->d.dim_ctx, P.rows, P.row_tile, P.xpack};
            CK(pack_rows_launch(&job, 1, h->opt_layout, st));
        }
        h->launches += 1;
        P.seg[0].pa = P.xpack;
    }
    return launch(h, &P, 1, st);
}

// initialize (model.py:239-242, 358-393)
static int run_initialize(sat_handle* h, const float* ctx, int n_img, float* c0, float* h0, cudaStream_t st,
                          uint8_t* h0_pa = nullptr, bool mean_ready = false) {
    const sat_dims& d = h->d;
    h->cur_tag = kTagInit;
    if (!mean_ready) {
        CK(ctx_mean_launch(ctx, h->mean, n_img, d.num_ctx, d.dim_ctx, st));
        h->launches += 1;
    }
    LinProblem P[2];
    if (d.num_initalize_layers == 1) {
        RET(plan(h, h->init_a1, P[0], {seg(h->mean, d.dim_ctx, d.dim_ctx)}, n_img, kEpiBias, c0, d.num_lstm_units, st, 0, 2));
        RET(plan(h, h->init_b1, P[1], {seg(h->mean, d.dim_ctx, d.dim_ctx)}, n_img, kEpiBias, h0, d.num_lstm_units, st, 0, 2));
        P[1].out_pa = h0_pa;
        return launch(h, P, 2, st);
    }
    const int I = d.dim_initalize_layer;
    RET(plan(h, h->init_a1, P[0], {seg(h->mean, d.dim_ctx, d.dim_ctx)}, n_img, kEpiBiasTanh, h->tmp_a, I, st, 0, 2));
    RET(plan(h, h->init_b1, P[1], {seg(h->mean, d.dim_ctx, d.dim_ctx)}, n_img, kEpiBiasTanh, h->tmp_b, I, st, 0, 2));
    RET(launch(h, P, 2, st));
    RET(plan(h, h->init_a2, P[0], {seg(h->tmp_a, I, I)}, n_img, kEpiBias, c0, d.num_lstm_units, st, 0, 2));
    RET(plan(h, h->init_b2, P[1], {seg(h->tmp_b, I, I)}, n_img, kEpiBias, h0, d.num_lstm_units, st, 0, 2));
    P[1].out_pa = h0_pa;
    return launch(h, P, 2, st);
}

static int prepare_impl(sat_handle* h, const float* ctx, int n_img, float* c0, float* h0, cudaStream_t st,
                        uint8_t* h0_pa = nullptr) {
    if (n_img < 1 || n_img > h->max_rows) return fail(SAT_ERR_INVALID, "n_img %d outside [1, %d]", n_img, h->max_rows);
    // the mean of the contexts first: the projection and the initialize layers are then consecutive dense
    // launches, chained by programmatic dependent launch instead of separated by a fully serialised small kernel
    const bool want_init = c0 && h0;
    // one pass over the conv features for the mean and the projection operand when the projection runs from packed rows
    const bool one_pass = want_init && h->opt_hoist && h->opt_prologue1 && h->d.num_attend_layers == 2 && h->opt_gemm != 0 &&
                          h->opt_pa && (h->d.dim_ctx % 128) == 0;
    bool mean_done = false;
    if (want_init && !one_pass) {
        CK(ctx_mean_launch(ctx, h->mean, n_img, h->d.num_ctx, h->d.dim_ctx, st));
        h->launches += 1;
        mean_done = true;
    }
    if (h->opt_hoist) {
        RET(project_contexts(h, ctx, n_img, st, one_pass ? &mean_done : nullptr));
        h->prep_ctx = ctx;
        h->prep_ni = n_img;
    }
    if (want_init) RET(run_initialize(h, ctx, n_img, c0, h0, st, h0_pa, mean_done));
    return SAT_OK;
}

extern "C" int sat_prepare_contexts(sat_handle* h, const float* contexts, int32_t n_img, float* initial_memory,
                                    float* initial_output, void* stream) {
    RET(require_ready(h));
    if (!contexts) return fail(SAT_ERR_INVALID, "contexts is null");
    if ((initial_memory == nullptr) != (initial_output == nullptr))
        return fail(SAT_ERR_INVALID, "initial_memory and initial_output must both be given or both be null");
    return prepare_impl(h, contexts, n_img, initial_memory, initial_output, (cudaStream_t)stream);
}

// ------------------------------------------------------------------- step
struct StepIO {
    const float* ctx;
    int n_img, group;
    const int32_t* last_word;
    const float *c_in, *h_in;
    float *c_out, *h_out, *logits, *probs, *alpha;
    RowsParams rows;  // softmax-stage extras (tokens / next_word / topk); logits/probs/V filled here
    bool want_rows;
    bool q_ready;      // the state branch q for this step was produced by the previous step's grouped launch
    bool make_next_q;  // also compute q of the NEXT step (from this step's output) alongside decode fc_1
    int pa_slot;       // packed h of this step's input lives in pa_h[pa_slot], the output goes to pa_h[pa_slot ^ 1]
    bool pa_h_valid;   // pa_h[pa_slot] was written by the producer of h_in (initialize / previous LSTM)
    bool pa_emb_valid; // pa_emb holds the embedding rows of last_word (previous step's fused argmax)
};

// state branch of attend: q = tanh(h*W1b + b1b) (model.py:421-424) or, 1-layer, h*fc_b (model.py:409-413)
static int plan_att_state(sat_handle* h, LinProblem& P, const float* h_in, int rows, cudaStream_t st, int group,
                          const uint8_t* h_pa = nullptr) {
    const sat_dims& d = h->d;
    if (d.num_attend_layers == 2)
        return plan(h, h->att_1b, P, {seg(h_in, d.num_lstm_units, d.num_lstm_units, nullptr, h_pa)}, rows, kEpiBiasTanh,
                    h->q, d.dim_attend_layer, st, 0, group);
    return plan(h, h->att_1b, P, {seg(h_in, d.num_lstm_units, d.num_lstm_units, nullptr, h_pa)}, rows, kEpiNone, h->q,
                d.num_ctx, st, 0, group);
}

static int attention_impl(sat_handle* h, const float* ctx, int n_img, int G, const float* h_in, float* alpha, float* z,
                          cudaStream_t st, bool q_ready = false, const int32_t* last_word = nullptr, int sm_budget = 0,
                          bool nowait = false) {
    const sat_dims& d = h->d;
    const int rows = n_img * G;
    AttParams ap;
    memset(&ap, 0, sizeof(ap));
    LinProblem P;
    if (d.num_attend_layers == 2) {
        if (!(h->opt_hoist && h->prep_ctx == ctx && h->prep_ni == n_img)) RET(project_contexts(h, ctx, n_img, st));
        h->cur_tag = kTagAttState;
        if (!q_ready) {
            RET(plan_att_state(h, P, h_in, rows, st, 1, h->pa_on ? h->pa_cur_h_in : nullptr));
            RET(launch(h, &P, 1, st));
        }
        ap.T = h->T1;
        ap.RL = d.dim_attend_layer;
        ap.q = h->q;
        ap.eadd = nullptr;
    } else {
        // logits2 = h * fc_b   (model.py:409-413), added to ctx . fc_a inside the kernel
        h->cur_tag = kTagAttState;
        if (!q_ready) {
            RET(plan_att_state(h, P, h_in, rows, st, 1, h->pa_on ? h->pa_cur_h_in : nullptr));
            RET(launch(h, &P, 1, st));
        }
        ap.T = ctx;
        ap.RL = d.dim_ctx;
        ap.q = nullptr;
        ap.eadd = h->q;
    }
    ap.vec = h->att_vec.dev;
    ap.ctx = ctx;
    ap.e = h->e;
    ap.rowcnt = h->rowcnt;
    ap.alpha = alpha ? alpha : h->alpha;
    ap.z = z;
    ap.NI = n_img;
    ap.G = G;
    ap.L = d.num_ctx;
    ap.D = d.dim_ctx;
    ap.l2_t = h->opt_l2_t;
    ap.l2_ctx = h->opt_l2_ctx;
    ap.occ = h->opt_att_occ;
    ap.warps = h->opt_att_warps;
    ap.wpc = h->opt_att_wpc;
    if (sm_budget <= 0 && h->opt_att_sms > 0) sm_budget = h->opt_att_sms;   // experiment knob
    if (!att_plan(ap, h->smem_optin, sm_budget > 0 ? sm_budget : h->num_sms))
        return fail(SAT_ERR_UNSUPPORTED, "attention shape unsupported (G=%d L=%d D=%d)", G, ap.L, ap.D);
    if (nowait && (!ap.wpc || (h->att_qflag && n_img > ap.grid))) {
        // running beside the predecessor only works when the kernel can skip the wait (warp-per-chunk kernel).  On
        // fewer SMs than images CTA row ranges cross image boundaries, which the decode loop's attention takes (on
        // an H100 the vocabulary layer leaves 53 SMs for 64 images); the chained launch wants one CTA per image.
        // Otherwise: whole GPU, in order
        nowait = false;
        ap.occ = h->opt_att_occ;
        ap.warps = h->opt_att_warps;
        ap.wpc = h->opt_att_wpc;
        if (!att_plan(ap, h->smem_optin, h->opt_att_sms > 0 ? h->opt_att_sms : h->num_sms))
            return fail(SAT_ERR_UNSUPPORTED, "attention shape unsupported (G=%d L=%d D=%d)", G, ap.L, ap.D);
    }
    const size_t pneed = att_part_floats(ap);
    if (pneed > h->att_part_floats) {
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "attention scratch growth during graph capture");
        CK(cudaDeviceSynchronize());
        drop_graphs(h);   // captured graphs hold the buffer freed below
        cudaFree(h->att_part);
        h->att_part = nullptr;
        h->att_part_floats = 0;
        RET(dmalloc(&h->att_part, pneed));
        h->att_part_floats = pneed;
    }
    ap.part = h->att_part;
    if (h->pa_on) {
        ap.pa_z = h->pa_cur_z ? h->pa_cur_z : h->pa_z;
        ap.pa_row_tile = row_tile_for(rows);
        ap.pa_mode = h->opt_layout;
        if (last_word) {   // the embedding rows of this step's words are packed on the side
            ap.emb = h->embedding;
            ap.emb_word = last_word;
            ap.emb_pa = h->pa_emb;
            ap.emb_E = h->d.dim_embedding;
        }
    }
    ap.pdl = h->opt_pdl ? 1 : 0;
    ap.nowait = (nowait && ap.pdl) ? 1 : 0;
    if (h->att_qflag) {
        if (!ap.nowait || !ap.wpc) return fail(SAT_ERR_STATE, "attention beside a chained launch needs the warp-per-chunk kernel");
        ap.qflag = h->att_qflag;
        ap.qtarget = h->att_qtarget;
    }
    if (q_ready && !h->opt_att_reuse_q) {
        h->att_loop_grid = ap.grid;
        h->att_loop_beside = ap.nowait;
    }
    ap.dbg = h->opt_trace == 2 ? h->trace : nullptr;
    ap.tl = nullptr;
    if (h->opt_trace == 3 && h->tl_count < 4000) {
        ap.tl = h->trace + 4 * h->tl_count++;
        h->tl_names.push_back("attention/" + std::to_string(ap.grid));
    }
    {
        ProfScope ps(h, kTagAtt, st);
        CK(att_launch(ap, st));
    }
    h->launches += 1;
    return SAT_OK;
}

static int lstm_impl(sat_handle* h, const float* z, const int32_t* last_word, const float* c_in, const float* h_in,
                     float* c_out, float* h_out, int rows, cudaStream_t st) {
    const sat_dims& d = h->d;
    h->cur_tag = kTagLstm;
    LinProblem P;
    // current_input = concat([context, word_embed]) (model.py:277); LSTMCell concat([x, h]) (TF)
    const bool pa = h->pa_on;
    RET(plan(h, h->lstm, P,
             {seg(z, d.dim_ctx, d.dim_ctx, nullptr, pa ? (h->pa_cur_z ? h->pa_cur_z : h->pa_z) : nullptr),
              seg(h->embedding, d.dim_embedding, d.dim_embedding, last_word, pa ? h->pa_emb : nullptr),
              seg(h_in, d.num_lstm_units, d.num_lstm_units, nullptr, pa ? h->pa_cur_h_in : nullptr)},
             rows, kEpiLstm, nullptr, 0, st));
    P.out_pa = pa ? h->pa_cur_h_out : nullptr;
    P.c_in = c_in;
    P.c_out = c_out;
    P.h_out = h_out;
    P.H = d.num_lstm_units;
    return launch(h, &P, 1, st);
}

// fused greedy argmax on the vocabulary layer: only when it runs un-split in one wave
static int attach_argmax(sat_handle* h, Layer& ly, LinProblem& P, const RowsParams* am, cudaStream_t st) {
    // (its tail is a grid barrier: every CTA of the layer must be resident at once)
    if (!am || P.splits != 1 || h->opt_gemm == 0 || P.n_tiles * P.n_row_tiles > h->num_sms) return 0;
    const size_t need = (size_t)P.n_row_tiles * P.n_tiles * P.row_tile;
    if (need > ly.am_n) {
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "%s: scratch growth during graph capture", ly.name.c_str());
        CK(cudaDeviceSynchronize());
        drop_graphs(h);   // captured graphs hold the buffer freed below
        cudaFree(ly.am_key);
        ly.am_key = nullptr; ly.am_n = 0;
        RET(dmalloc(&ly.am_key, need));
        ly.am_n = need;
        if (!ly.am_ctr) {
            RET(dmalloc(&ly.am_ctr, (size_t)2));   // {arrival counter, generation of "words picked"}
            CK(cudaMemset(ly.am_ctr, 0, 2 * sizeof(unsigned)));
        }
    }
    if (am->word_probs && ly.am_sum_n < ly.am_n) {   // (only handles that ask for word probabilities)
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "%s: scratch growth during graph capture", ly.name.c_str());
        CK(cudaDeviceSynchronize());
        drop_graphs(h);   // captured graphs hold the buffer freed below
        cudaFree(ly.am_sum);
        cudaFree(ly.am_wlogit);
        ly.am_sum = ly.am_wlogit = nullptr; ly.am_sum_n = 0;
        RET(dmalloc(&ly.am_sum, ly.am_n));
        RET(dmalloc(&ly.am_wlogit, (size_t)h->max_rows));
        ly.am_sum_n = ly.am_n;
    }
    if (am->sample && am->word_probs && ly.am_smp_n < ly.am_n) {   // (only handles that sample with word probabilities)
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "%s: scratch growth during graph capture", ly.name.c_str());
        CK(cudaDeviceSynchronize());
        drop_graphs(h);   // captured graphs hold the buffer freed below
        cudaFree(ly.am_smp);
        ly.am_smp = nullptr; ly.am_smp_n = 0;
        RET(dmalloc(&ly.am_smp, ly.am_n));
        ly.am_smp_n = ly.am_n;
    }
    P.am_key = ly.am_key; P.am_ctr = ly.am_ctr;
    P.am_tokens = am->tokens; P.am_tokens_ld = am->tokens_ld; P.am_step = am->step;
    P.am_next_word = am->next_word; P.am_forced = am->forced; P.am_forced_ld = am->forced_ld;
    if (am->word_probs) {
        P.am_probs = am->word_probs; P.am_probs_ld = am->tokens_ld;
        P.am_sum = ly.am_sum; P.am_wlogit = ly.am_wlogit;
    }
    if (am->sample) {   // without word probabilities the sampling instance keeps no softmax partials
        P.smp = am->sample;
        if (am->word_probs) P.am_smp = ly.am_smp;
    }
    return 1;
}

// returns 1 in *argmax_done if the prediction / next word were produced by the vocabulary layer itself
static int decode_impl(sat_handle* h, const float* h_out, const float* z, const int32_t* last_word, float* logits,
                       int rows, cudaStream_t st, bool make_next_q = false, const RowsParams* am = nullptr,
                       int* argmax_done = nullptr, int phase = 0, bool pack_next_emb = false) {
    const sat_dims& d = h->d;
    LinProblem P[2];
    int used = 0;
    if (argmax_done) *argmax_done = 0;
    // expanded_output = concat([output, context, word_embed]) (model.py:283-286)
    h->cur_tag = kTagDec1;
    if (d.num_decode_layers == 2) {
        const int group = make_next_q ? 2 : 1;
        const bool pa = h->pa_on;
        if (phase != 2) {
        RET(plan(h, h->dec_1, P[0],
                 {seg(h_out, d.num_lstm_units, d.num_lstm_units, nullptr, pa ? h->pa_cur_h_out : nullptr),
                  seg(z, d.dim_ctx, d.dim_ctx, nullptr, pa ? (h->pa_cur_z ? h->pa_cur_z : h->pa_z) : nullptr),
                  seg(h->embedding, d.dim_embedding, d.dim_embedding, last_word, pa ? h->pa_emb : nullptr)},
                 rows, kEpiBiasTanh, h->t_dec, d.dim_decode_layer, st, h->opt_dec1_splits, group));
        P[0].out_pa = pa ? h->pa_t : nullptr;
        int np = 1;
        if (make_next_q) {  // q of the next step depends on the same h_out: share the launch
            RET(plan_att_state(h, P[1], h_out, rows, st, 2, pa ? h->pa_cur_h_out : nullptr));
            np = 2;
        }
        RET(launch(h, P, np, st));
        }
        if (phase == 1) return SAT_OK;
        h->cur_tag = kTagDec2;
        RET(plan(h, h->dec_2, P[0], {seg(h->t_dec, d.dim_decode_layer, d.dim_decode_layer, nullptr, pa ? h->pa_t : nullptr)},
                 rows, kEpiBias, logits, d.vocabulary_size, st, am ? 1 : 0));   // the fused argmax needs whole rows per CTA
        used = attach_argmax(h, h->dec_2, P[0], am, st);
        if (used < 0) return used;
        if (used && logits == h->logits) P[0].out = nullptr;   // nobody asked for the logits: only the word is kept
        // the embedding row of the chosen word is normally packed by the next step's attention kernel; when
        // that kernel runs CONCURRENTLY with this layer (decode loop), the last CTA of this layer does it
        if (used && pa && pack_next_emb) {
            P[0].am_emb = h->embedding;
            P[0].am_E = d.dim_embedding;
            P[0].am_emb_pa = h->pa_emb;
        }
        RET(launch(h, P, 1, st));
        if (argmax_done) *argmax_done = used;
        return SAT_OK;
    }
    h->cur_tag = kTagDec2;
    const int group = make_next_q ? 2 : 1;
    const bool pa = h->pa_on;
    RET(plan(h, h->dec_2, P[0],
             {seg(h_out, d.num_lstm_units, d.num_lstm_units, nullptr, pa ? h->pa_cur_h_out : nullptr),
              seg(z, d.dim_ctx, d.dim_ctx, nullptr, pa ? (h->pa_cur_z ? h->pa_cur_z : h->pa_z) : nullptr),
              seg(h->embedding, d.dim_embedding, d.dim_embedding, last_word, pa ? h->pa_emb : nullptr)},
             rows, kEpiBias, logits, d.vocabulary_size, st, 0, group));
    int np = 1;
    if (make_next_q) {
        RET(plan_att_state(h, P[1], h_out, rows, st, 2, pa ? h->pa_cur_h_out : nullptr));
        np = 2;
    }
    // the fused argmax overwrites next_word, which this very launch still gathers embeddings with:
    // only safe when the embedding rows are not an operand of the vocabulary layer (2-layer decode)
    RET(launch(h, P, np, st));
    return SAT_OK;
}

static int step_impl(sat_handle* h, StepIO& io, cudaStream_t st) {
    const int rows = io.n_img * io.group;
    if (rows > h->max_rows) return fail(SAT_ERR_INVALID, "rows %d > max_batch %d", rows, h->max_rows);
    h->pa_on = h->pa_ok && h->opt_pa && h->opt_gemm != 0;
    if (h->pa_on) {
        h->pa_cur_h_in = h->pa_h[io.pa_slot & 1];
        h->pa_cur_h_out = h->pa_h[(io.pa_slot & 1) ^ 1];
        h->pa_cur_z = h->pa_z;
        PackJob jobs[2];
        int nj = 0;
        const int rtile = row_tile_for(rows);
        if (!io.pa_h_valid) jobs[nj++] = PackJob{io.h_in, nullptr, h->d.num_lstm_units, h->d.num_lstm_units, rows, rtile, h->pa_cur_h_in};
        if (nj) {
            CK(pack_rows_launch(jobs, nj, h->opt_layout, st));
            h->launches += 1;
        }
    }
    RET(attention_impl(h, io.ctx, io.n_img, io.group, io.h_in, io.alpha, h->z, st, io.q_ready, io.last_word));
    RET(lstm_impl(h, h->z, io.last_word, io.c_in, io.h_in, io.c_out, io.h_out, rows, st));
    float* logits = io.logits ? io.logits : h->logits;
    // (a filtered draw needs the row's logits: the per-row kernel makes it after the vocabulary layer)
    const bool argmax_only = io.want_rows && !io.probs && io.rows.topk == 0 && !io.rows.argmax && !io.rows.filter;
    int fused = 0;
    RET(decode_impl(h, io.h_out, h->z, io.last_word, logits, rows, st, io.make_next_q,
                    argmax_only ? &io.rows : nullptr, &fused));
    if ((io.probs || io.want_rows) && !fused) {
        RowsParams rp = io.rows;
        rp.logits = logits;
        rp.V = h->d.vocabulary_size;
        rp.probs = io.probs;
        if (rp.filter && h->opt_trace == 3 && h->tl_count < 4000) {
            rp.tl = h->trace + 4 * h->tl_count++;
            h->tl_names.push_back("filter/" + std::to_string(rows));
        }
        {
            ProfScope ps(h, kTagRows, st);
            CK(rows_softmax_launch(rp, rows, st));
        }
        h->launches += 1;
    }
    io.pa_emb_valid = h->pa_on && fused != 0;   // tells the caller whether the next step's embedding is packed
    h->pa_on = false;
    return SAT_OK;
}

extern "C" int sat_decode_step(sat_handle* h, const float* contexts, const int32_t* last_word,
                               const float* last_memory, const float* last_output, float* memory, float* output,
                               float* logits, float* probs, float* alpha, int32_t B, void* stream) {
    RET(require_ready(h));
    if (!contexts || !last_word || !last_memory || !last_output || !memory || !output)
        return fail(SAT_ERR_INVALID, "sat_decode_step: null tensor");
    if (B < 1 || B > h->max_rows) return fail(SAT_ERR_INVALID, "batch %d outside [1, %d]", B, h->max_rows);
    if (memory == last_memory || output == last_output)
        return fail(SAT_ERR_INVALID, "sat_decode_step: state outputs must not alias the inputs");
    StepIO io;
    memset(&io, 0, sizeof(io));
    io.ctx = contexts; io.n_img = B; io.group = 1; io.last_word = last_word;
    io.c_in = last_memory; io.h_in = last_output; io.c_out = memory; io.h_out = output;
    io.logits = logits; io.probs = probs; io.alpha = alpha;
    return step_impl(h, io, (cudaStream_t)stream);
}

// ------------------------------------------------------------ CUDA graphs
// host-side record of which contexts the hoisted projection T1 currently holds (nullptr: none / unknown)
static void note_projected(sat_handle* h, const float* ctx, int n_img) {
    if (ctx && h->opt_hoist && h->d.num_attend_layers == 2) { h->prep_ctx = ctx; h->prep_ni = n_img; }
    else { h->prep_ctx = nullptr; h->prep_ni = 0; }
}

template <typename F>
static int run_graphed(sat_handle* h, const std::vector<long long>& key, cudaStream_t st, F&& enqueue) {
    if (!h->opt_graphs || st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread) return enqueue();
    GraphEntry* ent = nullptr;
    for (auto& g : h->graphs)
        if (g.key == key) ent = &g;
    if (!ent) {
        if (h->graphs.size() >= 48) {
            if (h->graphs.front().exec) cudaGraphExecDestroy(h->graphs.front().exec);
            h->graphs.erase(h->graphs.begin());
        }
        h->graphs.push_back(GraphEntry());
        ent = &h->graphs.back();
        ent->key = key;
    }
    if (ent->exec) {
        CK(cudaGraphLaunch(ent->exec, st));
        h->launches += ent->kernels;
        return SAT_OK;
    }
    if (ent->seen == 0) {  // first use: run eagerly so that every workspace exists
        ent->seen = 1;
        return enqueue();
    }
    // contexts-dependent caches are part of the key, so replays stay valid
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const long long before = h->launches;
    int rc = enqueue();
    ent->kernels = h->launches - before;
    h->launches = before;
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc != SAT_OK) {
        if (graph) cudaGraphDestroy(graph);
        return rc;
    }
    if (ce != cudaSuccess) return fail(SAT_ERR_CUDA, "stream capture failed: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&ent->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) {
        ent->exec = nullptr;
        return fail(SAT_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
    }
    CK(cudaGraphLaunch(ent->exec, st));
    h->launches += ent->kernels;
    return SAT_OK;
}

// ------------------------------------------------------------------- loop
// Decode loop with the attention of step t+1 (needs only q(t+1) = f(h_t)) running CONCURRENTLY with the
// vocabulary layer of step t (needs only t_dec(t)); they join before the LSTM of step t+1, which consumes the
// context vector of the one and the chosen word of the other.
// alphas [T,B,L] / word_probs [B,T] (may be null): the per-word maps of sat_decode_loop_maps
static float* step_alpha(float* alphas, int t, int B, int L) { return alphas ? alphas + (size_t)t * B * L : nullptr; }

// Prologue of a loop over B = n_img x G rows: project the contexts and run initialize once per image; with G > 1
// (several sampled captions per image) every row then gets its image's initial state, and the packed h0 is built for the
// row tile of B rows.
static int loop_prologue(sat_handle* h, const float* ctx, int B, int G, cudaStream_t st, uint8_t* h0_pa) {
    if (G == 1) return prepare_impl(h, ctx, B, h->st_c[0], h->st_h[0], st, h0_pa);
    const int H = h->d.num_lstm_units;
    RET(prepare_impl(h, ctx, B / G, h->st_c[1], h->st_h[1], st));   // (slot 1 is free until step 0 writes it)
    CK(bcast_state_launch(h->st_c[1], h->st_h[1], h->st_c[0], h->st_h[0], B, G, H, st));
    h->launches += 1;
    if (h0_pa) {
        PackJob job{h->st_h[0], nullptr, H, H, B, row_tile_for(B), h0_pa};
        CK(pack_rows_launch(&job, 1, h->opt_layout, st));
        h->launches += 1;
    }
    return SAT_OK;
}

// G: rows per image (sampling: captions per image; the attention kernels share an image's contexts between them);
// smp: the sampling loop's {seed, 1 / temperature} (null: greedy / teacher forced)
static int loop_enqueue_overlap(sat_handle* h, const float* ctx, int B, int T, const int32_t* forced, int32_t* tokens,
                                float* logits_all, float* alphas, float* word_probs, cudaStream_t st, int G = 1,
                                const SampleParams* smp = nullptr) {
    if (!h->side) {
        CK(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
    }
    const sat_dims& d = h->d;
    RET(loop_prologue(h, ctx, B, G, st, h->pa_h[0]));
    CK(cudaMemsetAsync(h->word, 0, (size_t)B * sizeof(int32_t), st));  // <start> = 0 (model.py:254)
    for (int t = 0; t < T; ++t) {
        const float *c_in = h->st_c[t & 1], *h_in = h->st_h[t & 1];
        float *c_out = h->st_c[(t + 1) & 1], *h_out = h->st_h[(t + 1) & 1];
        h->pa_on = true;
        h->pa_cur_h_in = h->pa_h[t & 1];
        h->pa_cur_h_out = h->pa_h[(t + 1) & 1];
        float* zcur = h->z2[t & 1];          // context vector of this step (fp32 + packed), written by attention(t)
        h->pa_cur_z = h->pa_z2[t & 1];
        if (t == 0)   // q(0), attention(0) and the embedding of <start>
            RET(attention_impl(h, ctx, B / G, G, h_in, step_alpha(alphas, 0, B, d.num_ctx), zcur, st, false, h->word));
        RET(lstm_impl(h, zcur, h->word, c_in, h_in, c_out, h_out, B, st));
        float* logits = logits_all ? logits_all + (size_t)t * B * d.vocabulary_size : h->logits;
        if (t + 1 < T) {
            // fork right after the LSTM: the side stream computes q(t+1) = f(h_t) and then attention(t+1) while
            // this stream runs decode fc_1 and the vocabulary layer of step t
            CK(cudaEventRecord(h->ev_fork, st));
            CK(cudaStreamWaitEvent(h->side, h->ev_fork, 0));
            LinProblem Pq;
            h->cur_tag = kTagAttState;
            RET(plan_att_state(h, Pq, h_out, B, h->side, 1, h->pa_cur_h_out));
            RET(launch(h, &Pq, 1, h->side));
            h->pa_cur_h_in = h->pa_h[(t + 1) & 1];
            h->pa_cur_z = h->pa_z2[(t + 1) & 1];
            // it shares the GPU with decode fc_1 / the vocabulary layer (n_tiles CTAs, one per SM): size it for
            // the SMs left over
            int budget = h->opt_att_sms > 0 ? h->opt_att_sms : h->num_sms - h->dec_2.n_tiles;
            if (budget < h->num_sms / 4) budget = h->num_sms;
            RET(attention_impl(h, ctx, B / G, G, h_out, step_alpha(alphas, t + 1, B, d.num_ctx), h->z2[(t + 1) & 1], h->side,
                               true, nullptr, budget));
            CK(cudaEventRecord(h->ev_join, h->side));
            h->pa_cur_h_in = h->pa_h[t & 1];
            h->pa_cur_z = h->pa_z2[t & 1];
        }
        RET(decode_impl(h, h_out, zcur, h->word, logits, B, st, false, nullptr, nullptr, 1));   // fc_1
        RowsParams rp;
        memset(&rp, 0, sizeof(rp));
        rp.tokens = tokens; rp.tokens_ld = T; rp.step = t;
        rp.next_word = h->word; rp.forced = forced; rp.forced_ld = T; rp.word_probs = word_probs;
        rp.sample = smp;
        int fused = 0;
        RET(decode_impl(h, h_out, zcur, h->word, logits, B, st, false, &rp, &fused, 2, t + 1 < T));  // fc_2 + argmax
        if (!fused) {
            h->pa_on = false;
            return fail(SAT_ERR_STATE, "overlapped loop needs the fused argmax of the vocabulary layer");
        }
        if (t + 1 < T) CK(cudaStreamWaitEvent(st, h->ev_join, 0));   // join before the LSTM of step t+1
    }
    h->pa_on = false;
    h->pa_cur_z = nullptr;
    return SAT_OK;
}

// Single-stream loop built on programmatic dependent launch (option overlap = 2).  Launch order per step:
//   LSTM(t) -> [decode fc_1(t) || q(t+1)] -> vocabulary layer(t) -> attention(t+1)
// The attention kernel of step t+1 needs q(t+1) (two launches back: complete by the time it may start, see
// pdl_wait) and nothing from the vocabulary layer, so it starts on the SMs the vocabulary layer's one-wave
// grid leaves idle and the two run side by side without a second stream; it only waits for its predecessor
// right before it exits, which keeps "kernel k complete => kernel k-1 complete" for the LSTM that follows.
// Its grid is the SMs left over (132 - 79 = 53 on an H100 at V = 10000), also when that is fewer than the images:
// CTA row ranges then cross image boundaries.  It must stay the vocabulary layer's PDL successor on this stream:
// the layer's fused arg-max meets at a grid-wide counter (am_ctr, sat_linear.cu) and so needs all its CTAs
// resident at once; the attention only becomes launchable once every one of them has passed its pdl_wait, so it
// can never take an SM one of them still needs.
static int loop_enqueue_chain(sat_handle* h, const float* ctx, int B, int T, const int32_t* forced, int32_t* tokens,
                              float* logits_all, float* alphas, float* word_probs, cudaStream_t st, bool prepared = false,
                              int G = 1, const SampleParams* smp = nullptr) {
    const sat_dims& d = h->d;
    if (!prepared) RET(loop_prologue(h, ctx, B, G, st, h->pa_h[0]));
    CK(cudaMemsetAsync(h->word, 0, (size_t)B * sizeof(int32_t), st));  // <start> = 0 (model.py:254)
    int budget = h->opt_att_sms > 0 ? h->opt_att_sms : h->num_sms - h->dec_2.n_tiles;
    if (budget < h->num_sms / 4) budget = h->num_sms;
    for (int t = 0; t < T; ++t) {
        const float *c_in = h->st_c[t & 1], *h_in = h->st_h[t & 1];
        float *c_out = h->st_c[(t + 1) & 1], *h_out = h->st_h[(t + 1) & 1];
        h->pa_on = true;
        h->pa_cur_h_in = h->pa_h[t & 1];
        h->pa_cur_h_out = h->pa_h[(t + 1) & 1];
        h->pa_cur_z = h->pa_z;
        if (t == 0)   // q(0), attention(0) and the embedding of <start>
            RET(attention_impl(h, ctx, B / G, G, h_in, step_alpha(alphas, 0, B, d.num_ctx), h->z, st, false, h->word));
        RET(lstm_impl(h, h->z, h->word, c_in, h_in, c_out, h_out, B, st));
        float* logits = logits_all ? logits_all + (size_t)t * B * d.vocabulary_size : h->logits;
        RET(decode_impl(h, h_out, h->z, h->word, logits, B, st, t + 1 < T, nullptr, nullptr, 1));   // fc_1 || q(t+1)
        RowsParams rp;
        memset(&rp, 0, sizeof(rp));
        rp.tokens = tokens; rp.tokens_ld = T; rp.step = t;
        rp.next_word = h->word; rp.forced = forced; rp.forced_ld = T; rp.word_probs = word_probs;
        rp.sample = smp;
        int fused = 0;
        RET(decode_impl(h, h_out, h->z, h->word, logits, B, st, false, &rp, &fused, 2, t + 1 < T));  // fc_2 + argmax
        if (!fused) {
            h->pa_on = false;
            return fail(SAT_ERR_STATE, "chained loop needs the fused argmax of the vocabulary layer");
        }
        if (t + 1 < T) {
            h->pa_cur_h_in = h->pa_h[(t + 1) & 1];
            RET(attention_impl(h, ctx, B / G, G, h_out, step_alpha(alphas, t + 1, B, d.num_ctx), h->z, st, true, nullptr, budget,
                               true));
        }
    }
    h->pa_on = false;
    h->pa_cur_z = nullptr;
    return SAT_OK;
}

// The same step sequence with the three dense layers of a step as the phases of ONE persistent launch (sat_chain.cu):
//   chain(t) = { LSTM(t) -> [decode fc_1(t) || q(t+1)] -> vocabulary layer(t) + arg-max }  ->  attention(t+1)
// The attention kernel of step t+1 starts beside the chained launch, spins on the counter of its phase 1 (q(t+1) and
// everything older are complete then) and runs beside the vocabulary phase on the SMs whose CTAs have exited.
// OPT-IN (option "chain" = 1; default 0): its three epilogues and the last arriver's tail run from cold instruction
// caches, which made it slower than the per-layer launches where it was timed; and only validated for a 64-row tile (at B = 4 an eager, fully serialised run of it was seen to give wrong
// logits from the second step on while the replayed graph was right: unresolved, so smaller batches are refused).
static bool fused_loop_available(sat_handle* h, int B) {
    return h->opt_chain && h->pa_ok && h->opt_pa && h->opt_gemm != 0 && h->opt_overlap == 2 && h->opt_pdl &&
           h->d.num_decode_layers == 2 && h->d.num_attend_layers == 2 && h->opt_hoist && h->opt_att_wpc &&
           h->d.dim_attend_layer == 512 && h->d.dim_ctx == 512 && row_tile_for(B) == 64 && B <= h->num_sms &&
           (h->opt_trace == 0 || h->opt_trace >= 3) && h->opt_profile == 0;
}

static int loop_enqueue_fused(sat_handle* h, const float* ctx, int B, int T, const int32_t* forced, int32_t* tokens,
                              float* logits_all, cudaStream_t st, bool prepared) {
    const sat_dims& d = h->d;
    const size_t nctr = (size_t)kChainMaxPhase + (size_t)kChainMaxPhase * kChainMaxTiles;
    if (!h->chain_ctr) {
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "chained loop: workspace growth during graph capture");
        RET(dmalloc(&h->chain_ctr, nctr));
        RET(dmalloc(&h->chain_scratch, (size_t)h->num_sms * 64 * kTileN));
        RET(dmalloc(&h->chain_best, (size_t)h->max_rows));
        CK(cudaMemset(h->chain_best, 0, (size_t)h->max_rows * sizeof(unsigned long long)));
    }
    if (!prepared) RET(prepare_impl(h, ctx, B, h->st_c[0], h->st_h[0], st, h->pa_h[0]));
    CK(cudaMemsetAsync(h->word, 0, (size_t)B * sizeof(int32_t), st));  // <start> = 0 (model.py:254)
    CK(cudaMemsetAsync(h->chain_ctr, 0, nctr * sizeof(unsigned), st)); // counters are relative to the start of the loop
    int budget = h->opt_att_sms > 0 ? h->opt_att_sms : h->num_sms - h->dec_2.n_tiles;
    if (budget < B) budget = B;
    const int rtile = row_tile_for(B);
    const int stages = lin_chain_pick_stages(rtile);
    if (stages < 2) return fail(SAT_ERR_UNSUPPORTED, "chained loop: row tile %d does not fit", rtile);
    unsigned cta_sum[kChainMaxPhase] = {0, 0, 0}, split_sum[kChainMaxPhase] = {0, 0, 0};   // counter values after each launch
    for (int t = 0; t < T; ++t) {
        const float *c_in = h->st_c[t & 1], *h_in = h->st_h[t & 1];
        float *c_out = h->st_c[(t + 1) & 1], *h_out = h->st_h[(t + 1) & 1];
        h->pa_on = true;
        h->pa_cur_h_in = h->pa_h[t & 1];
        h->pa_cur_h_out = h->pa_h[(t + 1) & 1];
        h->pa_cur_z = h->pa_z;
        if (t == 0)   // q(0), attention(0) and the embedding of <start>
            RET(attention_impl(h, ctx, B, 1, h_in, nullptr, h->z, st, false, h->word));
        float* logits = logits_all ? logits_all + (size_t)t * B * d.vocabulary_size : nullptr;
        LinChain C;
        memset(&C, 0, sizeof(C));
        C.nphase = 3;
        // phase 0: current_input = concat([context, word_embed]) (model.py:277); LSTMCell concat([x, h]) (TF)
        {
            LinProblem& P = C.ph[0].p[0];
            RET(plan(h, h->lstm, P,
                     {seg(h->z, d.dim_ctx, d.dim_ctx, nullptr, h->pa_z),
                      seg(h->embedding, d.dim_embedding, d.dim_embedding, h->word, h->pa_emb),
                      seg(h_in, d.num_lstm_units, d.num_lstm_units, nullptr, h->pa_cur_h_in)},
                     B, kEpiLstm, nullptr, 0, st));
            P.out_pa = h->pa_cur_h_out;
            P.c_in = c_in; P.c_out = c_out; P.h_out = h_out; P.H = d.num_lstm_units;
            C.ph[0].nprob = 1;
        }
        // phase 1: expanded_output = concat([output, context, word_embed]) (model.py:283-286) -> fc_1; q of step t+1
        {
            const bool nq = t + 1 < T;
            LinProblem& P = C.ph[1].p[0];
            RET(plan(h, h->dec_1, P,
                     {seg(h_out, d.num_lstm_units, d.num_lstm_units, nullptr, h->pa_cur_h_out),
                      seg(h->z, d.dim_ctx, d.dim_ctx, nullptr, h->pa_z),
                      seg(h->embedding, d.dim_embedding, d.dim_embedding, h->word, h->pa_emb)},
                     B, kEpiBiasTanh, h->t_dec, d.dim_decode_layer, st, h->opt_dec1_splits, nq ? 2 : 1));
            P.out_pa = h->pa_t;
            C.ph[1].nprob = 1;
            if (nq) {
                RET(plan_att_state(h, C.ph[1].p[1], h_out, B, st, 2, h->pa_cur_h_out));
                C.ph[1].nprob = 2;
                // one split factor for the pair, like the grouped launch of the per-layer path (bit-identical sums)
                const int sm = C.ph[1].p[0].splits < C.ph[1].p[1].splits ? C.ph[1].p[0].splits : C.ph[1].p[1].splits;
                C.ph[1].p[0].splits = C.ph[1].p[1].splits = sm;
            }
        }
        // phase 2: logits = t * Wd2 + b, arg-max, embedding of the word fed to step t+1
        {
            LinProblem& P = C.ph[2].p[0];
            RET(plan(h, h->dec_2, P, {seg(h->t_dec, d.dim_decode_layer, d.dim_decode_layer, nullptr, h->pa_t)}, B, kEpiBias,
                     logits, d.vocabulary_size, st, 1));
            P.am_key = h->chain_best;
            P.am_tokens = tokens; P.am_tokens_ld = T; P.am_step = t;
            P.am_next_word = h->word; P.am_forced = forced; P.am_forced_ld = T;
            if (t + 1 < T) { P.am_emb = h->embedding; P.am_E = d.dim_embedding; P.am_emb_pa = h->pa_emb; }
            C.ph[2].nprob = 1;
        }
        int grid = 0;
        for (int ph = 0; ph < C.nphase; ++ph) {
            int begin = 0, tiles = 0;
            for (int i = 0; i < C.ph[ph].nprob; ++i) {
                LinProblem& P = C.ph[ph].p[i];
                if (P.n_row_tiles != 1 || P.row_tile != rtile) return fail(SAT_ERR_UNSUPPORTED, "chained loop: one row tile per layer");
                for (int sgi = 0; sgi < P.nseg; ++sgi)
                    if (!P.seg[sgi].pa) return fail(SAT_ERR_STATE, "chained loop: operands must arrive packed");
                P.cta_begin = begin;
                P.cta_count = P.n_tiles * P.splits;
                begin += P.cta_count;
                tiles += P.n_tiles;
            }
            if (tiles > kChainMaxTiles || begin > h->num_sms) return fail(SAT_ERR_UNSUPPORTED, "chained loop: %d tiles / %d CTAs in one phase", tiles, begin);
            for (int i = 1; i < C.ph[ph].nprob; ++i)
                if (C.ph[ph].p[i].splits != C.ph[ph].p[0].splits) return fail(SAT_ERR_STATE, "chained loop: one split factor per phase");
            C.ph[ph].ctas = begin;
            cta_sum[ph] += (unsigned)begin;                     // (the last step has no q tiles: sums, not multiples)
            split_sum[ph] += (unsigned)C.ph[ph].p[0].splits;
            C.target[ph] = cta_sum[ph];
            C.tile_target[ph] = split_sum[ph];
            if (begin > grid) grid = begin;
        }
        C.layout_mode = h->opt_layout;
        C.stages = stages;
        C.l2_w = h->opt_l2_w >= 0 ? h->opt_l2_w : 2;   // (the chained launch keeps one evict_last policy)
        C.pdl = 1;
        C.row_tile = rtile;
        C.ctr = h->chain_ctr;
        C.tile_ctr = h->chain_ctr + kChainMaxPhase;
        C.scratch = h->chain_scratch;
        // split-K partials through distributed shared memory when the splits of every tile fall inside one cluster
        // (option "chain_cluster" 0: through the L2 scratch buffer instead)
        {
            int cs = 1;
            bool ok = h->opt_chain_cluster != 0;
            for (int ph = 0; ph < C.nphase; ++ph)
                for (int i = 0; i < C.ph[ph].nprob; ++i) {
                    const LinProblem& P = C.ph[ph].p[i];
                    if (P.splits > cs) cs = P.splits;
                }
            for (int ph = 0; ph < C.nphase && ok; ++ph)
                for (int i = 0; i < C.ph[ph].nprob; ++i) {
                    const LinProblem& P = C.ph[ph].p[i];
                    if (P.splits > 1 && (P.cta_begin % P.splits || cs % P.splits)) ok = false;
                }
            C.cluster = 1;
            if (ok && cs > 1 && cs <= 8) {
                const int padded = (grid + cs - 1) / cs * cs;   // (CTAs past the last tile have no work and exit)
                // every cluster of the launch must be resident at once (the phases meet at grid-wide counters)
                if (h->chain_clusters[cs] < 0) h->chain_clusters[cs] = lin_chain_max_clusters(rtile, stages, cs);
                if (padded <= h->num_sms && h->chain_clusters[cs] * cs >= padded) { C.cluster = cs; grid = padded; }
            }
        }
        if (h->opt_trace == 3 && h->tl_count + 4 <= 4000) {   // four timeline entries: the launch, then its phases
            C.tl = h->trace + 4 * h->tl_count;
            h->tl_count += 4;
            h->tl_names.push_back("chain/" + std::to_string(grid));
            for (int ph = 0; ph < 3; ++ph) h->tl_names.push_back("  phase" + std::to_string(ph) + "/" + std::to_string(C.ph[ph].ctas));
        }
        if (h->opt_trace >= 4 && h->opt_trace <= 8 && h->trace_at-- == 0) { C.dbg = h->trace; C.dbg_mode = h->opt_trace - 4; }   // per-CTA stamps of this one launch
        CK(lin_chain_launch(C, grid, st));
        h->launches += 1;
        if (t + 1 < T) {
            h->pa_cur_h_in = h->pa_h[(t + 1) & 1];
            h->att_qflag = h->chain_ctr + 1;          // phase 1 of the launch above
            h->att_qtarget = C.target[1];
            const int rc = attention_impl(h, ctx, B, 1, h_out, nullptr, h->z, st, true, nullptr, budget, true);
            h->att_qflag = nullptr;
            RET(rc);
        }
    }
    h->pa_on = false;
    h->pa_cur_z = nullptr;
    return SAT_OK;
}

// The overlapped and chained loops hand the chosen word on inside the vocabulary layer: they need its fused arg-max,
// i.e. every CTA of that layer resident in one wave.
static bool vocab_argmax_fits(sat_handle* h, int B) {
    return h->dec_2.n_tiles * ((B + kMaxRowTile - 1) / kMaxRowTile) <= h->num_sms;
}

// G, smp: see loop_enqueue_overlap (the sampling loop runs G = num_samples rows per image)
// filter: filtered sampling (smp->top_k / top_p): the per-step layout, the vocabulary layer writes the logits and the
// filtered per-row kernel draws (the overlapped and chained layouts need the fused arg-max)
static int loop_enqueue(sat_handle* h, const float* ctx, int B, int T, const int32_t* forced, int32_t* tokens,
                        float* logits_all, float* alphas, float* word_probs, cudaStream_t st, int G = 1,
                        const SampleParams* smp = nullptr, bool filter = false) {
    const bool pa = h->pa_ok && h->opt_pa && h->opt_gemm != 0;
    const bool am = pa && vocab_argmax_fits(h, B) && !filter;
    const bool maps = alphas || word_probs;   // (the experimental chained launch takes no maps, and does not sample)
    if (!maps && !smp && fused_loop_available(h, B)) return loop_enqueue_fused(h, ctx, B, T, forced, tokens, logits_all, st, false);
    if (am && h->opt_overlap == 2 && h->opt_pdl && h->d.num_decode_layers == 2)
        return loop_enqueue_chain(h, ctx, B, T, forced, tokens, logits_all, alphas, word_probs, st, false, G, smp);
    if (am && h->opt_overlap && h->d.num_decode_layers == 2 && st != nullptr && st != cudaStreamLegacy)
        return loop_enqueue_overlap(h, ctx, B, T, forced, tokens, logits_all, alphas, word_probs, st, G, smp);
    RET(loop_prologue(h, ctx, B, G, st, pa ? h->pa_h[0] : nullptr));
    CK(cudaMemsetAsync(h->word, 0, (size_t)B * sizeof(int32_t), st));  // <start> = 0 (model.py:254)
    bool emb_valid = false;
    for (int t = 0; t < T; ++t) {
        StepIO io;
        memset(&io, 0, sizeof(io));
        io.ctx = ctx; io.n_img = B / G; io.group = G; io.last_word = h->word;
        io.c_in = h->st_c[t & 1]; io.h_in = h->st_h[t & 1];
        io.c_out = h->st_c[(t + 1) & 1]; io.h_out = h->st_h[(t + 1) & 1];
        io.logits = logits_all ? logits_all + (size_t)t * B * h->d.vocabulary_size : nullptr;
        io.alpha = step_alpha(alphas, t, B, h->d.num_ctx);
        io.want_rows = true;
        io.rows.tokens = tokens; io.rows.tokens_ld = T; io.rows.step = t;
        io.rows.next_word = h->word; io.rows.forced = forced; io.rows.forced_ld = T;
        io.rows.word_probs = word_probs;
        io.rows.sample = smp;
        io.rows.filter = filter ? 1 : 0;
        io.q_ready = t > 0;
        io.make_next_q = t + 1 < T;
        io.pa_slot = t & 1;          // initialize / the previous LSTM wrote the packed h into this slot
        io.pa_h_valid = pa;
        io.pa_emb_valid = emb_valid;
        RET(step_impl(h, io, st));
        emb_valid = io.pa_emb_valid;
    }
    return SAT_OK;
}

static bool chain_loop_available(sat_handle* h, int B) {
    return h->pa_ok && h->opt_pa && h->opt_gemm != 0 && h->opt_overlap == 2 && h->opt_pdl && h->d.num_decode_layers == 2 &&
           h->opt_hoist && h->d.num_attend_layers == 2 && vocab_argmax_fits(h, B);
}

// Greedy / teacher-forced loop with its prologue on a second stream (option "xbatch", and always for the pipelined
// host-buffer API): the context projection, mean and initialize layers of this call write one of two buffer sets
// (T1, c0/h0, packed h0) on `xb_stream` and only wait for the previous user of that set, so they run while the
// previous call's decode steps are still executing on `st`; the steps of this call wait for them.  `input_ready`
// (may be null) is an event the contexts depend on; with a null event the CALLER guarantees that the contexts are
// complete when the call is made (they must not be produced by earlier work queued on `st`).
static int decode_loop_xbatch(sat_handle* h, const float* contexts, int B, int T, const int32_t* forced, int32_t* tokens,
                              float* logits_all, float* alphas, float* word_probs, cudaStream_t st, cudaEvent_t input_ready) {
    const sat_dims& d = h->d;
    if (!h->xb_stream) {
        CK(cudaStreamCreateWithFlags(&h->xb_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CK(cudaEventCreateWithFlags(&h->xb[i].ev_prep, cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&h->xb[i].ev_done, cudaEventDisableTiming));
        }
        h->xb[0].T1 = h->T1; h->xb[0].c0 = h->st_c[0]; h->xb[0].h0 = h->st_h[0]; h->xb[0].pa_h0 = h->pa_h[0];
        const size_t R = (size_t)h->max_rows, RP = R + 272;
        RET(dmalloc(&h->xb[1].T1, R * d.num_ctx * d.dim_attend_layer));
        RET(dmalloc(&h->xb[1].c0, R * d.num_lstm_units));
        RET(dmalloc(&h->xb[1].h0, R * d.num_lstm_units));
        RET(dmalloc(&h->xb[1].pa_h0, RP * d.num_lstm_units * 4));
    }
    const int slot = h->xb_next;
    h->xb_next ^= 1;
    sat_handle::XbSlot& S = h->xb[slot];
    if (h->ops_since_xb > 1) {
        // some other entry point (step, beam search, prepare ...) was called since the last overlapped loop; it
        // uses the handle's own buffers (= set 0) in `st` order: let the prologue stream see all of `st` once
        cudaEvent_t ev = h->xb[0].ev_prep;
        CK(cudaEventRecord(ev, st));
        CK(cudaStreamWaitEvent(h->xb_stream, ev, 0));
    }
    h->ops_since_xb = 0;
    // this set's previous user (two calls back) must have finished decoding; the one in between uses the other set
    if (S.used) CK(cudaStreamWaitEvent(h->xb_stream, S.ev_done, 0));
    if (input_ready) CK(cudaStreamWaitEvent(h->xb_stream, input_ready, 0));
    // swap the set in: everything enqueued / captured below bakes these pointers in
    float *T1_keep = h->T1, *c_keep = h->st_c[0], *h_keep = h->st_h[0];
    uint8_t* pa_keep = h->pa_h[0];
    h->T1 = S.T1; h->st_c[0] = S.c0; h->st_h[0] = S.h0; h->pa_h[0] = S.pa_h0;
    int rc = run_graphed(h, {3, (long long)contexts, B, slot, (long long)alphas, (long long)word_probs}, h->xb_stream, [&]() -> int {
        return prepare_impl(h, contexts, B, h->st_c[0], h->st_h[0], h->xb_stream, h->pa_h[0]);
    });
    if (rc == SAT_OK) {
        cudaEventRecord(S.ev_prep, h->xb_stream);
        cudaStreamWaitEvent(st, S.ev_prep, 0);
        h->prep_ctx = contexts;
        h->prep_ni = B;
        rc = run_graphed(h, {4, (long long)contexts, B, T, (long long)forced, (long long)tokens, (long long)logits_all, slot,
                             (long long)alphas, (long long)word_probs}, st,
                         [&]() -> int {
                             return (fused_loop_available(h, B) && !alphas && !word_probs)
                                        ? loop_enqueue_fused(h, contexts, B, T, forced, tokens, logits_all, st, true)
                                        : loop_enqueue_chain(h, contexts, B, T, forced, tokens, logits_all, alphas, word_probs, st, true);
                         });
        cudaEventRecord(S.ev_done, st);
        S.used = true;
    }
    h->T1 = T1_keep; h->st_c[0] = c_keep; h->st_h[0] = h_keep; h->pa_h[0] = pa_keep;
    h->prep_ctx = nullptr;   // the handle's own T1 no longer matches any contexts
    return rc;
}

extern "C" int sat_decode_loop(sat_handle* h, const float* contexts, int32_t B, int32_t T, const int32_t* forced_words,
                               int32_t* tokens, float* logits_all, void* stream) {
    return sat_decode_loop_maps(h, contexts, B, T, forced_words, tokens, logits_all, nullptr, nullptr, stream);
}

extern "C" int sat_decode_loop_maps(sat_handle* h, const float* contexts, int32_t B, int32_t T, const int32_t* forced_words,
                                    int32_t* tokens, float* logits_all, float* alphas, float* word_probs, void* stream) {
    RET(require_ready(h));
    if (!contexts || !tokens) return fail(SAT_ERR_INVALID, "sat_decode_loop: null tensor");
    if (B < 1 || B > h->max_rows) return fail(SAT_ERR_INVALID, "batch %d outside [1, %d]", B, h->max_rows);
    if (T < 1) return fail(SAT_ERR_INVALID, "T must be >= 1");
    cudaStream_t st = (cudaStream_t)stream;
    if (h->opt_xbatch && chain_loop_available(h, B) && st != nullptr && st != cudaStreamLegacy && st != cudaStreamPerThread)
        return decode_loop_xbatch(h, contexts, B, T, forced_words, tokens, logits_all, alphas, word_probs, st, nullptr);
    // the map buffers are part of the key: a replayed graph writes into the buffers it was captured with
    std::vector<long long> key = {1, (long long)contexts, B, T, (long long)forced_words, (long long)tokens,
                                  (long long)logits_all, (long long)alphas, (long long)word_probs};
    const int rc = run_graphed(h, key, st, [&]() -> int {
        return loop_enqueue(h, contexts, B, T, forced_words, tokens, logits_all, alphas, word_probs, st);
    });
    // A replayed graph re-projects `contexts` into T1 on the device without passing through prepare_impl: the host-side
    // record of what T1 holds must follow in every case (eager, capture, replay), or a later single step on other
    // contexts would skip its projection.
    note_projected(h, rc == SAT_OK ? contexts : nullptr, B);
    return rc;
}

// ------------------------------------------------------------ sampling
extern "C" double sat_sample_uniform(uint64_t seed, int64_t row, int32_t step, int32_t word) {
    const uint32_t bits = sample_bits(sample_key(seed, row, step), word);
    return ((double)bits + 0.5) * 2.3283064365386963e-10;   // (bits + 1/2) 2^-32: exact in fp64
}

extern "C" int sat_sample_loop(sat_handle* h, const float* contexts, int32_t n_img, int32_t num_samples, int32_t T,
                               float temperature, uint64_t seed, int32_t* tokens, float* word_probs, void* stream) {
    if (!h) return fail(SAT_ERR_INVALID, "null handle");
    if (!contexts || !tokens) return fail(SAT_ERR_INVALID, "sat_sample_loop: null tensor");
    if (!(temperature > 0.0f) || !isfinite(temperature) || !isfinite(1.0f / temperature))
        return fail(SAT_ERR_INVALID, "temperature %g must be positive and finite", (double)temperature);
    if (num_samples < 1) return fail(SAT_ERR_INVALID, "num_samples %d < 1", num_samples);
    if (n_img < 1 || (long long)n_img * num_samples > h->max_rows)
        return fail(SAT_ERR_INVALID, "n_img*num_samples %lld outside [1, %d]", (long long)n_img * num_samples, h->max_rows);
    if (T < 1) return fail(SAT_ERR_INVALID, "T must be >= 1");
    // the rows of an image share its contexts inside the attention kernels, which take up to 4 rows per image
    if (num_samples > 4) return fail(SAT_ERR_UNSUPPORTED, "num_samples %d > 4 (draw more with further seeds)", num_samples);
    RET(require_ready(h));
    cudaStream_t st = (cudaStream_t)stream;
    if (!h->smp) {
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "sat_sample_loop: allocation during graph capture");
        RET(dmalloc(&h->smp, 1));
    }
    // seed and temperature live in device memory, written here outside any capture: a graph captured for these buffers
    // replays with any seed or temperature
    CK(sample_params_launch(h->smp, seed, 1.0f / temperature, st));
    h->launches += 1;
    const int B = n_img * num_samples;
    std::vector<long long> key = {5, (long long)contexts, n_img, num_samples, T, (long long)tokens, (long long)word_probs};
    const int rc = run_graphed(h, key, st, [&]() -> int {
        return loop_enqueue(h, contexts, B, T, nullptr, tokens, nullptr, nullptr, word_probs, st, num_samples, h->smp);
    });
    note_projected(h, rc == SAT_OK ? contexts : nullptr, n_img);   // (see sat_decode_loop)
    return rc;
}

extern "C" int sat_sample_loop_filtered(sat_handle* h, const float* contexts, int32_t n_img, int32_t num_samples,
                                        int32_t T, float temperature, int32_t top_k, float top_p, uint64_t seed,
                                        int32_t* tokens, float* word_probs, void* stream) {
    if (!h) return fail(SAT_ERR_INVALID, "null handle");
    if (top_k < 0) return fail(SAT_ERR_INVALID, "top_k %d < 0", top_k);
    if (!(top_p > 0.0f && top_p <= 1.0f)) return fail(SAT_ERR_INVALID, "top_p %g outside (0, 1]", (double)top_p);
    if (top_k == 0 && top_p == 1.0f)
        return sat_sample_loop(h, contexts, n_img, num_samples, T, temperature, seed, tokens, word_probs, stream);
    if (!contexts || !tokens) return fail(SAT_ERR_INVALID, "sat_sample_loop_filtered: null tensor");
    if (!(temperature > 0.0f) || !isfinite(temperature) || !isfinite(1.0f / temperature))
        return fail(SAT_ERR_INVALID, "temperature %g must be positive and finite", (double)temperature);
    if (num_samples < 1) return fail(SAT_ERR_INVALID, "num_samples %d < 1", num_samples);
    if (n_img < 1 || (long long)n_img * num_samples > h->max_rows)
        return fail(SAT_ERR_INVALID, "n_img*num_samples %lld outside [1, %d]", (long long)n_img * num_samples, h->max_rows);
    if (T < 1) return fail(SAT_ERR_INVALID, "T must be >= 1");
    if (num_samples > 4) return fail(SAT_ERR_UNSUPPORTED, "num_samples %d > 4 (draw more with further seeds)", num_samples);
    RET(require_ready(h));
    cudaStream_t st = (cudaStream_t)stream;
    if (!h->smp) {
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "sat_sample_loop_filtered: allocation during graph capture");
        RET(dmalloc(&h->smp, 1));
    }
    // the filters live in device memory beside seed and temperature: a captured graph replays with any of them
    CK(sample_params_launch(h->smp, seed, 1.0f / temperature, st, top_k, top_p));
    h->launches += 1;
    const int B = n_img * num_samples;
    std::vector<long long> key = {6, (long long)contexts, n_img, num_samples, T, (long long)tokens, (long long)word_probs};
    const int rc = run_graphed(h, key, st, [&]() -> int {
        return loop_enqueue(h, contexts, B, T, nullptr, tokens, nullptr, nullptr, word_probs, st, num_samples, h->smp, true);
    });
    note_projected(h, rc == SAT_OK ? contexts : nullptr, n_img);   // (see sat_decode_loop)
    return rc;
}

// ------------------------------------------------------------ beam search
static int beam_enqueue(sat_handle* h, const float* ctx, int NI, int beam, int T, int eos, int32_t* sentences,
                        int32_t* lengths, double* scores, int32_t* n_results, int32_t* is_complete, float* alphas,
                        float* word_probs, cudaStream_t st) {
    const bool maps = alphas || word_probs;
    const sat_dims& d = h->d;
    const int H = d.num_lstm_units;
    // states: st_*[0] = inputs of the current step, st_*[1] = outputs
    RET(prepare_impl(h, ctx, NI, h->st_c[0], h->st_h[0], st));               // base_model.py:168-170
    CK(cudaMemsetAsync(h->comp_n, 0, (size_t)NI * sizeof(int32_t), st));
    BeamParams bp;
    memset(&bp, 0, sizeof(bp));
    bp.NI = NI; bp.beam = beam; bp.T = T; bp.eos_id = eos; bp.H = H;
    bp.topk_idx = h->topk_idx; bp.topk_p = h->topk_p;
    bp.part_score = h->part_score; bp.part_n = h->part_n;
    bp.sent[0] = h->sent[0]; bp.sent[1] = h->sent[1];
    bp.comp_heap = (CItem*)h->comp_heap; bp.comp_n = h->comp_n; bp.comp_sent = h->comp_sent;
    bp.c_out = h->st_c[1]; bp.h_out = h->st_h[1]; bp.c_next = h->st_c[0]; bp.h_next = h->st_h[0];
    bp.next_word = h->word;
    bp.res_sent = sentences; bp.res_len = lengths; bp.res_score = scores; bp.res_n = n_results;
    bp.res_complete = is_complete;
    const size_t NB = (size_t)NI * beam;
    if (maps) {
        bp.hist_alpha = h->hist_alpha; bp.hist_parent = h->hist_parent; bp.hist_p = h->hist_p;
        bp.comp_prov = h->comp_prov; bp.comp_p = h->comp_p; bp.res_src = h->res_src;
        bp.L = d.num_ctx; bp.res_alpha = alphas; bp.res_probs = word_probs;
    }
    for (int idx = 0; idx < T; ++idx) {                                       // base_model.py:184
        const int G = idx == 0 ? 1 : beam;                                    // base_model.py:191
        StepIO io;
        memset(&io, 0, sizeof(io));
        io.ctx = ctx; io.n_img = NI; io.group = G;
        if (maps) io.alpha = h->hist_alpha + (size_t)idx * NB * d.num_ctx;   // rows img*G + g
        io.last_word = idx == 0 ? h->zero_word : h->word;                     // base_model.py:193-198
        io.c_in = h->st_c[0]; io.h_in = h->st_h[0]; io.c_out = h->st_c[1]; io.h_out = h->st_h[1];
        io.want_rows = true;
        io.rows.topk = beam + 1; io.rows.topk_idx = h->topk_idx; io.rows.topk_p = h->topk_p;
        RET(step_impl(h, io, st));
        bp.nlive = G; bp.step = idx;
        {
            ProfScope ps(h, kTagBeam, st);
            CK(beam_update_launch(bp, st));
        }
        h->launches += 1;
    }
    bp.step = T;
    CK(beam_finalize_launch(bp, st));
    h->launches += 1;
    if (maps) {
        CK(beam_maps_launch(bp, st));
        h->launches += 1;
    }
    return SAT_OK;
}

extern "C" int sat_beam_search(sat_handle* h, const float* contexts, int32_t n_img, int32_t beam_size, int32_t T,
                               int32_t eos_id, int32_t* sentences, int32_t* lengths, double* scores,
                               int32_t* n_results, int32_t* is_complete, void* stream) {
    return sat_beam_search_maps(h, contexts, n_img, beam_size, T, eos_id, sentences, lengths, scores, n_results,
                                is_complete, nullptr, nullptr, stream);
}

extern "C" int sat_beam_search_maps(sat_handle* h, const float* contexts, int32_t n_img, int32_t beam_size, int32_t T,
                                    int32_t eos_id, int32_t* sentences, int32_t* lengths, double* scores,
                                    int32_t* n_results, int32_t* is_complete, float* alphas, float* word_probs,
                                    void* stream) {
    RET(require_ready(h));
    if (!contexts || !sentences || !lengths || !scores || !n_results || !is_complete)
        return fail(SAT_ERR_INVALID, "sat_beam_search: null tensor");
    if (beam_size < 1 || beam_size > h->d.max_beam) return fail(SAT_ERR_INVALID, "beam_size %d outside [1, %d]", beam_size, h->d.max_beam);
    if (T < 1 || T > h->d.max_caption_length) return fail(SAT_ERR_INVALID, "T %d outside [1, %d]", T, h->d.max_caption_length);
    if (n_img < 1 || (long long)n_img * beam_size > h->max_rows)
        return fail(SAT_ERR_INVALID, "n_img*beam %lld > max_batch %d", (long long)n_img * beam_size, h->max_rows);
    if (h->d.vocabulary_size < beam_size + 2) return fail(SAT_ERR_INVALID, "vocabulary too small for beam %d", beam_size);
    cudaStream_t st = (cudaStream_t)stream;
    if ((alphas || word_probs) && !h->hist_alpha) {   // history of the first request, sized for the handle's limits
        if (T > 1024) return fail(SAT_ERR_UNSUPPORTED, "beam maps: T %d > 1024", T);
        if (stream_capturing(st)) return fail(SAT_ERR_STATE, "beam maps: allocation during graph capture");
        const size_t R = (size_t)h->max_rows, TM = (size_t)h->d.max_caption_length;
        RET(dmalloc(&h->hist_alpha, TM * R * h->d.num_ctx));
        RET(dmalloc(&h->hist_parent, TM * R));
        RET(dmalloc(&h->hist_p, TM * R));
        RET(dmalloc(&h->comp_prov, R));
        RET(dmalloc(&h->comp_p, R));
        RET(dmalloc(&h->res_src, R));
    }
    std::vector<long long> key = {2, (long long)contexts, n_img, beam_size, T, eos_id, (long long)sentences,
                                  (long long)lengths, (long long)scores, (long long)n_results, (long long)is_complete,
                                  (long long)alphas, (long long)word_probs};
    const int rc = run_graphed(h, key, st, [&]() -> int {
        return beam_enqueue(h, contexts, n_img, beam_size, T, eos_id, sentences, lengths, scores, n_results,
                            is_complete, alphas, word_probs, st);
    });
    note_projected(h, rc == SAT_OK ? contexts : nullptr, n_img);   // (see sat_decode_loop)
    return rc;
}

// ---------------------------------------------------------- host-buffer forms
static int ensure_stage(sat_handle* h, size_t misc_bytes) {
    const sat_dims& d = h->d;
    if (!h->stage_ctx) RET(dmalloc(&h->stage_ctx, (size_t)h->max_rows * d.num_ctx * d.dim_ctx));
    if (misc_bytes > h->stage_misc_bytes) {
        CK(cudaDeviceSynchronize());
        cudaFree(h->stage_misc);
        h->stage_misc = nullptr;
        h->stage_misc_bytes = 0;
        RET(dmalloc((uint8_t**)&h->stage_misc, misc_bytes));
        h->stage_misc_bytes = misc_bytes;
    }
    return SAT_OK;
}

extern "C" int sat_decode_step_host(sat_handle* h, const float* contexts_host, int32_t contexts_changed,
                                    const int32_t* last_word_host, const float* last_memory_host,
                                    const float* last_output_host, float* memory_host, float* output_host,
                                    float* probs_host, int32_t B, void* stream) {
    RET(require_ready(h));
    if (!contexts_host || !last_word_host || !last_memory_host || !last_output_host || !memory_host || !output_host ||
        !probs_host)
        return fail(SAT_ERR_INVALID, "sat_decode_step_host: null buffer");
    if (B < 1 || B > h->max_rows) return fail(SAT_ERR_INVALID, "batch %d outside [1, %d]", B, h->max_rows);
    const sat_dims& d = h->d;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t HB = (size_t)B * d.num_lstm_units * sizeof(float), VB = (size_t)B * d.vocabulary_size * sizeof(float);
    RET(ensure_stage(h, 4 * HB + VB + (size_t)B * sizeof(int32_t)));
    uint8_t* m = (uint8_t*)h->stage_misc;
    float *c_in = (float*)m, *h_in = (float*)(m + HB), *c_out = (float*)(m + 2 * HB), *h_out = (float*)(m + 3 * HB);
    float* probs = (float*)(m + 4 * HB);
    int32_t* lw = (int32_t*)(m + 4 * HB + VB);
    if (contexts_changed || h->prep_ctx != h->stage_ctx || h->prep_ni != B) {
        CK(cudaMemcpyAsync(h->stage_ctx, contexts_host, (size_t)B * d.num_ctx * d.dim_ctx * sizeof(float),
                           cudaMemcpyHostToDevice, st));
        RET(prepare_impl(h, h->stage_ctx, B, nullptr, nullptr, st));
    }
    CK(cudaMemcpyAsync(lw, last_word_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(c_in, last_memory_host, HB, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h_in, last_output_host, HB, cudaMemcpyHostToDevice, st));
    StepIO io;
    memset(&io, 0, sizeof(io));
    io.ctx = h->stage_ctx; io.n_img = B; io.group = 1; io.last_word = lw;
    io.c_in = c_in; io.h_in = h_in; io.c_out = c_out; io.h_out = h_out; io.probs = probs;
    RET(step_impl(h, io, st));
    CK(cudaMemcpyAsync(memory_host, c_out, HB, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(output_host, h_out, HB, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(probs_host, probs, VB, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SAT_OK;
}

extern "C" int sat_decode_loop_host(sat_handle* h, const float* contexts_host, int32_t B, int32_t T,
                                    const int32_t* forced_words_host, int32_t* tokens_host, void* stream) {
    RET(require_ready(h));
    if (!contexts_host || !tokens_host) return fail(SAT_ERR_INVALID, "sat_decode_loop_host: null buffer");
    if (B < 1 || B > h->max_rows || T < 1) return fail(SAT_ERR_INVALID, "bad B/T");
    const sat_dims& d = h->d;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t TB = (size_t)B * T * sizeof(int32_t);
    RET(ensure_stage(h, 2 * TB));
    int32_t* tok = (int32_t*)h->stage_misc;
    int32_t* forced = forced_words_host ? (int32_t*)((uint8_t*)h->stage_misc + TB) : nullptr;
    CK(cudaMemcpyAsync(h->stage_ctx, contexts_host, (size_t)B * d.num_ctx * d.dim_ctx * sizeof(float),
                       cudaMemcpyHostToDevice, st));
    if (forced) CK(cudaMemcpyAsync(forced, forced_words_host, TB, cudaMemcpyHostToDevice, st));
    RET(sat_decode_loop(h, h->stage_ctx, B, T, forced, tok, nullptr, stream));
    CK(cudaMemcpyAsync(tokens_host, tok, TB, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SAT_OK;
}

// Pipelined host-buffer loop.  submit(slot) enqueues, without blocking the host: the upload of the batch on a copy
// stream into staging slot `slot`, the decode loop behind it on `stream`, and the download of the tokens; wait(slot)
// returns once that batch's tokens are in tokens_host.  Submitting batch i+1 (other slot) before waiting for batch
// i overlaps its upload with batch i's decode: the caller's pageable/pinned buffers must stay valid until wait().
extern "C" int sat_decode_loop_host_submit(sat_handle* h, const float* contexts_host, int32_t B, int32_t T,
                                           const int32_t* forced_words_host, int32_t* tokens_host, int32_t slot,
                                           void* stream) {
    RET(require_ready(h));
    if (!contexts_host || !tokens_host) return fail(SAT_ERR_INVALID, "sat_decode_loop_host_submit: null buffer");
    if (B < 1 || B > h->max_rows || T < 1) return fail(SAT_ERR_INVALID, "bad B/T");
    if (slot < 0 || slot > 1) return fail(SAT_ERR_INVALID, "slot must be 0 or 1");
    if (h->pipe_busy[slot]) return fail(SAT_ERR_STATE, "slot %d was submitted and not waited for", slot);
    const sat_dims& d = h->d;
    cudaStream_t st = (cudaStream_t)stream;
    if (!h->pipe_copy) {
        CK(cudaStreamCreateWithFlags(&h->pipe_copy, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
            CK(cudaEventCreateWithFlags(&h->pipe_up[i], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&h->pipe_done[i], cudaEventDisableTiming));
        }
    }
    if (!h->pipe_ctx[slot]) RET(dmalloc(&h->pipe_ctx[slot], (size_t)h->max_rows * d.num_ctx * d.dim_ctx));
    const size_t TB = (size_t)B * T;
    if (2 * TB > h->pipe_tok_elems[slot]) {
        CK(cudaDeviceSynchronize());
        cudaFree(h->pipe_tok[slot]);
        h->pipe_tok[slot] = nullptr;
        h->pipe_tok_elems[slot] = 0;
        RET(dmalloc(&h->pipe_tok[slot], 2 * TB));
        h->pipe_tok_elems[slot] = 2 * TB;
    }
    int32_t* tok = h->pipe_tok[slot];
    int32_t* forced = forced_words_host ? tok + TB : nullptr;
    // (the previous batch of this slot was waited for, so its staging buffers are free)
    CK(cudaMemcpyAsync(h->pipe_ctx[slot], contexts_host, (size_t)B * d.num_ctx * d.dim_ctx * sizeof(float),
                       cudaMemcpyHostToDevice, h->pipe_copy));
    if (forced) CK(cudaMemcpyAsync(forced, forced_words_host, TB * sizeof(int32_t), cudaMemcpyHostToDevice, h->pipe_copy));
    CK(cudaEventRecord(h->pipe_up[slot], h->pipe_copy));
    CK(cudaStreamWaitEvent(st, h->pipe_up[slot], 0));      // (forced words; and the contexts when not overlapped)
    if (chain_loop_available(h, B) && st != nullptr && st != cudaStreamLegacy && st != cudaStreamPerThread)
        RET(decode_loop_xbatch(h, h->pipe_ctx[slot], B, T, forced, tok, nullptr, nullptr, nullptr, st, h->pipe_up[slot]));
    else
        RET(sat_decode_loop(h, h->pipe_ctx[slot], B, T, forced, tok, nullptr, stream));
    CK(cudaMemcpyAsync(tokens_host, tok, TB * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(h->pipe_done[slot], st));
    h->pipe_busy[slot] = true;
    return SAT_OK;
}

extern "C" int sat_decode_loop_host_wait(sat_handle* h, int32_t slot) {
    if (!h) return fail(SAT_ERR_INVALID, "null handle");
    if (slot < 0 || slot > 1) return fail(SAT_ERR_INVALID, "slot must be 0 or 1");
    if (!h->pipe_busy[slot]) return fail(SAT_ERR_STATE, "slot %d has no batch in flight", slot);
    CK(cudaEventSynchronize(h->pipe_done[slot]));
    h->pipe_busy[slot] = false;
    return SAT_OK;
}

extern "C" int sat_beam_search_host(sat_handle* h, const float* contexts_host, int32_t n_img, int32_t beam_size,
                                    int32_t T, int32_t eos_id, int32_t* sentences_host, int32_t* lengths_host,
                                    double* scores_host, int32_t* n_results_host, int32_t* is_complete_host,
                                    void* stream) {
    RET(require_ready(h));
    if (!contexts_host || !sentences_host || !lengths_host || !scores_host || !n_results_host || !is_complete_host)
        return fail(SAT_ERR_INVALID, "sat_beam_search_host: null buffer");
    if (n_img < 1 || beam_size < 1 || T < 1 || (long long)n_img * beam_size > h->max_rows)
        return fail(SAT_ERR_INVALID, "bad n_img/beam/T");
    const sat_dims& d = h->d;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t nb = (size_t)n_img * beam_size;
    const size_t o_sc = 0, o_sent = nb * 8, o_len = o_sent + nb * T * 4, o_n = o_len + nb * 4, o_c = o_n + n_img * 4,
                 total = o_c + n_img * 4;
    RET(ensure_stage(h, total));
    uint8_t* m = (uint8_t*)h->stage_misc;
    CK(cudaMemcpyAsync(h->stage_ctx, contexts_host, (size_t)n_img * d.num_ctx * d.dim_ctx * sizeof(float),
                       cudaMemcpyHostToDevice, st));
    RET(sat_beam_search(h, h->stage_ctx, n_img, beam_size, T, eos_id, (int32_t*)(m + o_sent), (int32_t*)(m + o_len),
                        (double*)(m + o_sc), (int32_t*)(m + o_n), (int32_t*)(m + o_c), stream));
    CK(cudaMemcpyAsync(scores_host, m + o_sc, nb * 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(sentences_host, m + o_sent, nb * T * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(lengths_host, m + o_len, nb * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(n_results_host, m + o_n, (size_t)n_img * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(is_complete_host, m + o_c, (size_t)n_img * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SAT_OK;
}

// ------------------------------------------------- individually callable kernels
extern "C" int sat_attention_fwd(sat_handle* h, const float* contexts, const float* output, float* alpha,
                                 float* context, int32_t n_img, int32_t group, void* stream) {
    RET(require_ready(h));
    if (!contexts || !output || !context) return fail(SAT_ERR_INVALID, "sat_attention_fwd: null tensor");
    if (n_img < 1 || group < 1 || (long long)n_img * group > h->max_rows)
        return fail(SAT_ERR_INVALID, "n_img*group outside [1, %d]", h->max_rows);
    // (debug option "att_reuse_q": keep the state branch of the previous call, launch the attention kernel alone)
    return attention_impl(h, contexts, n_img, group, output, alpha, context, (cudaStream_t)stream, h->opt_att_reuse_q != 0);
}

extern "C" int sat_lstm_fwd(sat_handle* h, const float* context, const int32_t* last_word, const float* last_memory,
                            const float* last_output, float* memory, float* output, int32_t rows, void* stream) {
    RET(require_ready(h));
    if (!context || !last_word || !last_memory || !last_output || !memory || !output)
        return fail(SAT_ERR_INVALID, "sat_lstm_fwd: null tensor");
    if (rows < 1 || rows > h->max_rows) return fail(SAT_ERR_INVALID, "rows outside [1, %d]", h->max_rows);
    return lstm_impl(h, context, last_word, last_memory, last_output, memory, output, rows, (cudaStream_t)stream);
}

extern "C" int sat_vocab_gemm(sat_handle* h, const float* output, const float* context, const int32_t* last_word,
                              float* logits, int32_t rows, void* stream) {
    RET(require_ready(h));
    if (!output || !context || !last_word || !logits) return fail(SAT_ERR_INVALID, "sat_vocab_gemm: null tensor");
    if (rows < 1 || rows > h->max_rows) return fail(SAT_ERR_INVALID, "rows outside [1, %d]", h->max_rows);
    return decode_impl(h, output, context, last_word, logits, rows, (cudaStream_t)stream);
}

extern "C" int sat_dense_fwd(sat_handle* h, const float* x, const float* w_tf, const float* b, float* y, int32_t rows,
                             int32_t K, int32_t n_out, int32_t act, int32_t splits, void* stream) {
    if (!h || !x || !w_tf || !y) return fail(SAT_ERR_INVALID, "sat_dense_fwd: null argument");
    if (rows < 1 || K < 8 || K % 8 || n_out < 1) return fail(SAT_ERR_INVALID, "sat_dense_fwd: bad shape");
    cudaStream_t st = (cudaStream_t)stream;
    Layer ly;
    std::vector<Layer*> keep = h->layers;  // layer_setup registers the layer; undo below
    int rc = layer_setup(h, ly, "dense_fwd", K, n_out, false, true);
    h->layers = keep;
    if (rc == SAT_OK) {
        auto body = [&]() -> int {
            CK(lin_repack_weight(w_tf, K, n_out, 0, ly.wpack, h->opt_layout, st));
            CK(lin_repack_bias(b, n_out, 0, ly.bias, st));
            LinProblem P;
            RET(plan(h, ly, P, {seg(x, K, K)}, rows, act ? kEpiBiasTanh : kEpiBias, y, n_out, st, splits));
            RET(launch(h, &P, 1, st));
            CK(cudaStreamSynchronize(st));
            return SAT_OK;
        };
        rc = body();
    }
    layer_free(ly);
    return rc;
}
