// sat_rows.cuh — per-row vocabulary kernels + device beam bookkeeping (see sat_rows.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sat {

struct SampleParams;   // sat_linear.cuh

constexpr int kMaxTopK = 8;
constexpr int kMaxBeam = 7;

struct RowsParams {
    const float* logits;  // [rows, V]
    int V;
    float* probs;         // [rows, V] or null
    int32_t* argmax;      // [rows] or null
    int32_t* tokens;      // [rows, tokens_ld] or null: tokens[row, step] = argmax
    int tokens_ld;
    int step;
    int32_t* next_word;   // [rows] or null: word fed to the next step
    const int32_t* forced;  // [rows, forced_ld] teacher-forced words or null (greedy)
    int forced_ld;
    int topk;             // 0 or beam+1
    int32_t* topk_idx;    // [rows, topk]
    float* topk_p;        // [rows, topk]
    float* word_probs;    // [rows, tokens_ld] or null: word_probs[row, step] = softmax[next word]
                          // (0 for a forced word outside [0, V))
    const SampleParams* sample;   // sampling loop (no forced words, no top-k): the word is the arg-max of
                                  // logit / temperature + the Gumbel noise of (seed, row, step, word), as in the fused
                                  // vocabulary layer; word_probs stay softmax(logits) at temperature 1
    int filter;           // with `sample`: draw only among the words kept by sample->top_k / top_p (filtered instance)
    unsigned long long* tl;   // optional timeline cells of the filtered instance (debug option "trace" = 3)
};

struct PItem;
struct CItem;

struct BeamParams {
    int NI, beam, nlive, T, step, eos_id, H;
    const int32_t* topk_idx;  // [NI*nlive, beam+1]
    const float* topk_p;
    double* part_score;       // [NI, beam]   partial heap (array order == row order of the next step)
    int32_t* part_n;          // [NI]
    int32_t* sent[2];         // [NI, beam, T] ping-pong by step parity
    CItem* comp_heap;         // [NI, beam]
    int32_t* comp_n;          // [NI]
    int32_t* comp_sent;       // [NI, beam, T]
    const float* c_out;       // [NI*nlive, H] states computed this step
    const float* h_out;
    float* c_next;            // [NI*beam, H] states fed to the next step
    float* h_next;
    int32_t* next_word;       // [NI*beam]
    // results (finalize)
    int32_t* res_sent;        // [NI, beam, T], -1 padded
    int32_t* res_len;         // [NI, beam]
    double* res_score;        // [NI, beam]
    int32_t* res_n;           // [NI]
    int32_t* res_complete;    // [NI]
    // per-word maps (null: not requested).  A back-pointer history instead of copies of every beam's maps:
    const float* hist_alpha;  // [T, NI*beam, L] alpha of step t, rows img*G + g (written by the attention launches)
    int32_t* hist_parent;     // [T, NI*beam] live row of step t that survivor j of step t came from
    float* hist_p;            // [T, NI*beam] probability of survivor j's word of step t
    int32_t* comp_prov;       // [NI, beam] per completed-caption slot: live row it completed from
    float* comp_p;            // [NI, beam] and the probability of its last word
    int32_t* res_src;         // [NI, beam] finalize: completed slot / partial beam of result j, -1 if none
    int L;
    float* res_alpha;         // [NI, beam, T, L]
    float* res_probs;         // [NI, beam, T]
};

cudaError_t rows_softmax_launch(const RowsParams& p, int rows, cudaStream_t st);
cudaError_t beam_update_launch(const BeamParams& p, cudaStream_t st);
cudaError_t beam_finalize_launch(const BeamParams& p, cudaStream_t st);
cudaError_t beam_maps_launch(const BeamParams& p, cudaStream_t st);   // after finalize, when res_alpha / res_probs
size_t beam_citem_bytes();
// sampling loop: *dst = {seed, inv_tau, top_k, top_p} (one thread, queued on the caller's stream ahead of a replayed
// graph)
cudaError_t sample_params_launch(SampleParams* dst, unsigned long long seed, float inv_tau, cudaStream_t st,
                                 int top_k = 0, float top_p = 1.0f);
// rows [r] of c_dst / h_dst = rows [r / G] of c_src / h_src ([rows / G, H] -> [rows, H], H % 4 == 0)
cudaError_t bcast_state_launch(const float* c_src, const float* h_src, float* c_dst, float* h_dst, int rows, int G, int H,
                               cudaStream_t st);

}  // namespace sat
