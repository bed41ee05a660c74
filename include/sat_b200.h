/* sat_b200.h — C ABI of libsat_b200.so: the soft-attention LSTM decode path of
 * Cheng-Lin-Li/show-attend-and-tell on NVIDIA H100 (sm_90a).
 *
 * The reference has no FFI: its boundary is the Python attribute surface of
 * CaptionGenerator consumed through tf.Session.run feeds/fetches.  Each entry point
 * below names the reference interface it replaces (paths relative to the reference
 * repository root).
 *
 * Conventions
 *   - return 0 (SAT_OK) on success, a negative SAT_ERR_* code otherwise; nothing is
 *     thrown or aborted across the boundary; sat_last_error() describes the failure
 *     (thread local).
 *   - every tensor argument is a DEVICE pointer unless the name ends in _host;
 *     the caller owns every tensor buffer; the library owns its workspace and its
 *     repacked copies of the weights.
 *   - all tensors are dense row-major fp32 (model.py:205-213) except word ids, which
 *     are int32 (model.py:214-216).
 *   - calls are asynchronous on `stream` (a cudaStream_t passed as void*); no hidden
 *     synchronisation except in *_host entry points, which return after the results
 *     are in host memory.
 *   - a handle is bound to the CUDA device current at sat_create and is not thread
 *     safe (the reference's driver loop is single threaded: base_model.py:184-212).
 */
#ifndef SAT_B200_H_
#define SAT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SAT_OK 0
#define SAT_ERR_INVALID (-1)     /* bad argument / shape mismatch (TF InvalidArgumentError) */
#define SAT_ERR_CUDA (-2)        /* a CUDA runtime / driver call failed */
#define SAT_ERR_STATE (-3)       /* weights missing, contexts not prepared, ... */
#define SAT_ERR_UNSUPPORTED (-4) /* shape outside what the kernels implement */
#define SAT_ERR_NOMEM (-5)

typedef struct sat_handle sat_handle;

/* Static shape of the decoder graph.  Field names follow config.py:9-17,67 (including the
 * `initalize` spelling); L and D are num_ctx / dim_ctx of model.py:54-59,103-108. */
typedef struct sat_dims {
    int32_t max_batch;            /* max rows per step = images x beam            */
    int32_t num_ctx;              /* L                                            */
    int32_t dim_ctx;              /* D                                            */
    int32_t num_lstm_units;       /* H                                            */
    int32_t dim_embedding;        /* E                                            */
    int32_t dim_attend_layer;     /* A                                            */
    int32_t dim_decode_layer;     /* Dd                                           */
    int32_t dim_initalize_layer;  /* I                                            */
    int32_t vocabulary_size;      /* V                                            */
    int32_t num_attend_layers;    /* 1 or 2                                       */
    int32_t num_decode_layers;    /* 1 or 2                                       */
    int32_t num_initalize_layers; /* 1 or 2                                       */
    int32_t max_caption_length;   /* max steps of a loop / beam search            */
    int32_t max_beam;             /* max beam_size (<= 4); 0 or 1 = no beam search */
} sat_dims;

/* replaces CaptionGenerator(config) (main.py:48,61,69; model.py:7-13, build_rnn :190-356) */
int sat_create(const sat_dims* dims, sat_handle** out);
void sat_destroy(sat_handle* h);
const char* sat_last_error(void);
int sat_version(void);

/* integer knobs (defaults in brackets; all of them are for experiments and tests, none changes results beyond
 * the summation order noted):
 *   "gemm"        1 = wgmma tensor cores [1], 0 = CUDA-core bring-up kernels
 *   "umma_layout" 0 = interleaved [0], 1 = 128B swizzle; must be set before sat_set_weight
 *   "graphs"      1 = replay CUDA graphs in loops [1]
 *   "hoist"       1 = project the contexts once per image batch [1]; 0 = recompute every step like model.py:259-262
 *   "pa"          1 = activations travel between dense layers as packed MMA operands [1]
 *   "xpack"       1 = cooperative activation pre-pass when operands are not packed [1]; 0 = producer warps
 *   "pdl"         1 = launches carry the programmatic-dependent-launch attribute [1]
 *   "overlap"     launch layout of the greedy loop: 2 = one stream, the attention kernel of step t+1 runs beside the
 *                 vocabulary layer of step t without waiting for it [2]; 1 = two streams, fork/join; 0 = in order.
 *                 (the attention grid, hence the split-L merge order, differs between 0 and 1/2)
 *   "xbatch"      1 = sat_decode_loop runs its prologue (context projection, initialize) on a stream of the library's
 *                 own into one of two buffer sets, so that it overlaps the decode steps of the previous call [0].
 *                 Contract: the contexts passed to sat_decode_loop are COMPLETE when the call is made (not produced
 *                 by earlier work queued on the same stream).  The pipelined host API does this by itself.
 *   "prologue1"   1 = the pass that packs the contexts for the hoisted projection also takes their mean over the
 *                 locations (one pass over the conv features for initialize and attend/fc_1a) [1]
 *   "chain"       1 = greedy loops at 64-row batches run the three dense layers of a step as phases of ONE persistent
 *                 launch (sat_chain.cu; an experiment, slower than the default chained launches) [0]
 *   "warm"        1 = idle epilogue warps pre-run the epilogue code to warm the instruction caches [1]
 *   "att_wpc"     1 = warp-per-chunk attention kernel for 512-float rows [1]
 *   "l2_w"        L2 policy of every dense weight stream: 1 = evict_first, 2 = evict_last, 3 = evict_normal;
 *                 -1 = evict_first in launches with one row tile (the decode step), evict_last otherwise [-1]
 *   "att_sms", "att_occ", "att_warps", "l2_vocab", "l2_t", "l2_ctx", "l2_prefetch": grid / cache-policy knobs
 *   "profile"     1 = record CUDA events around every eager kernel launch; read back with sat_get_info
 *                 "prof_ns_<family>" / "prof_n_<family>"
 *   "trace"       1 / 2 / 3 = in-kernel globaltimer stamps of a dense launch ("trace_at") / of the attention kernel /
 *                 of every launch of a loop
 * Environment: SAT_PDL=0 creates handles with "pdl" off (for tools that expect one kernel of a stream at a time).
 * A handle expects the GPU to itself while a loop runs: the fused arg-max of the vocabulary layer ends in a grid-wide
 * rendezvous of its one-wave launch (a stuck rendezvous traps with a message after a few seconds). */
int sat_set_option(sat_handle* h, const char* key, int64_t value);
int sat_get_info(sat_handle* h, const char* key, int64_t* value);

/* replaces BaseModel.load's per-variable assign (base_model.py:257-278).  `tf_var_name` is
 * the TF variable name with or without ":0" (e.g. "lstm/lstm_cell/kernel"); `dev` holds the
 * variable in the reference's layout: dense kernels [in, units] (rows=in, cols=units), biases
 * [units] (rows=1), the LSTM kernel [D+E+H, 4H] with column blocks i,j,f,o, the embedding [V,E].
 * The repack into the library's own storage is queued on `stream` (no host synchronisation: a training loop that
 * refreshes the decode weights pays one sync, not twenty): `dev` must stay valid until `stream` has passed this
 * call, and work that uses the weights must be ordered after it (the same stream, or an event). */
int sat_set_weight(sat_handle* h, const char* tf_var_name, const float* dev, int64_t rows, int64_t cols,
                   void* stream);
/* number of variables still missing (0 = ready) */
int sat_weights_missing(sat_handle* h);

/* replaces sess.run([conv_feats, initial_memory, initial_output], {images})
 * (base_model.py:168-170) minus the CNN: projects the contexts (attend fc_1a, model.py:417-420,
 * hoisted out of the step loop) and runs initialize (model.py:239-242, 358-393).
 * contexts [n_img, L, D]; initial_memory / initial_output [n_img, H] may be NULL. */
int sat_prepare_contexts(sat_handle* h, const float* contexts, int32_t n_img, float* initial_memory,
                         float* initial_output, void* stream);

/* replaces sess.run([memory, output, probs], {contexts, last_word, last_memory, last_output})
 * (base_model.py:207-212; graph model.py:258-290).  All of memory/output [B,H] are required;
 * logits / probs [B,V] and alpha [B,L] may be NULL.  `contexts` must be the buffer last given
 * to sat_prepare_contexts with n_img == B (otherwise the projection is redone here). */
int sat_decode_step(sat_handle* h, const float* contexts, const int32_t* last_word, const float* last_memory,
                    const float* last_output, float* memory, float* output, float* logits, float* probs,
                    float* alpha, int32_t B, void* stream);

/* T steps on the device without host round trips: prepare + initialize + T x step, the word fed
 * to step t+1 being argmax of step t (model.py:289) or forced_words[b, t] (teacher forcing,
 * model.py:310).  tokens [B,T] receives the argmax words; logits_all [T,B,V] may be NULL. */
int sat_decode_loop(sat_handle* h, const float* contexts, int32_t B, int32_t T, const int32_t* forced_words,
                    int32_t* tokens, float* logits_all, void* stream);

/* replaces BaseModel.beam_search (base_model.py:163-240) with TopN/CaptionData semantics of
 * utils/misc.py:38-87; `eos_id` stands for vocabulary.words[w] == '.' (base_model.py:229).
 * Outputs per image, sorted by descending score: sentences [n_img, beam, T] (-1 padded),
 * lengths [n_img, beam], scores [n_img, beam] (fp64 products of probabilities,
 * base_model.py:224), n_results [n_img], is_complete [n_img]. */
int sat_beam_search(sat_handle* h, const float* contexts, int32_t n_img, int32_t beam_size, int32_t T,
                    int32_t eos_id, int32_t* sentences, int32_t* lengths, double* scores, int32_t* n_results,
                    int32_t* is_complete, void* stream);

/* Per-word maps: where the model looked for each word and how probable each word was.  Either output may be NULL; a
 * call that requests neither runs exactly what sat_decode_loop / sat_beam_search run.
 * With the default 2-layer attend, alpha does not depend on the LSTM state in inference (model.py:417-436: the score
 * is w2.tanh(fc_1a(ctx)) + w2.tanh(fc_1b(h)), and the second term, the same for every location, cancels in the
 * softmax), so the map of an image is the same for every word, as in the reference; the 1-layer attend gives
 * word-dependent maps.
 *
 * sat_decode_loop_maps: sat_decode_loop plus alphas [T,B,L] (the layout of logits_all; alphas[t] is the alpha of the word emitted at step t)
 * and word_probs [B,T] = softmax(logits of step t)[w], w the word fed to step t+1: the argmax (greedy) or
 * forced_words[b,t] (teacher forced; a forced word outside [0, V) gets probability 0).  A call with maps runs the
 * default launch layouts (never the experimental "chain" = 1 launch). */
int sat_decode_loop_maps(sat_handle* h, const float* contexts, int32_t B, int32_t T, const int32_t* forced_words,
                         int32_t* tokens, float* logits_all, float* alphas, float* word_probs, void* stream);
/* sat_beam_search_maps: sat_beam_search plus, for each returned caption (same order as sentences): alphas [n_img, beam, T, L] and
 * word_probs [n_img, beam, T], zero past lengths[k, j]; scores[k, j] is the product of word_probs[k, j, :len] in
 * step order (fp64).  The first call with maps allocates a history of max_caption_length x max_batch x L floats. */
int sat_beam_search_maps(sat_handle* h, const float* contexts, int32_t n_img, int32_t beam_size, int32_t T,
                         int32_t eos_id, int32_t* sentences, int32_t* lengths, double* scores, int32_t* n_results,
                         int32_t* is_complete, float* alphas, float* word_probs, void* stream);

/* Sampling: captions drawn from the model instead of its arg-max (several different captions per image; sampled
 * captions with the probability of each word for self-critical / REINFORCE fine-tuning and Monte-Carlo scoring).
 * n_img images x num_samples captions each, drawn word by word from softmax(logits / temperature); the sampled word
 * is fed to the next step (<start> = 0 first, like sat_decode_loop).  contexts [n_img, L, D] are shared by the
 * num_samples rows of an image (not replicated).  Row r = image * num_samples + k.
 * tokens [n_img, num_samples, T] (required); word_probs [n_img, num_samples, T] or NULL: softmax(logits of step t)[w]
 * at temperature 1 (the model's own probability of the sampled word w, whatever the temperature).  Without word_probs
 * the vocabulary layer keeps no softmax partials: the draw is all that sampling adds to it.
 * The draw is the Gumbel-max trick, w = argmax_i(logit_i / temperature - log(-log u(seed, r, t, i))), inside the
 * fused arg-max of the vocabulary layer (or the per-row kernel when that layer does not fit one wave); u is a
 * counter-based hash, so the draws are a pure function of (seed, r, t, word): the same call with the same seed gives
 * the same tokens.  Seed and temperature are not part of the CUDA-graph key: a new seed replays the captured graph.
 * Errors: SAT_ERR_INVALID for temperature <= 0 or not finite, num_samples < 1, n_img * num_samples > max_batch, T < 1
 * or a null contexts / tokens (nothing is enqueued); SAT_ERR_UNSUPPORTED for num_samples > 4 (the rows of an image
 * share its contexts in the attention kernels, which take up to 4; draw more captions with further seeds, as
 * CaptionGenerator.sample does). */
int sat_sample_loop(sat_handle* h, const float* contexts, int32_t n_img, int32_t num_samples, int32_t T,
                    float temperature, uint64_t seed, int32_t* tokens, float* word_probs, void* stream);
/* sat_sample_loop_filtered: sat_sample_loop with the two filters of text generation, applied after the temperature.
 * Words of a row rank by (logit desc, index asc).  top_k >= 1 keeps the first top_k words of that order (0, or
 * top_k >= V: all words); top_p in (0, 1) then keeps the shortest prefix, in the same order, of those words whose
 * softmax(logits / temperature), renormalised over them, sums to top_p or more (1: all of them).  At least one word is
 * always kept.  The draw is sat_sample_loop's Gumbel arg-max restricted to the kept words: when the unfiltered draw of
 * the same (seed, r, t) is kept, it is the filtered draw too.  word_probs keep sat_sample_loop's meaning (the model's
 * probability of the word at temperature 1 over the whole vocabulary, not a filtered probability).
 * With a filter on, the vocabulary layer writes the logits and a per-row kernel selects the kept words (integer radix
 * selection; the nucleus mass is summed in 64-bit fixed point, so the result does not depend on the launch) and
 * draws; top_k == 0 && top_p == 1 runs exactly sat_sample_loop.  top_k and top_p, like seed and temperature, are not
 * part of the CUDA-graph key: new values replay the captured graph.
 * Errors: those of sat_sample_loop, and SAT_ERR_INVALID for top_k < 0 or top_p NaN, <= 0 or > 1 (nothing is
 * enqueued). */
int sat_sample_loop_filtered(sat_handle* h, const float* contexts, int32_t n_img, int32_t num_samples, int32_t T,
                             float temperature, int32_t top_k, float top_p, uint64_t seed, int32_t* tokens,
                             float* word_probs, void* stream);
/* the uniform variate behind the Gumbel noise of (seed, row, step, word), u = (bits + 0.5) * 2^-32 in (0, 1), computed
 * on the host (tests rebuild every draw with it) */
double sat_sample_uniform(uint64_t seed, int64_t row, int32_t step, int32_t word);

/* host-buffer forms: copy in, run, copy out, synchronise (what a sess.run caller sees) */
int sat_decode_step_host(sat_handle* h, const float* contexts_host, int32_t contexts_changed,
                         const int32_t* last_word_host, const float* last_memory_host,
                         const float* last_output_host, float* memory_host, float* output_host,
                         float* probs_host, int32_t B, void* stream);
int sat_decode_loop_host(sat_handle* h, const float* contexts_host, int32_t B, int32_t T,
                         const int32_t* forced_words_host, int32_t* tokens_host, void* stream);
/* Pipelined form of sat_decode_loop_host for a stream of batches (what a caption server / the eval loop of
 * base_model.py:94-140 does batch after batch).  submit() enqueues upload (own copy stream) -> loop -> download for
 * staging slot 0 or 1 and returns; wait() blocks until that slot's tokens are in tokens_host.  Submit batch i+1 on
 * the other slot before waiting for batch i and its upload overlaps batch i's decode.  The host buffers must stay
 * valid (and, for true overlap, be pinned) until wait(). */
int sat_decode_loop_host_submit(sat_handle* h, const float* contexts_host, int32_t B, int32_t T,
                                const int32_t* forced_words_host, int32_t* tokens_host, int32_t slot, void* stream);
int sat_decode_loop_host_wait(sat_handle* h, int32_t slot);
int sat_beam_search_host(sat_handle* h, const float* contexts_host, int32_t n_img, int32_t beam_size, int32_t T,
                         int32_t eos_id, int32_t* sentences_host, int32_t* lengths_host, double* scores_host,
                         int32_t* n_results_host, int32_t* is_complete_host, void* stream);

/* individually callable kernels of one step (profiling / unit tests).  Rows = n_img * group;
 * `group` rows of one image share its contexts (beams).
 *   sat_attention_fwd : attend + context vector (model.py:262-264) given the state h [rows,H]: alpha [rows,L]
 *                       (may be NULL) and context [rows,D].  With the 2-layer attend the projection of the contexts
 *                       is cached by contexts pointer and n_img, as for sat_decode_step: after writing new values
 *                       into the same contexts buffer, call sat_prepare_contexts again
 *   sat_lstm_fwd      : embedding lookup + LSTMCell (model.py:272-279) on context [rows,D], last_word [rows],
 *                       last_memory and last_output [rows,H]: writes memory (c) and output (h) [rows,H]
 *   sat_vocab_gemm    : decode (model.py:282-287) of output [rows,H], context [rows,D] and last_word [rows]:
 *                       writes logits [rows,V] and nothing else (no arg-max: words are chosen by the loops)
 * Both gather embedding rows without a range check: every last_word must lie in [0, V).      */
int sat_attention_fwd(sat_handle* h, const float* contexts, const float* output, float* alpha, float* context,
                      int32_t n_img, int32_t group, void* stream);
int sat_lstm_fwd(sat_handle* h, const float* context, const int32_t* last_word, const float* last_memory,
                 const float* last_output, float* memory, float* output, int32_t rows, void* stream);
int sat_vocab_gemm(sat_handle* h, const float* output, const float* context, const int32_t* last_word,
                   float* logits, int32_t rows, void* stream);
/* generic dense layer y = act(x W + b) through the same tensor-core kernel (tests):
 * x [rows,K], w_tf [K,n_out] (TF layout), b [n_out] or NULL, act 0 none / 1 tanh. */
int sat_dense_fwd(sat_handle* h, const float* x, const float* w_tf, const float* b, float* y, int32_t rows,
                  int32_t K, int32_t n_out, int32_t act, int32_t splits, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training step (model.py:250-334 losses, :461-511 optimizer; driver base_model.py:39-68), for the 1- and 2-layer
 * variants of initialize / attend / decode (config.py:15-19; sat_train_var enumerates the variables of the chosen graph).
 * The trainable variables live in ONE flat fp32 device buffer owned by the caller (parameters), with
 * parallel buffers for the gradient and the two Adam slots; sat_train_var describes the layout
 * (TF variable name, offset in floats, TF shape).  A data-parallel step is
 *     sat_train_forward_backward  ->  all-reduce(sum) of `grads` across ranks (NCCL)  ->  sat_train_apply
 * Dropout masks come from a counter-based generator keyed by `seed` (0 = dropout off), so a step is
 * reproducible; ranks must use different seeds.
 * Knobs: sat_set_option "train_tc" 1 = the large products of the step run on the wgmma dense kernel [1], 0 = fp32
 * CUDA-core SGEMM everywhere.  Environment switches, read once per process, for A/B timing (results agree to round-off):
 * SAT_TRAIN_PDL=0 launches the step's kernels without the programmatic-serialization attribute; SAT_TRAIN_DEC_ALL=0 keeps
 * the decode layers inside the time loop (default: one stacked product per layer for all T steps); SAT_TRAIN_SIDE=0 keeps
 * the attend/fc_1a products on the caller's stream (default: a second, low-priority stream of the library's own; 2 / 3:
 * only the forward / only the backward ones);
 * SAT_TRAIN_FUSE_SOFTMAX=0 / 2 un-fuses the softmax kernels (both directions / the backward one only); SAT_TRAIN_FUSE_PACK=0
 * packs the operands of the batch-row products in launches of their own instead of in their producer kernels;
 * SAT_TRAIN_ATTBWD_WAVE=1 runs the attention scorer's backward as one resident wave (a 64-register build of the kernel).
 * params, grads and contexts must be 16-byte aligned (the step reads them with vector loads); every entry point below
 * returns SAT_ERR_INVALID, with nothing enqueued, for a buffer that is not.
 * Word ids outside [0, vocabulary_size) read as zero rows, contribute no gradient and are counted
 * (sat_get_info "train_bad_ids"). */
int sat_train_init(sat_handle* h, int32_t B, int32_t T, float fc_drop_rate, float lstm_drop_rate,
                   float attention_loss_factor, float fc_kernel_regularizer_scale);
int sat_train_num_vars(sat_handle* h);
/* the counter-based dropout generator, U[0,1) with 24 bits: mask = floor(keep + u) (host function, no GPU) */
float sat_train_rng_uniform(uint64_t seed, uint64_t stream, uint64_t index);
/* i in [0, num_vars): name / offset / rows / cols / regularised of variable i; total = floats in the flat buffer */
int sat_train_var(sat_handle* h, int32_t i, const char** name, int64_t* offset, int64_t* rows, int64_t* cols,
                  int32_t* regularised, int64_t* total);
/* replaces the forward+backward half of sess.run(opt_op) (base_model.py:57-60).  contexts [B,L,D], sentences
 * int32 [B,T], masks [B,T]; global_mask_sum / global_batch are the normalisers of the WHOLE (all ranks) batch
 * (model.py:316-318, 324-326).  losses (device, 4 floats): cross_entropy, accuracy, attention, reg.
 * grads is overwritten with this shard's gradient WITHOUT the regulariser term. */
int sat_train_forward_backward(sat_handle* h, const float* params, float* grads, const float* contexts,
                               const int32_t* sentences, const float* masks, int32_t B, int32_t T, uint64_t seed,
                               double global_mask_sum, int32_t global_batch, float* losses, void* stream);
/* the same with the whole-batch mask sum read from DEVICE memory (one double, e.g. the output of an all-reduce
 * queued on `stream` just before): nothing of a data-parallel step then waits for the host. */
int sat_train_forward_backward_dsum(sat_handle* h, const float* params, float* grads, const float* contexts,
                                    const int32_t* sentences, const float* masks, int32_t B, int32_t T, uint64_t seed,
                                    const double* global_mask_sum_dev, int32_t global_batch, float* losses, void* stream);
/* Grouped training step: several captions per image (sampled captions for self-critical training, or the reference
 * captions of an image) with the image's contexts shared by its rows instead of replicated.
 * rows = n_img * group; row r is a caption of image r / group.  sat_train_init(h, B, T, ...) ==
 * sat_train_init_grouped(h, B, 1, T, ...).  What depends on the image alone (context mean, initialize, attend/fc_1a and
 * its stash) is computed once per image, with the init_* and att_ctx dropout masks drawn for n_img rows (n_img * L for
 * att_ctx); every other mask is drawn per row.  The tensor-core attend/fc_1a path needs n_img * L % 128 == 0. */
int sat_train_init_grouped(sat_handle* h, int32_t n_img, int32_t group, int32_t T, float fc_drop_rate,
                           float lstm_drop_rate, float attention_loss_factor, float fc_kernel_regularizer_scale);
/* contexts [n_img, L, D]; sentences / masks [rows, T]; row_weights [rows] or NULL (= 1): row r's cross entropy and its
 * gradient are multiplied by row_weights[r] (e.g. a policy-gradient advantage, any sign; read on the device at run time,
 * so new values in the same buffer replay the captured graph).  Accuracy and the attention loss are not weighted.
 * global_batch counts rows (coverage normaliser); losses[0] = sum_r w_r sum_t m_rt CE_rt / global mask sum.
 * sat_train_forward_backward(_dsum) compute the same with group 1 and NULL weights.
 * Errors: SAT_ERR_INVALID, with nothing enqueued, for group < 1, an (n_img, group, T) other than the one of
 * sat_train_init_grouped, or a null required argument; the values in row_weights are not checked. */
int sat_train_forward_backward_grouped(sat_handle* h, const float* params, float* grads, const float* contexts,
                                       int32_t n_img, int32_t group, const int32_t* sentences, const float* masks,
                                       const float* row_weights, int32_t T, uint64_t seed,
                                       const double* global_mask_sum_dev, int32_t global_batch, float* losses,
                                       void* stream);
/* caption masks of token rows (e.g. sat_sample_loop's output), on the device: masks[r, t] = 1 for t <= the first t'
 * with tokens[r, t'] == eos_id (all T if there is none), else 0; *mask_sum (device double, may be NULL) = their sum.
 * Needs no handle: runs on the current device.  SAT_ERR_INVALID for null tokens / masks, rows < 0 or T < 1. */
int sat_caption_masks(const int32_t* tokens, int32_t rows, int32_t T, int32_t eos_id, float* masks,
                      double* mask_sum, void* stream);
/* CIDEr-D (the semantics of coco-caption's cider_scorer.py and of the CiderD scorer of self-critical training) of
 * word-id captions against their references: the reward of self-critical training and a validation metric.
 * A row (candidate or reference) ends after its first eos_id (which counts as a word), or before its first id < 0
 * (padding) or >= vocabulary_size.  For n = 1..4, v_n(c)[g] = count_c(g) * (log N - log max(1, df(g))) over the n-grams
 * g of c; "length" = the number of bigrams (both reference scorers compute it so); per reference r,
 * s_n = sum over distinct g of c of min(v_n(c)[g], v_n(r)[g]) * v_n(r)[g], divided by |v_n(c)| |v_n(r)| when both are
 * non-zero, times exp(-(len(c) - len(r))^2 / 72); CIDEr-D = 10 * mean over the non-empty references of mean over n of
 * s_n (0 for an image without one).  df(g) = number of corpus images whose references, taken together, contain g, and
 * N = the corpus's number of images: self-critical training builds the table from the training references,
 * coco-caption from the evaluated set's own references.
 *
 * sat_cider_create: the document-frequency table of a corpus refs_host [n_img, R, T_ref] int32 on the HOST (an
 * all-padding row is no reference), built on the host and uploaded to the device current at the call (a table of
 * about 12 bytes x 2 x the corpus's distinct n-grams).  SAT_ERR_INVALID for n_img < 1, R < 1, T_ref < 1 or
 * vocabulary_size outside [2, 65535] (an n-gram key holds four 16-bit word ids).
 * sat_cider_d: scores [n_img, C] (device float) = CIDEr-D of candidates [n_img, C, T] against refs [n_img, R, T_ref]
 * (device int32), with the eos_id, vocabulary_size and table of `c`.  One CTA per image: the references' n-gram
 * weights are formed once and shared by the C candidates.  fp64 arithmetic in a fixed summation order: the result is
 * bit-reproducible.  Asynchronous on `stream`.  Limits: R <= 8, T <= 64, T_ref <= 64 (SAT_ERR_UNSUPPORTED beyond);
 * SAT_ERR_INVALID for null pointers, n_img < 0 or C, T, R, T_ref < 1.  Nothing is enqueued on an error. */
typedef struct sat_cider sat_cider;
int sat_cider_create(const int32_t* refs_host, int64_t n_img, int32_t R, int32_t T_ref, int32_t eos_id,
                     int32_t vocabulary_size, sat_cider** out);
void sat_cider_destroy(sat_cider* c);
int sat_cider_d(const sat_cider* c, const int32_t* candidates, int32_t n_img, int32_t C, int32_t T,
                const int32_t* refs, int32_t R, int32_t T_ref, float* scores, void* stream);

/* adds the L2-regulariser gradient, clips by the global norm (clip_gradients, config.py:36) and applies TF Adam
 * (config.py:32-43).  step counts from 1.  grad_norm (device, 1 float, may be NULL) receives the squared norm. */
int sat_train_apply(sat_handle* h, float* params, float* grads, float* adam_m, float* adam_v, int64_t step, float lr,
                    float beta1, float beta2, float epsilon, float clip, float* grad_norm, void* stream);

/* The optimizer of model.py:479-503 as plain data (field names of config.py:30-43).  kind: SAT_OPT_*.
 *   Adam      tf.train.AdamOptimizer(learning_rate, beta1, beta2, epsilon)              slots: m, v
 *   RMSProp   tf.train.RMSPropOptimizer(learning_rate, decay, momentum, epsilon, centered)
 *                                                   slots: rms (STARTS AT ONE: sat_train_fill), mg (centered only), momentum
 *   Momentum  tf.train.MomentumOptimizer(learning_rate, momentum, use_nesterov)        slots: accumulator
 *   SGD       tf.train.GradientDescentOptimizer(learning_rate)                          slots: none
 * clip_gradients: optimize_loss(clip_gradients=...) = clip_by_global_norm, applied for every optimizer.
 * (The reference passes an Optimizer INSTANCE to tf.contrib.layers.optimize_loss, so its learning_rate_decay_fn only feeds
 * the "learning_rate" summary: the optimizer keeps initial_learning_rate.  The facade reproduces that and offers the
 * decayed rate as an option; this ABI simply takes the rate to use.) */
#define SAT_OPT_ADAM 0
#define SAT_OPT_RMSPROP 1
#define SAT_OPT_MOMENTUM 2
#define SAT_OPT_SGD 3
typedef struct sat_optimizer {
    int32_t kind;
    float learning_rate, beta1, beta2, epsilon, decay, momentum;
    int32_t centered, use_nesterov;
    float clip_gradients;
} sat_optimizer;
/* sat_train_apply for any of the four optimizers; slot0..2 in the order listed above (unused ones may be NULL). */
int sat_train_apply_opt(sat_handle* h, float* params, float* grads, float* slot0, float* slot1, float* slot2, int64_t step,
                        const sat_optimizer* opt, float* grad_norm, void* stream);
/* buf[0..n) = value on the device (initial value of an optimizer slot) */
int sat_train_fill(sat_handle* h, float* buf, float value, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SAT_B200_H_ */
