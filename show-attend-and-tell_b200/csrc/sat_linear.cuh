// sat_linear.cuh — descriptors of the small-batch dense layer kernels
// (tf.layers.dense / LSTMCell matmul of the reference: utils/nn.py:85-105,
// model.py:276-279, 438-459) as executed on sm_90a.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>

namespace sat {

constexpr int kBK = 64;                                  // K elements per pipeline stage
constexpr int kTileN = 128;                              // outputs per CTA tile (wgmma M of two warpgroups)
constexpr int kWHalfBytes = kTileN * kBK * 2;            // one bf16 half (hi or lo) of a W tile
constexpr int kWStageBytes = 2 * kWHalfBytes;            // hi + lo, contiguous in the packed image
constexpr int kLinThreads = 320;                         // warps 0-7 MMA / X-producer / epilogue, warp 8 TMA, warp 9 X TMA
constexpr int kLinProducers = 256;                       // the consumer warps 0-7 (two warpgroups)
constexpr int kMaxRowTile = 128;                         // batch rows per CTA tile (wgmma N), multiple of 16: the
                                                         // accumulator (N / 2 registers per consumer thread) fits
constexpr int kMaxSeg = 3;
constexpr int kMaxProb = 4;

enum LinEpilogue : int {
    kEpiBias = 0,      // out = acc + bias                      (decode fc_2 / fc, initialize fc_*2)
    kEpiBiasTanh = 1,  // out = tanh(acc + bias)                (attend fc_1a/fc_1b, decode fc_1, initialize fc_*1)
    kEpiLstm = 2,      // TF LSTMCell gates i,j,f,o -> (c, h)   (model.py:278)
    kEpiNone = 3       // out = acc (bias-free dense: attend fc_a / fc_b, model.py:403-413)
};

// One K-segment of the activation operand: X[b, k0 + j] = ptr[row(b) * ld + j],
// row(b) = gather ? gather[b] (embedding lookup, model.py:273) : b / row_div.
struct LinSeg {
    const float* ptr;
    const int32_t* gather;
    int ld;
    int width;   // multiple of 8
    int row_div; // >= 1; b / row_div selects the source row (beams sharing one image row)
    const uint8_t* pa;  // same operand already packed by its producer (see PackedAct), or null
};

// A "packed activation": an fp32 [rows, width] tensor (width % 64 == 0) kept by its PRODUCER kernel in
// the bf16 hi/lo MMA operand image  [n_row_tiles][width/64][hi|lo][row_tile x 64 bf16]  so that the
// consuming dense layer fetches its X stages by TMA with no conversion pass.
__host__ __device__ __forceinline__ size_t pa_stage_bytes(int row_tile) { return (size_t)row_tile * kBK * 2 * 2; }

struct SampleParams;   // sampling loop: see sample_key below

struct LinProblem {
    LinSeg seg[kMaxSeg];
    int nseg;
    int K;          // sum of widths
    int k_blocks;   // ceil(K / kBK)
    int rows;       // valid activation rows (batch)
    int row_tile;   // activation rows per CTA = wgmma N, multiple of 16, <= kMaxRowTile
    int n_row_tiles;
    int n_out;      // valid outputs
    int n_tiles;    // ceil(n_out / 128)
    int splits;     // split-K factor = thread-block cluster size (1, 2, 4 or 8)
    const uint8_t* wpack;  // [n_tiles][k_blocks][hi|lo][128 x 64 bf16, canonical K-major MMA operand layout]
    int l2_w;              // L2 eviction policy of the weight stream (see l2_policy)
    const float* bias;     // packed output order, n_tiles*128 entries (zero padded); may be null for kEpiNone
    uint8_t* xpack;        // x_mode 1: packed activations [n_row_tiles][k_blocks][hi|lo][row_tile x 64 bf16]
    unsigned* xbar;        // x_mode 1: grid barrier {count, generation}
    int epi;
    float* out;            // [rows, ldo]
    int ldo;
    int accumulate;        // out += result instead of out = result (training: gradient accumulated over time steps)
    const float* c_in;     // LSTM: [rows, H]
    float* c_out;
    float* h_out;
    int H;
    // optional fused greedy argmax over the outputs (decode fc_2 -> prediction, model.py:289):
    // per-tile candidates, then the last CTA of the problem picks the word of every row
    unsigned long long* am_key;   // [n_row_tiles * n_tiles * row_tile] candidates, see argmax_key
    unsigned* am_ctr;      // zero between launches
    int32_t* am_tokens;    // [rows, am_tokens_ld] or null
    int am_tokens_ld;
    int am_step;
    int32_t* am_next_word; // [rows] or null
    const int32_t* am_forced;  // teacher-forced next words [rows, am_forced_ld] or null
    int am_forced_ld;
    // optional probability of the word fed to the next step, softmax(logits)[w] (w = forced word or the arg-max),
    // from per-tile partials (tile maximum = value half of the key, sum of exp(v - max)) merged online.  Needs the
    // word-probability instance of the kernel (lin_launch picks it when am_probs is set).
    float* am_probs;       // [rows, am_probs_ld] or null
    int am_probs_ld;
    float* am_sum;         // laid out like am_key: sum over the tile row of exp(v - tile maximum)
    float* am_wlogit;      // [rows] teacher forcing: logit of the forced word, stored by the tile that owns it
    uint8_t* out_pa;      // optional packed copy of the output for the next dense layer (width n_out)
    // fused epilogue of the vocabulary layer in loops: pack the embedding row of the chosen next word
    const float* am_emb;   // [V, E] embedding matrix or null
    int am_E;
    uint8_t* am_emb_pa;    // packed [rows, E]
    int cta_begin;         // first CTA of this problem in the grouped grid
    int cta_count;
    // optional sampling (sat_sample_loop): the fused arg-max picks argmax_i(logit_i / temperature + g(seed, row, step, i))
    // (Gumbel-max: a draw from softmax(logits / temperature)); the softmax partials stay on the raw logits.  Runs a
    // sampling instance of the kernel (lin_launch picks it when smp is set); with am_probs also am_sum and am_smp.
    const SampleParams* smp;   // device {seed, 1 / temperature}: read at run time, so graphs replay any seed
    float2* am_smp;        // laid out like am_key: {raw tile maximum, raw logit of the tile's sampled candidate}
};

struct LinLaunch {
    LinProblem p[kMaxProb];
    int nprob;
    int layout_mode;  // 0 = no-swizzle (interleaved 8x16B core matrices), 1 = 128B swizzle
    int stages;
    unsigned long long* dbg;  // optional [grid][16] timeline stamps
    unsigned long long* tl;   // optional {min start, max end} of this launch
    int pdl;          // launched with programmatic stream serialization (see pdl_wait)
    int w_dynamic;    // the weight operand was written by the preceding kernel (training): no weight fetch before the wait
    int l2_prefetch;  // (with pdl) prefetch the CTA's whole weight stream into L2 before waiting for the predecessor
    int warm_epilogue;  // idle epilogue warps pre-run the epilogue code (no side effects) to warm the instruction caches
    int x_mode;       // 0 = producer warps convert X per stage; 1 = cooperative pre-pack + TMA (grid <= #SMs);
                      // 2 = every operand segment arrives packed from its producer (TMA from t = 0)
};

// byte offset of the 16-byte group (row r, k-group kg in [0,8)) inside a [rows x 64] bf16
// K-major operand tile.  Both modes place 8-row groups 1024 B apart.
__host__ __device__ __forceinline__ uint32_t mma_tile_off(int mode, int r, int kg) {
    return mode == 0 ? (uint32_t)((r >> 3) * 1024 + kg * 128 + (r & 7) * 16)
                     : (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((kg ^ (r & 7)) * 16));
}

// store one fp32 value into a packed activation (2-byte hi and lo stores)
#ifdef __CUDACC__
__device__ __forceinline__ void pa_store(uint8_t* pa, int mode, int row_tile, int kblocks, int b, int col, float v) {
    const int rt = b / row_tile, r = b - rt * row_tile;
    const int kb = col >> 6, kg = (col & 63) >> 3, e = col & 7;
    const size_t half = (size_t)row_tile * kBK * 2;
    uint8_t* dst = pa + ((size_t)rt * kblocks + kb) * 2 * half + mma_tile_off(mode, r, kg) + e * 2;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    const __nv_bfloat16 l = __float2bfloat16_rn(v - __bfloat162float(h));
    *reinterpret_cast<__nv_bfloat16*>(dst) = h;
    *reinterpret_cast<__nv_bfloat16*>(dst + half) = l;
}
// four consecutive outputs (col % 4 == 0): one 8-byte store per half
__device__ __forceinline__ void pa_store4(uint8_t* pa, int mode, int row_tile, int kblocks, int b, int col, const float* v) {
    const int rt = b / row_tile, r = b - rt * row_tile;
    const int kb = col >> 6, kg = (col & 63) >> 3, e = col & 7;
    const size_t half = (size_t)row_tile * kBK * 2;
    uint8_t* dst = pa + ((size_t)rt * kblocks + kb) * 2 * half + mma_tile_off(mode, r, kg) + e * 2;
    uint32_t h[2], l[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const __nv_bfloat16 h0 = __float2bfloat16_rn(v[2 * i]), h1 = __float2bfloat16_rn(v[2 * i + 1]);
        const __nv_bfloat16 l0 = __float2bfloat16_rn(v[2 * i] - __bfloat162float(h0));
        const __nv_bfloat16 l1 = __float2bfloat16_rn(v[2 * i + 1] - __bfloat162float(h1));
        h[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        l[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    *reinterpret_cast<uint2*>(dst) = make_uint2(h[0], h[1]);
    *reinterpret_cast<uint2*>(dst + half) = make_uint2(l[0], l[1]);
}
// arg-max candidate as one ordered 64-bit key: larger value wins, then the smaller index (tf.argmax keeps the
// first maximum).  0 is below every real candidate.
__device__ __forceinline__ unsigned long long argmax_key(float v, int idx) {
    const unsigned bits = __float_as_uint(v + 0.0f);                      // -0 -> +0
    const unsigned ord = (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u);
    return ((unsigned long long)ord << 32) | (unsigned long long)(0xffffffffu - (unsigned)idx);
}
__device__ __forceinline__ int argmax_key_index(unsigned long long key) { return (int)(0xffffffffu - (unsigned)(key & 0xffffffffull)); }
__device__ __forceinline__ float argmax_key_value(unsigned long long key) {
    const unsigned ord = (unsigned)(key >> 32);
    return __uint_as_float((ord & 0x80000000u) ? (ord & 0x7fffffffu) : ~ord);
}
// online-softmax merge of (max, sum of exp(v - max)) pairs; (-inf, 0) is the empty pair
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
    const float M = fmaxf(m, m2);
    if (M == -INFINITY) return;
    s = s * expf(m - M) + s2 * expf(m2 - M);
    m = M;
}
#endif

constexpr int kAmSmemWords = 1024;   // rows whose chosen word the last CTA keeps in shared memory

// Counter-based dropout masks of the training path (sat_train.cu): element `idx` of mask stream `stream` is kept
// when floor(keep + U) == 1, U = rng_u24(seed, stream, idx) in [0, 1) with 24 bits (oracle/train_ref.py:uniform24 is
// the same function in numpy).  A 32-bit integer hash (two multiplies, three xor-shifts; the stream key enters before
// the first and between the two multiplies) — the masks are regenerated wherever they are needed instead of being
// stored, so the generator is on the critical path of the element-wise kernels.  The packing kernels below can
// apply such a mask while they convert, so a dropped copy of a large operand is never materialised in fp32.
struct DropKey {
    uint32_t k0, k1;
};
__host__ __device__ inline DropKey drop_key(unsigned long long seed, unsigned long long stream) {
    const unsigned long long K = seed ^ (stream * 0x9E3779B97F4A7C15ull);
    return DropKey{(uint32_t)K, (uint32_t)(K >> 32)};
}
__host__ __device__ inline uint32_t rng_bits24(DropKey k, unsigned long long idx) {
    uint32_t x = (uint32_t)idx ^ k.k0;
    x ^= x >> 16;
    x *= 0x21F0AAADu;
    x ^= x >> 15;
    x += k.k1 ^ ((uint32_t)(idx >> 32) * 0x9E3779B1u);
    x *= 0x735A2D97u;
    x ^= x >> 15;
    return x >> 8;
}
__host__ __device__ inline float rng_u24(unsigned long long seed, unsigned long long stream, unsigned long long idx) {
    return (float)rng_bits24(drop_key(seed, stream), idx) * 5.9604644775390625e-08f;  // 2^-24
}
__host__ __device__ inline float drop_scale(unsigned long long seed, unsigned long long stream, unsigned long long idx, float keep) {
    // x / keep * floor(keep + U), floor(keep + U) in {0, 1}
    return keep + rng_u24(seed, stream, idx) >= 1.0f ? 1.0f / keep : 0.0f;
}
// The same mask with the per-element work reduced to the hash and one integer compare: kt is the smallest 24-bit
// count k with fl32(keep + k * 2^-24) >= 1 (the sum is monotone in k), so "kept" <=> rng_bits24 >= kt, bit for bit
// the float formula above.  Built once per thread.
struct DropGen {
    DropKey k;
    uint32_t kt;
    float inv;
    __device__ __forceinline__ float scale(unsigned long long idx) const { return rng_bits24(k, idx) >= kt ? inv : 0.0f; }
};
__host__ __device__ inline DropGen drop_gen(unsigned long long seed, unsigned long long stream, float keep) {
    DropGen g;
    g.k = drop_key(seed, stream);
    g.inv = 1.0f / keep;
    const float c = ceilf((1.0f - keep) * 16777216.0f);
    uint32_t kt = c > 0.0f ? (uint32_t)c : 0u;
    if (kt > (1u << 24)) kt = 1u << 24;
    while (kt > 0 && keep + (float)(kt - 1) * 5.9604644775390625e-08f >= 1.0f) --kt;
    while (kt < (1u << 24) && keep + (float)kt * 5.9604644775390625e-08f < 1.0f) ++kt;
    g.kt = kt;
    return g;
}
// Counter-based generator of the sampling loop (sat_sample_loop): the uniform variate of (seed, row, step, word) is
// u = (bits + 0.5) * 2^-32, strictly inside (0, 1), with bits a 32-bit hash; g = -log(-log u) is its Gumbel(0, 1) noise.
// (seed, row, step) is mixed once per row by two rounds of splitmix64 into a 64-bit key; each word then costs one
// keyed 32-bit hash (lowbias32 with the key's halves entering before the first and between the two multiplies, a
// bijection of the word for a given key).  sat_sample_uniform is this function on the host.
// top_k / top_p are the filters of sat_sample_loop_filtered (0 / 1: off), read only by the filtered per-row kernel.
struct SampleParams {
    unsigned long long seed;
    float inv_tau;          // 1 / temperature
    float pad;
    int top_k;              // draw among the top_k most probable words (0 or >= V: all)
    float top_p;            // ... and among the smallest prefix of those whose probability mass reaches top_p (1: all)
};
struct SampleKey {
    uint32_t k0, k1;
};
__host__ __device__ inline unsigned long long splitmix64(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__host__ __device__ inline SampleKey sample_key(unsigned long long seed, long long row, int step) {
    const unsigned long long z = splitmix64(seed ^ splitmix64(((unsigned long long)row << 32) | (uint32_t)step));
    return SampleKey{(uint32_t)z, (uint32_t)(z >> 32)};
}
__host__ __device__ inline uint32_t sample_bits(SampleKey k, int word) {
    uint32_t x = (uint32_t)word ^ k.k0;
    x ^= x >> 16;
    x *= 0x7FEB352Du;
    x ^= x >> 15;
    x += k.k1;
    x *= 0x846CA68Bu;
    x ^= x >> 16;
    return x;
}
#ifdef __CUDACC__
// g = -log(e), e = -log(u) ~ Exp(1), in fp32 without losing the tail: for u >= 1/2 the complement w = 1 - u =
// (~bits + 0.5) * 2^-32 is formed exactly and e = -log1p(-w) — its series for w < 1/16 (relative error < 1e-8) — so
// the largest draws keep their 32-bit resolution (g up to 22.9; a float u would stop at 16.6).  Two fast logarithms
// (MUFU; absolute error ~4e-7 near 1, relative ~3 ulp elsewhere) and a short polynomial per draw, branch free: this
// runs once per logit in the vocabulary layer's epilogue.
__device__ __forceinline__ float sample_gumbel(uint32_t bits) {
    const bool top = (bits >> 31) != 0u;
    const float w = fmaf((float)(top ? ~bits : bits), 2.3283064365386963e-10f, 1.1641532182693481e-10f);  // u, or 1 - u
    const float l = -__logf(top ? 1.0f - w : w);
    const float s = w * fmaf(w, fmaf(w, fmaf(w, fmaf(w, fmaf(w, 1.0f / 6, 0.2f), 0.25f), 1.0f / 3), 0.5f), 1.0f);
    return -__logf(top && w < 0.0625f ? s : l);
}
#endif

struct DropSpec {          // seedp == nullptr or *seedp == 0: no dropout
    const unsigned long long* seedp;
    unsigned long long stream;
    float keep;
};

struct PackJob {           // fp32 rows (optionally gathered) -> packed activation
    const float* src;
    const int32_t* gather;
    int ld, width, rows, row_tile;
    uint8_t* pa;
    int k_blocks;   // K blocks per row tile of the destination (0 = width / 64).  Larger than width / 64 when the
                    // consumer rounds a ragged width up; the caller keeps the unwritten tail of the last block zero.
};
// drop (optional) applies to every job: mask index = row * width + column of the (un-gathered) source row
// pdl: launch with the programmatic-serialization attribute (the kernel then waits for its predecessor itself and
// lets its successor launch early; used by the training step, whose neighbours all follow that convention)
cudaError_t pack_rows_launch(const PackJob* jobs, int njobs, int layout_mode, cudaStream_t st, const DropSpec* drop = nullptr,
                             int pdl = 0);

// ------------------------------------------------------------------------------------------------------------
// Chained launch (sat_chain.cu): the dense layers of ONE decode step of the greedy loop — LSTM -> [decode fc_1 ||
// attend fc_1b of the next step] -> vocabulary layer + arg-max — as the phases of one persistent launch (one CTA per
// SM).  A phase needs the outputs of ALL CTAs of the phase before it (h, then t = tanh(fc_1)), so phases meet at
// grid-wide arrival counters in global memory; what a separate launch per layer cannot do and this does: every CTA is
// resident from the start, and its TMA lane streams the (immutable) weights of its next tile into the pipeline
// stages as they free up, i.e. under the epilogue and the rendezvous of the current phase.
//   * all operands arrive packed (x_mode 2 of lin_mma_kernel), one row tile (rows <= row_tile <= 64);
//   * split-K partial tiles meet in a global (L2 resident) scratch buffer behind a per-tile arrival counter, summed in
//     fixed split order (bit-identical to the cluster / DSMEM reduction of lin_mma_kernel);
//   * arg-max of the vocabulary phase: one atomicMax per (row, tile) on the ordered 64-bit key; every CTA but the
//     last to arrive exits at once (its SM is free for the next launch); the last arriver records the words and packs
//     their embedding rows for the next step.
// Counters are monotonic: the host zeroes them at the start of a loop and passes the expected values per launch.
constexpr int kChainMaxPhase = 3;
constexpr int kChainMaxTiles = 128;
struct ChainPhase {
    LinProblem p[2];
    int nprob;
    int ctas;              // CTAs with a tile in this phase (blockIdx.x < ctas)
};
struct LinChain {
    ChainPhase ph[kChainMaxPhase];
    int nphase;
    int layout_mode, stages, l2_w, pdl, row_tile;
    unsigned* ctr;         // [kChainMaxPhase] CTAs that finished phase i (since the counters were zeroed)
    unsigned target[kChainMaxPhase];   // value of ctr[i] that means "phase i of THIS launch is complete"
    unsigned* tile_ctr;    // [kChainMaxPhase][kChainMaxTiles] split-K arrivals per (phase, tile)
    unsigned tile_target[kChainMaxPhase];   // value of a tile counter of phase i that means "every split of THIS launch arrived"
                                            // (= split factors of the phase summed over the launches since the zeroing)
    float* scratch;        // [grid][row_tile x 128] split-K partial tiles (cluster == 1 only)
    int cluster;           // > 1: the launch is cut into thread-block clusters of this size and the splits of a tile (all in
                           // one cluster) exchange their partial tiles through distributed shared memory behind a pair
                           // of mbarriers per phase; 1: through `scratch` in L2 behind the tile counters
    unsigned long long* tl;   // optional timeline cells (see tl_begin)
    unsigned long long* dbg;  // optional [grid][16] per-CTA stamps
    int dbg_mode;             // 0: phase milestones; 1: phase 0 per K block (slots 0-7 operands landed, 8-15 weight copy issued)
};
size_t lin_chain_smem_bytes(int row_tile, int stages);
int lin_chain_pick_stages(int row_tile);
int lin_chain_max_clusters(int row_tile, int stages, int cluster);
cudaError_t lin_chain_launch(const LinChain& C, int grid, cudaStream_t st);

size_t lin_smem_bytes(int row_tile, int stages);
int lin_pick_stages(int row_tile);
cudaError_t lin_launch(const LinLaunch& L, cudaStream_t st, bool use_simt);
// drop (optional): mask index = k * n_out + column of the source
cudaError_t lin_repack_weight(const float* w_tf, int K, int n_out, int perm_H, uint8_t* wpack, int layout_mode,
                              cudaStream_t st, const DropSpec* drop = nullptr, int pdl = 0);
cudaError_t lin_repack_bias(const float* b_tf, int n_out, int perm_H, float* bias_packed, cudaStream_t st);
cudaError_t lin_init_attrs();
int device_sm_count();   // SMs of the current device (sizes grids and split factors)

}  // namespace sat
