// sat_rows.cu — per-row vocabulary kernels and the device-side beam bookkeeping.
//   softmax / argmax over V            model.py:288-289
//   top-(beam+1) words per row         base_model.py:215-219
//   TopN / CaptionData heap updates    base_model.py:222-232, utils/misc.py:38-87
#include "sat_common.cuh"
#include "sat_linear.cuh"
#include "sat_rows.cuh"

namespace sat {

constexpr int kRowThreads = 256;

struct ValIdx {
    float v;
    int i;
};
// ordering of the reference's stable descending sort (base_model.py:217-218) and of
// tf.argmax (first maximum): larger value first, then lower index.
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ ValIdx block_best(ValIdx x, ValIdx* sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, x.v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, x.i, o);
        if (better(ov, oi, x.v, x.i)) { x.v = ov; x.i = oi; }
    }
    __syncthreads();
    if (lane == 0) sm[warp] = x;
    __syncthreads();
    ValIdx r = sm[0];
    for (int w = 1; w < kRowThreads / 32; ++w)
        if (better(sm[w].v, sm[w].i, r.v, r.i)) r = sm[w];
    return r;
}

__device__ __forceinline__ float block_sum(float x, float* sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    x = warp_sum(x);
    __syncthreads();
    if (lane == 0) sm[warp] = x;
    __syncthreads();
    float r = 0.f;
    for (int w = 0; w < kRowThreads / 32; ++w) r += sm[w];
    return r;
}

// One block per row.  The row is read from global memory ONCE into shared memory (CACHED: V % 4 == 0 and 4*V bytes
// of dynamic shared memory available) and the three passes — arg-max, sum of exponentials, probabilities + top-k
// — run on that copy in small ROLLED loops (this kernel runs once per step from a cold instruction cache: a
// fully unrolled register-cached version executed 6 k instructions per warp and was instruction-fetch bound).
// SMP: sampling (RowsParams::sample) — best ranks logit / temperature + Gumbel noise, the draw of the fused vocabulary
// layer (sat_linear.cu) for the same (seed, row, step, word); m stays the raw row maximum.  An instance of its own.
template <bool CACHED, bool SMP = false>
__global__ void __launch_bounds__(kRowThreads) rows_softmax_kernel(const RowsParams p) {
    extern __shared__ __align__(16) float row_s[];
    __shared__ ValIdx sm_vi[kRowThreads / 32];
    __shared__ float sm_f[kRowThreads / 32];
    const int row = blockIdx.x;
    const float* x = p.logits + (size_t)row * p.V;
    const int V = p.V, n4 = V >> 2;
    const float4* src4 = CACHED ? reinterpret_cast<const float4*>(row_s) : reinterpret_cast<const float4*>(x);

    ValIdx best = {-INFINITY, 0x7fffffff};
    if constexpr (SMP) {
        const SampleKey sk = sample_key(p.sample->seed, row, p.step);
        const float itau = p.sample->inv_tau;
        float mr = -INFINITY;
        auto offer = [&](float v, int i) {
            mr = fmaxf(mr, v);
            const float g = fmaf(v, itau, sample_gumbel(sample_bits(sk, i)));
            if (better(g, i, best.v, best.i)) { best.v = g; best.i = i; }
        };
        if (CACHED) {
            const float4* x4 = reinterpret_cast<const float4*>(x);
            float4* d4 = reinterpret_cast<float4*>(row_s);
#pragma unroll 1
            for (int i4 = threadIdx.x; i4 < n4; i4 += kRowThreads) {
                const float4 v = x4[i4];
                d4[i4] = v;
                offer(v.x, 4 * i4); offer(v.y, 4 * i4 + 1); offer(v.z, 4 * i4 + 2); offer(v.w, 4 * i4 + 3);
            }
        } else {
#pragma unroll 1
            for (int i = threadIdx.x; i < V; i += kRowThreads) offer(x[i], i);
        }
        best = block_best(best, sm_vi);
        const ValIdx mx = block_best(ValIdx{mr, 0}, sm_vi);
        if (threadIdx.x == 0) {
            if (p.tokens) p.tokens[(size_t)row * p.tokens_ld + p.step] = best.i;
            if (p.next_word) p.next_word[row] = best.i;
        }
        if (!p.word_probs) return;
        const float m = mx.v;
        float s = 0.f;
#pragma unroll 1
        for (int i = threadIdx.x; i < V; i += kRowThreads) s += expf((CACHED ? row_s[i] : x[i]) - m);
        s = block_sum(s, sm_f);
        if (threadIdx.x == 0)   // (a row of NaN logits picks no word: probability 0, no read past the row)
            p.word_probs[(size_t)row * p.tokens_ld + p.step] = (best.i >= 0 && best.i < V) ? expf(x[best.i] - m) / s : 0.f;
        return;
    }
    if (CACHED) {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* d4 = reinterpret_cast<float4*>(row_s);
#pragma unroll 2
        for (int i4 = threadIdx.x; i4 < n4; i4 += kRowThreads) {
            const float4 v = x4[i4];
            d4[i4] = v;
            const int i = 4 * i4;
            if (better(v.x, i, best.v, best.i)) { best.v = v.x; best.i = i; }
            if (better(v.y, i + 1, best.v, best.i)) { best.v = v.y; best.i = i + 1; }
            if (better(v.z, i + 2, best.v, best.i)) { best.v = v.z; best.i = i + 2; }
            if (better(v.w, i + 3, best.v, best.i)) { best.v = v.w; best.i = i + 3; }
        }
    } else {
        for (int i = threadIdx.x; i < V; i += kRowThreads) {
            const float v = x[i];
            if (better(v, i, best.v, best.i)) { best.v = v; best.i = i; }
        }
    }
    best = block_best(best, sm_vi);       // (its barriers also publish row_s)
    const float m = best.v;
    if (threadIdx.x == 0) {
        if (p.argmax) p.argmax[row] = best.i;
        if (p.tokens) p.tokens[(size_t)row * p.tokens_ld + p.step] = best.i;
        if (p.next_word) p.next_word[row] = p.forced ? p.forced[(size_t)row * p.forced_ld + p.step] : best.i;
    }
    if (!p.probs && p.topk == 0 && !p.word_probs) return;  // greedy / teacher-forced loops only need the argmax

    float s = 0.f;
    if (CACHED) {
#pragma unroll 1
        for (int i4 = threadIdx.x; i4 < n4; i4 += kRowThreads) {
            const float4 v = src4[i4];
            s += expf(v.x - m) + expf(v.y - m) + expf(v.z - m) + expf(v.w - m);
        }
    } else {
        for (int i = threadIdx.x; i < V; i += kRowThreads) s += expf(x[i] - m);
    }
    s = block_sum(s, sm_f);
    const float inv = 1.0f / s;
    if (p.word_probs) {
        if (threadIdx.x == 0) {
            const int w = p.forced ? p.forced[(size_t)row * p.forced_ld + p.step] : best.i;
            p.word_probs[(size_t)row * p.tokens_ld + p.step] = (w >= 0 && w < V) ? expf(x[w] - m) * inv : 0.f;
        }
        if (!p.probs && p.topk == 0) return;
    }

    // probabilities + thread-local top-kMaxTopK, kept sorted by (prob desc, index asc) with a compare-and-swap
    // chain on registers (static indices only)
    float tv[kMaxTopK];
    int ti[kMaxTopK];
#pragma unroll
    for (int k = 0; k < kMaxTopK; ++k) { tv[k] = -1.f; ti[k] = 0x7fffffff; }
    auto offer = [&](float pv, int i) {
        if (!better(pv, i, tv[kMaxTopK - 1], ti[kMaxTopK - 1])) return;
#pragma unroll
        for (int k = 0; k < kMaxTopK; ++k) {
            if (better(pv, i, tv[k], ti[k])) {
                const float fv = tv[k]; const int fi = ti[k];
                tv[k] = pv; ti[k] = i;
                pv = fv; i = fi;
            }
        }
    };
    float* pr = p.probs ? p.probs + (size_t)row * V : nullptr;
    const int n_el = CACHED ? V : 0;
#pragma unroll 1
    for (int i = threadIdx.x; i < n_el; i += kRowThreads) {      // element-wise: one copy of `offer` in the binary
        const float pv = expf(row_s[i] - m) * inv;
        if (pr) pr[i] = pv;
        if (p.topk > 0) offer(pv, i);
    }
    if (!CACHED) {
#pragma unroll 1
        for (int i = threadIdx.x; i < V; i += kRowThreads) {
            const float pv = expf(x[i] - m) * inv;
            if (pr) pr[i] = pv;
            if (p.topk > 0) offer(pv, i);
        }
    }
    if (p.topk > 0) {
#pragma unroll 1
        for (int k = 0; k < p.topk; ++k) {
            ValIdx cnd;
            cnd.v = tv[0];
            cnd.i = ti[0];
            const ValIdx w = block_best(cnd, sm_vi);
            if (w.i == cnd.i && w.v == cnd.v && cnd.i != 0x7fffffff) {   // this thread's head won: pop it
#pragma unroll
                for (int q = 0; q + 1 < kMaxTopK; ++q) { tv[q] = tv[q + 1]; ti[q] = ti[q + 1]; }
                tv[kMaxTopK - 1] = -1.f;
                ti[kMaxTopK - 1] = 0x7fffffff;
            }
            if (threadIdx.x == 0) {
                p.topk_idx[(size_t)row * p.topk + k] = w.i;
                p.topk_p[(size_t)row * p.topk + k] = w.v;
            }
        }
    }
}

// ------------------------------------------------------------ filtered sampling (top-k / nucleus)
// Words rank by (logit desc, index asc), the order of better().  Selection runs on order-preserving uint32 keys of the
// raw logits (a larger float has a larger key; -0 is keyed as +0, so equal logits have equal keys) in three radix
// digits of 11, 11 and 10 bits, with one 2048-bin histogram in shared memory.
constexpr int kFiltBins = 2048;
constexpr int kFiltBinsPerThread = kFiltBins / kRowThreads;

__device__ __forceinline__ uint32_t filt_key(float v) {
    const uint32_t u = __float_as_uint(v == 0.f ? 0.f : v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float filt_unkey(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// a word's nucleus mass: exp((x - max) / temperature) in 32.32 fixed point (at most 2^32 per word, so sums over any
// V < 2^32 fit in 64 bits).  Integer sums are exact, hence independent of the order of the atomics.  NaN weighs 0.
__device__ __forceinline__ unsigned long long filt_mass(float v, float mx, float itau) {
    const float e = expf((v - mx) * itau);
    return e > 0.f ? __float2ull_rz(e * 4294967296.0f) : 0ull;
}

// Radix descent.  weight(i, v, key) is the weight of word i (0: not a candidate).  Returns the key b of the word at which
// the running weight, taken in key-descending order, first reaches `need` (weights of equal keys taken together); in
// *left the weight still needed among the words of key b, in *eq their total weight.  frac >= 0: need = max(1,
// ceil(frac * total weight)), fixed after the first digit (a total of 0 returns at once with *left = 0).  Otherwise
// need must lie in [1, total weight].
template <bool CACHED, typename W>
__device__ uint32_t filt_descend(const float* x, const float* row_s, int V, unsigned long long need, double frac,
                                 W weight, unsigned long long* hist, unsigned long long* sm_u,
                                 unsigned long long* left, unsigned long long* eq) {
    __shared__ uint32_t s_bin;
    __shared__ unsigned long long s_left, s_eq;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t prefix = 0;
#pragma unroll 1
    for (int pass = 0; pass < 3; ++pass) {
        const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
        const uint32_t hi_mask = pass == 0 ? 0u : (pass == 1 ? 0xffe00000u : 0xfffffc00u);
        const uint32_t dmask = pass == 2 ? 0x3ffu : 0x7ffu;
#pragma unroll
        for (int j = 0; j < kFiltBinsPerThread; ++j) hist[tid * kFiltBinsPerThread + j] = 0ull;
        __syncthreads();
        // (every thread has read the previous digit's result by now; the boundary bin is written after two barriers)
        if (tid == 0) { s_bin = 0; s_left = 1; s_eq = 0; }
#pragma unroll 1
        for (int i = tid; i < V; i += kRowThreads) {
            const float v = CACHED ? row_s[i] : x[i];
            const uint32_t key = filt_key(v);
            if ((key & hi_mask) != prefix) continue;
            const unsigned long long w = weight(i, v, key);
            if (w) atomicAdd(&hist[(key >> shift) & dmask], w);
        }
        __syncthreads();
        // thread t owns bins [8t, 8t + 8): the weight above its bins is a suffix sum over the threads after it
        unsigned long long own = 0;
#pragma unroll
        for (int j = 0; j < kFiltBinsPerThread; ++j) own += hist[tid * kFiltBinsPerThread + j];
        unsigned long long suf = own;   // inclusive suffix sum inside the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_down_sync(0xffffffffu, suf, o);
            if (lane + o < 32) suf += y;
        }
        if (lane == 0) sm_u[warp] = suf;
        __syncthreads();
        unsigned long long above = suf - own, total = 0;
        for (int w = 0; w < kRowThreads / 32; ++w) {
            total += sm_u[w];
            if (w > warp) above += sm_u[w];
        }
        if (pass == 0 && frac >= 0.0) {
            if (total == 0) {   // (uniform: every thread summed the same warp totals)
                *left = *eq = 0ull;
                return 0u;
            }
            const double c = ceil(frac * (double)total);
            need = c < 1.0 ? 1ull : (c >= (double)total ? total : (unsigned long long)c);
        }
        if (above < need && need <= above + own) {
#pragma unroll 1
            for (int j = kFiltBinsPerThread - 1; j >= 0; --j) {
                const unsigned long long hb = hist[tid * kFiltBinsPerThread + j];
                if (need <= above + hb) {
                    s_bin = tid * kFiltBinsPerThread + j;
                    s_left = need - above;
                    s_eq = hb;
                    break;
                }
                above += hb;
            }
        }
        __syncthreads();
        prefix |= s_bin << shift;
        need = s_left;
    }
    *left = need;
    *eq = s_eq;
    return prefix;
}

// Index of the c-th word (1 <= c, in index order) with key k that `cand` admits: a block prefix count over chunks of
// kRowThreads consecutive words, stopping at the chunk that holds it.
template <bool CACHED, typename C>
__device__ int filt_nth(const float* x, const float* row_s, int V, uint32_t k, unsigned long long c, C cand,
                        int* sm_cnt) {
    __shared__ int s_idx;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_idx = V - 1;
    unsigned long long base = 0;
#pragma unroll 1
    for (int i0 = 0; i0 < V; i0 += kRowThreads) {
        const int i = i0 + tid;
        const bool f = i < V && filt_key(CACHED ? row_s[i] : x[i]) == k && cand(i);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) sm_cnt[warp] = __popc(bal);
        __syncthreads();
        int off = 0, tot = 0;
        for (int w = 0; w < kRowThreads / 32; ++w) {
            if (w < warp) off += sm_cnt[w];
            tot += sm_cnt[w];
        }
        if (f && base + off + __popc(bal & ((1u << lane) - 1u)) + 1 == c) s_idx = i;
        base += tot;
        __syncthreads();
        if (base >= c) break;
    }
    return s_idx;
}

// Filtered sampling: one block per row.  Word i is kept when it is among the top_k words of the row (ties at the
// boundary to the lower index) and inside the shortest prefix of those, in rank order, whose softmax(logits /
// temperature) mass renormalised over them reaches top_p.  The draw is the Gumbel arg-max of the SMP instance over the
// kept words, so a word that the unfiltered draw of the same (seed, row, step) picks is picked here when it is kept;
// word_probs stay softmax(logits)[word] at temperature 1 over the whole row.
template <bool CACHED>
__global__ void __launch_bounds__(kRowThreads) rows_filter_kernel(const RowsParams p) {
    extern __shared__ __align__(16) float row_s[];
    __shared__ unsigned long long hist[kFiltBins];
    __shared__ unsigned long long sm_u[kRowThreads / 32];
    __shared__ ValIdx sm_vi[kRowThreads / 32];
    __shared__ float sm_f[kRowThreads / 32];
    __shared__ int sm_cnt[kRowThreads / 32];
    if (threadIdx.x == 0) tl_begin(p.tl);
    const int row = blockIdx.x;
    const float* x = p.logits + (size_t)row * p.V;
    const int V = p.V, n4 = V >> 2;
    const SampleParams* sp = p.sample;
    const float itau = sp->inv_tau;
    const int top_k = sp->top_k;
    const float top_p = sp->top_p;

    float mr = -INFINITY;
    if (CACHED) {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* d4 = reinterpret_cast<float4*>(row_s);
#pragma unroll 1
        for (int i4 = threadIdx.x; i4 < n4; i4 += kRowThreads) {
            const float4 v = x4[i4];
            d4[i4] = v;
            mr = fmaxf(fmaxf(mr, v.x), fmaxf(v.y, fmaxf(v.z, v.w)));
        }
    } else {
#pragma unroll 1
        for (int i = threadIdx.x; i < V; i += kRowThreads) mr = fmaxf(mr, x[i]);
    }
    const float m = block_best(ValIdx{mr, 0}, sm_vi).v;   // (its barriers also publish row_s)

    // top-k: kept when key > kk, or key == kk and i <= ki
    uint32_t kk = 0u;
    int ki = 0x7fffffff;
    if (top_k > 0 && top_k < V) {
        unsigned long long left, eq;
        kk = filt_descend<CACHED>(x, row_s, V, (unsigned long long)top_k, -1.0,
                                  [](int, float, uint32_t) { return 1ull; }, hist, sm_u, &left, &eq);
        if (left < eq) ki = filt_nth<CACHED>(x, row_s, V, kk, left, [](int) { return true; }, sm_cnt);
    }
    auto in_k = [&](int i, uint32_t key) { return key > kk || (key == kk && i <= ki); };

    // nucleus over the top-k words: kept when also key > pk, or key == pk and i <= pi
    uint32_t pk = 0u;
    int pi = 0x7fffffff;
    if (top_p < 1.0f) {
        const auto mass = [&](int i, float v, uint32_t key) { return in_k(i, key) ? filt_mass(v, m, itau) : 0ull; };
        unsigned long long left, eq;
        const uint32_t b = filt_descend<CACHED>(x, row_s, V, 0ull, (double)top_p, mass, hist, sm_u, &left, &eq);
        if (left > 0) {   // (a row whose words all weigh 0, e.g. all -inf, keeps the top-k words)
            pk = b;
            // words of equal key weigh the same: the first ceil(left / w) of them in index order are kept
            const unsigned long long w = filt_mass(filt_unkey(pk), m, itau);
            const unsigned long long c = w ? (left + w - 1) / w : 1ull;
            if (c * w < eq)
                pi = filt_nth<CACHED>(x, row_s, V, pk, c, [&](int i) { return in_k(i, pk); }, sm_cnt);
        }
    }

    const SampleKey sk = sample_key(sp->seed, row, p.step);
    ValIdx best = {-INFINITY, 0x7fffffff};
#pragma unroll 1
    for (int i = threadIdx.x; i < V; i += kRowThreads) {
        const float v = CACHED ? row_s[i] : x[i];
        const uint32_t key = filt_key(v);
        if (!in_k(i, key) || !(key > pk || (key == pk && i <= pi))) continue;
        const float g = fmaf(v, itau, sample_gumbel(sample_bits(sk, i)));
        if (better(g, i, best.v, best.i)) { best.v = g; best.i = i; }
    }
    best = block_best(best, sm_vi);
    if (threadIdx.x == 0) {
        if (p.tokens) p.tokens[(size_t)row * p.tokens_ld + p.step] = best.i;
        if (p.next_word) p.next_word[row] = best.i;
    }
    if (p.word_probs) {
        float s = 0.f;
#pragma unroll 1
        for (int i = threadIdx.x; i < V; i += kRowThreads) s += expf((CACHED ? row_s[i] : x[i]) - m);
        s = block_sum(s, sm_f);
        if (threadIdx.x == 0)   // (a row of NaN logits picks no word: probability 0, no read past the row)
            p.word_probs[(size_t)row * p.tokens_ld + p.step] = (best.i >= 0 && best.i < V) ? expf(x[best.i] - m) / s : 0.f;
    }
    if (threadIdx.x == 0) tl_end(p.tl);
}

cudaError_t rows_softmax_launch(const RowsParams& p, int rows, cudaStream_t st) {
    if (p.topk > kMaxTopK) return cudaErrorInvalidValue;
    const size_t bytes = (size_t)p.V * sizeof(float);
    const bool cached = (p.V % 4) == 0 && bytes <= 96 * 1024 && (reinterpret_cast<uintptr_t>(p.logits) % 16) == 0;
    if (p.sample && p.filter) {
        if (p.forced || p.topk || p.probs || p.argmax || p.V < 2) return cudaErrorInvalidValue;
        if (cached) {
            static bool filt_attr_set = false;
            if (!filt_attr_set) {
                cudaError_t e = cudaFuncSetAttribute(rows_filter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     96 * 1024);
                if (e != cudaSuccess) return e;
                filt_attr_set = true;
            }
            rows_filter_kernel<true><<<rows, kRowThreads, bytes, st>>>(p);
        } else {
            rows_filter_kernel<false><<<rows, kRowThreads, 0, st>>>(p);
        }
        return cudaGetLastError();
    }
    if (p.sample) {
        if (p.forced || p.topk || p.probs || p.argmax) return cudaErrorInvalidValue;
        if (cached) {
            static bool smp_attr_set = false;
            if (!smp_attr_set) {
                cudaError_t e = cudaFuncSetAttribute(rows_softmax_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     96 * 1024);
                if (e != cudaSuccess) return e;
                smp_attr_set = true;
            }
            rows_softmax_kernel<true, true><<<rows, kRowThreads, bytes, st>>>(p);
        } else {
            rows_softmax_kernel<false, true><<<rows, kRowThreads, 0, st>>>(p);
        }
        return cudaGetLastError();
    }
    if (cached) {
        static bool attr_set = false;
        if (!attr_set) {
            cudaError_t e = cudaFuncSetAttribute(rows_softmax_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
            if (e != cudaSuccess) return e;
            attr_set = true;
        }
        rows_softmax_kernel<true><<<rows, kRowThreads, bytes, st>>>(p);
    } else {
        rows_softmax_kernel<false><<<rows, kRowThreads, 0, st>>>(p);
    }
    return cudaGetLastError();
}

// ------------------------------------------------------------------ beam search
// Python heapq semantics (CPython Lib/heapq.py) on tiny arrays, so that ties are
// broken exactly as utils/misc.py:62-87 (TopN) does.
struct PItem { double score; int parent; int word; float p; };
struct CItem { double score; int slot; int len; };

template <typename T>
__device__ void heap_siftdown(T* h, int startpos, int pos) {
    T item = h[pos];
    while (pos > startpos) {
        const int parent = (pos - 1) >> 1;
        if (item.score < h[parent].score) { h[pos] = h[parent]; pos = parent; continue; }
        break;
    }
    h[pos] = item;
}
template <typename T>
__device__ void heap_siftup(T* h, int n, int pos) {
    const int startpos = pos;
    T item = h[pos];
    int child = 2 * pos + 1;
    while (child < n) {
        const int right = child + 1;
        if (right < n && !(h[child].score < h[right].score)) child = right;
        h[pos] = h[child];
        pos = child;
        child = 2 * pos + 1;
    }
    h[pos] = item;
    heap_siftdown(h, startpos, pos);
}

__global__ void __launch_bounds__(256) beam_update_kernel(const BeamParams p) {
    __shared__ PItem newp[kMaxBeam];
    __shared__ int newn;
    __shared__ int s_idx[kMaxBeam * (kMaxBeam + 1)];
    __shared__ float s_p[kMaxBeam * (kMaxBeam + 1)];
    __shared__ double s_ps[kMaxBeam];
    const int img = blockIdx.x;
    const int beam = p.beam, K = p.beam + 1, G = p.nlive, T = p.T, idx = p.step;
    const int* sent_cur = p.sent[idx & 1] + (size_t)img * beam * T;
    int* sent_next = p.sent[(idx + 1) & 1] + (size_t)img * beam * T;

    // the candidates of this image (G live beams x K words) and the beams' scores: one parallel round trip
    if ((int)threadIdx.x < G * K) {
        s_idx[threadIdx.x] = p.topk_idx[(size_t)img * G * K + threadIdx.x];
        s_p[threadIdx.x] = p.topk_p[(size_t)img * G * K + threadIdx.x];
    }
    if ((int)threadIdx.x < G) s_ps[threadIdx.x] = idx == 0 ? 1.0 : p.part_score[(size_t)img * beam + threadIdx.x];   // base_model.py:178
    __syncthreads();

    if (threadIdx.x == 0) {
        int np = 0;
        CItem* ch = p.comp_heap + (size_t)img * beam;
        int cn = p.comp_n[img];
        for (int b = 0; b < G; ++b) {
            const double ps = s_ps[b];
            for (int j = 0; j < K; ++j) {
                const int w = s_idx[b * K + j];
                const double sc = ps * (double)s_p[b * K + j];                           // base_model.py:224
                if (w == p.eos_id) {                                                   // base_model.py:229-230
                    int slot = -1;
                    if (cn < beam) {
                        slot = cn;
                        ch[cn].score = sc; ch[cn].slot = slot; ch[cn].len = idx + 1;
                        ++cn;
                        heap_siftdown(ch, 0, cn - 1);
                    } else if (ch[0].score < sc) {
                        slot = ch[0].slot;
                        ch[0].score = sc; ch[0].len = idx + 1;
                        heap_siftup(ch, cn, 0);
                    }
                    if (slot >= 0) {
                        int* dst = p.comp_sent + ((size_t)img * beam + slot) * T;
                        for (int t = 0; t < idx; ++t) dst[t] = sent_cur[(size_t)b * T + t];
                        dst[idx] = w;
                        if (p.comp_prov) {   // (the step is len - 1 of the slot's CItem)
                            p.comp_prov[(size_t)img * beam + slot] = b;
                            p.comp_p[(size_t)img * beam + slot] = s_p[b * K + j];
                        }
                    }
                } else {                                                               // base_model.py:231-232
                    if (np < beam) {
                        newp[np].score = sc; newp[np].parent = b; newp[np].word = w; newp[np].p = s_p[b * K + j];
                        ++np;
                        heap_siftdown(newp, 0, np - 1);
                    } else if (newp[0].score < sc) {
                        newp[0].score = sc; newp[0].parent = b; newp[0].word = w; newp[0].p = s_p[b * K + j];
                        heap_siftup(newp, np, 0);
                    }
                }
            }
        }
        p.comp_n[img] = cn;
        newn = np;
        p.part_n[img] = np;
        for (int j = 0; j < np; ++j) p.part_score[(size_t)img * beam + j] = newp[j].score;
    }
    __syncthreads();
    // materialise the surviving beams: sentences, last word, LSTM state rows (float4 rows, all beams in one sweep)
    const int np = newn;
    for (int u = threadIdx.x; u < np * idx; u += blockDim.x) {
        const int j = u / idx, t = u - j * idx;
        sent_next[(size_t)j * T + t] = sent_cur[(size_t)newp[j].parent * T + t];
    }
    if ((int)threadIdx.x < np) {
        sent_next[(size_t)threadIdx.x * T + idx] = newp[threadIdx.x].word;
        p.next_word[(size_t)img * beam + threadIdx.x] = newp[threadIdx.x].word;
        if (p.hist_parent) {
            const size_t hi = (size_t)idx * p.NI * beam + (size_t)img * beam + threadIdx.x;
            p.hist_parent[hi] = newp[threadIdx.x].parent;
            p.hist_p[hi] = newp[threadIdx.x].p;
        }
    }
    const int H4 = p.H >> 2;   // H % 32 == 0 (sat_create)
    for (int u = threadIdx.x; u < np * H4; u += blockDim.x) {
        const int j = u / H4, q = u - j * H4;
        const int b = newp[j].parent;
        reinterpret_cast<float4*>(p.c_next + ((size_t)img * beam + j) * p.H)[q] =
            reinterpret_cast<const float4*>(p.c_out + ((size_t)img * G + b) * p.H)[q];
        reinterpret_cast<float4*>(p.h_next + ((size_t)img * beam + j) * p.H)[q] =
            reinterpret_cast<const float4*>(p.h_out + ((size_t)img * G + b) * p.H)[q];
    }
}

// base_model.py:234-238: complete captions if any, else the partial ones, sorted by
// descending score (list.sort(reverse=True) is stable: equal scores keep heap order).
__global__ void beam_finalize_kernel(const BeamParams p) {
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= p.NI) return;
    const int beam = p.beam, T = p.T;
    const int cn = p.comp_n[img];
    const bool use_comp = cn > 0;
    const int n = use_comp ? cn : p.part_n[img];
    int order[kMaxBeam];
    double sc[kMaxBeam];
    for (int j = 0; j < n; ++j) {
        order[j] = j;
        sc[j] = use_comp ? p.comp_heap[(size_t)img * beam + j].score : p.part_score[(size_t)img * beam + j];
    }
    for (int a = 1; a < n; ++a) {  // stable insertion sort, descending
        const int o = order[a];
        const double s = sc[a];
        int k = a;
        while (k > 0 && sc[k - 1] < s) { sc[k] = sc[k - 1]; order[k] = order[k - 1]; --k; }
        sc[k] = s; order[k] = o;
    }
    const int* part_sent = p.sent[p.step & 1] + (size_t)img * beam * T;   // p.step = number of steps taken
    for (int j = 0; j < beam; ++j) {
        int* dst = p.res_sent + ((size_t)img * beam + j) * T;
        if (j < n) {
            const int o = order[j];
            int len;
            const int* src;
            if (use_comp) {
                const CItem& it = p.comp_heap[(size_t)img * beam + o];
                len = it.len;
                src = p.comp_sent + ((size_t)img * beam + it.slot) * T;
            } else {
                len = p.step;
                src = part_sent + (size_t)o * T;
            }
            for (int t = 0; t < T; ++t) dst[t] = t < len ? src[t] : -1;
            p.res_len[(size_t)img * beam + j] = len;
            p.res_score[(size_t)img * beam + j] = sc[j];
            if (p.res_src) p.res_src[(size_t)img * beam + j] = use_comp ? p.comp_heap[(size_t)img * beam + o].slot : o;
        } else {
            for (int t = 0; t < T; ++t) dst[t] = -1;
            p.res_len[(size_t)img * beam + j] = 0;
            p.res_score[(size_t)img * beam + j] = 0.0;
            if (p.res_src) p.res_src[(size_t)img * beam + j] = -1;
        }
    }
    p.res_n[img] = n;
    p.res_complete[img] = use_comp ? 1 : 0;
}

// Per-word maps of result (img, j): walk the caption back from its last word through the back-pointers
//   word t of survivor j of step t came from live row r_t = hist_parent[t][j]; the survivor of step t-1 is j = r_t
// and gather alpha rows and probabilities, zero past the caption's length.  One block per result.
__global__ void __launch_bounds__(256) beam_maps_kernel(const BeamParams p) {
    extern __shared__ int rows_s[];   // [T] live row of step t (row index inside the image's group)
    __shared__ float p_s[1024];
    const int res = blockIdx.x, img = res / p.beam;
    const int beam = p.beam, T = p.T, L = p.L, NB = p.NI * beam;
    const int src = p.res_src[res];
    const int len = src < 0 ? 0 : p.res_len[res];
    if (threadIdx.x == 0 && len > 0) {
        int t = len - 1, j;
        if (p.res_complete[img]) {   // completed at step len - 1 from live row comp_prov
            const int b = p.comp_prov[(size_t)img * beam + src];
            rows_s[t] = b;
            p_s[t] = p.comp_p[(size_t)img * beam + src];
            j = b;
            --t;
        } else {
            j = src;                 // partial beam src after the last step
        }
        for (; t >= 0; --t) {
            const size_t hi = (size_t)t * NB + (size_t)img * beam + j;
            const int r = p.hist_parent[hi];
            rows_s[t] = r;
            p_s[t] = p.hist_p[hi];
            j = r;
        }
    }
    __syncthreads();
    if (p.res_probs)
        for (int t = threadIdx.x; t < T; t += blockDim.x) p.res_probs[(size_t)res * T + t] = t < len ? p_s[t] : 0.f;
    if (p.res_alpha) {
        float* dst = p.res_alpha + (size_t)res * T * L;
        for (int u = threadIdx.x; u < T * L; u += blockDim.x) {
            const int t = u / L, l = u - t * L;
            float v = 0.f;
            if (t < len) {
                const int G = t == 0 ? 1 : beam;
                v = p.hist_alpha[((size_t)t * NB + (size_t)img * G + rows_s[t]) * L + l];
            }
            dst[u] = v;
        }
    }
}

cudaError_t beam_update_launch(const BeamParams& p, cudaStream_t st) {
    if (p.beam > kMaxBeam) return cudaErrorInvalidValue;
    beam_update_kernel<<<p.NI, 256, 0, st>>>(p);
    return cudaGetLastError();
}
cudaError_t beam_finalize_launch(const BeamParams& p, cudaStream_t st) {
    beam_finalize_kernel<<<(p.NI + 63) / 64, 64, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t beam_maps_launch(const BeamParams& p, cudaStream_t st) {
    if (!p.res_src || p.T > 1024) return cudaErrorInvalidValue;
    beam_maps_kernel<<<p.NI * p.beam, 256, (size_t)p.T * sizeof(int), st>>>(p);
    return cudaGetLastError();
}

size_t beam_citem_bytes() { return sizeof(CItem); }

// ---------------------------------------------------------------- sampling loop
__global__ void sample_params_kernel(SampleParams* dst, unsigned long long seed, float inv_tau, int top_k, float top_p) {
    dst->seed = seed;
    dst->inv_tau = inv_tau;
    dst->pad = 0.f;
    dst->top_k = top_k;
    dst->top_p = top_p;
}

cudaError_t sample_params_launch(SampleParams* dst, unsigned long long seed, float inv_tau, cudaStream_t st, int top_k,
                                 float top_p) {
    sample_params_kernel<<<1, 1, 0, st>>>(dst, seed, inv_tau, top_k, top_p);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) bcast_state_kernel(const float4* c_src, const float4* h_src, float4* c_dst,
                                                          float4* h_dst, int rows, int G, int H4) {
    const long long n = (long long)rows * H4;
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const long long r = i / H4, q = i - r * H4;
        const long long s = (r / G) * H4 + q;
        c_dst[i] = c_src[s];
        h_dst[i] = h_src[s];
    }
}

cudaError_t bcast_state_launch(const float* c_src, const float* h_src, float* c_dst, float* h_dst, int rows, int G, int H,
                               cudaStream_t st) {
    if (G < 1 || H % 4) return cudaErrorInvalidValue;
    const long long n = (long long)rows * (H / 4);
    int grid = (int)((n + 255) / 256);
    if (grid > 1024) grid = 1024;
    bcast_state_kernel<<<grid < 1 ? 1 : grid, 256, 0, st>>>(reinterpret_cast<const float4*>(c_src), reinterpret_cast<const float4*>(h_src),
                                                       reinterpret_cast<float4*>(c_dst), reinterpret_cast<float4*>(h_dst), rows, G, H / 4);
    return cudaGetLastError();
}

}  // namespace sat
