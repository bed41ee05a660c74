// sat_cider.cu — CIDEr-D of word-id captions against their references (the reward of self-critical training and a
// validation metric), with the semantics of coco-caption's cider_scorer.py / the CiderD scorer of SCST codebases.
//
// A caption row ends after its first eos_id, or before its first id < 0 or >= vocabulary_size.  Its n-grams (n = 1..4)
// are packed into 64-bit keys: four 16-bit fields of (word + 1), the first word in the top field, unused fields 0 (so
// the number of non-zero fields is n and no key is 0).  Document frequencies live in an open-addressing hash table
// (linear probing, key 0 = empty slot, load factor <= 1/2) built once on the host from a reference corpus.
//
// sat_cider_d runs one CTA per image.  Phase 1: warp r extracts the n-grams of reference r into a scratch array, sorts
// them (bitonic, within the warp), run-length counts them into the distinct keys with their tf-idf weights, and takes
// the per-n norms.  Phase 2: one warp per candidate does the same for the candidate, then intersects its distinct
// n-grams with each reference's sorted list (binary search).  All arithmetic is fp64 and every sum runs in a fixed
// order (lane-strided partial sums, then a fixed butterfly), so scores are bit-reproducible.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <new>
#include <vector>

#include "../../include/sat_b200.h"
#include "sat_internal.h"

namespace {

#define CCK(x)                                                                                          \
    do {                                                                                                \
        cudaError_t e_ = (x);                                                                           \
        if (e_ != cudaSuccess) return sat_fail(SAT_ERR_CUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
    } while (0)

constexpr int kMaxRefs = 8;    // references per image (COCO has 5-7)
constexpr int kMaxLen = 64;    // words per candidate / reference row
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr double kSigma = 6.0;

__host__ __device__ inline uint64_t mix64(uint64_t x) {   // splitmix64 finaliser: the table's hash
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}

// n-grams of a row of `len` words
__host__ __device__ inline int gram_count(int len) {
    int g = 0;
    for (int n = 1; n <= 4; ++n) g += len - n + 1 > 0 ? len - n + 1 : 0;
    return g;
}

inline int pow2_at_least(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

__device__ inline int gram_n(uint64_t key) { return 4 - (__ffsll((long long)key) - 1) / 16; }

struct Table {
    const uint64_t* keys;
    const uint32_t* df;
    uint64_t mask;
    double log_n;
};

__device__ inline uint32_t df_lookup(const Table& t, uint64_t key) {
    uint64_t i = mix64(key) & t.mask;
    for (;;) {
        const uint64_t k = __ldg(t.keys + i);
        if (k == key) return __ldg(t.df + i);
        if (k == 0) return 0;
        i = (i + 1) & t.mask;
    }
}

__device__ inline double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One warp: the distinct n-grams of a caption row, sorted by key, with their tf-idf weights.
// scratch: pow2_at_least(gram_count(T)) keys; dk / w: room for as many distinct n-grams.
// Returns the number of distinct n-grams; *len = words kept; norm[n-1] = ||v_n||.
__device__ int warp_ngrams(const int32_t* __restrict__ row, int T, int eos, int V, const Table& tab,
                           uint64_t* scratch, uint64_t* dk, double* w, int* len_out, double norm[4]) {
    const int lane = threadIdx.x & 31;
    int len = T;
    for (int base = 0; base < T; base += 32) {
        const int t = base + lane;
        const int x = t < T ? row[t] : 0;
        const bool before = t < T && (x < 0 || x >= V);
        const bool after = t < T && !before && x == eos;
        const unsigned b = __ballot_sync(0xffffffffu, before || after);
        const unsigned a = __ballot_sync(0xffffffffu, after);
        if (b) {
            const int p = __ffs(b) - 1;
            len = base + p + ((a >> p) & 1);
            break;
        }
    }
    const int G = gram_count(len);
    int P = 1;
    while (P < G) P <<= 1;
    int off = 0;
    for (int n = 1; n <= 4; ++n) {
        const int cnt = len - n + 1;
        for (int i = lane; i < cnt; i += 32) {
            uint64_t key = 0;
            for (int m = 0; m < n; ++m) key |= (uint64_t)(uint32_t)(row[i + m] + 1) << (48 - 16 * m);
            scratch[off + i] = key;
        }
        off += cnt > 0 ? cnt : 0;
    }
    for (int i = G + lane; i < P; i += 32) scratch[i] = ~0ull;   // sorts last: the first G sorted keys are the row's
    __syncwarp();
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < P; i += 32) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const uint64_t a = scratch[i], b = scratch[ixj];
                    if ((a > b) == ((i & k) == 0)) {
                        scratch[i] = b;
                        scratch[ixj] = a;
                    }
                }
            }
            __syncwarp();
        }
    }
    // run-length count: lane l owns the sorted positions [lo, hi); heads (first of a run) are numbered in order
    const int chunk = (G + 31) / 32;
    const int lo = min(lane * chunk, G), hi = min(lo + chunk, G);
    int heads = 0;
    for (int i = lo; i < hi; ++i) heads += i == 0 || scratch[i] != scratch[i - 1];
    int pos = heads;
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, pos, o);
        if (lane >= o) pos += v;
    }
    const int nd = __shfl_sync(0xffffffffu, pos, 31);
    pos -= heads;
    for (int i = lo; i < hi; ++i) {
        if (i == 0 || scratch[i] != scratch[i - 1]) {
            int e = i + 1;
            while (e < G && scratch[e] == scratch[i]) ++e;
            dk[pos] = scratch[i];
            w[pos] = (double)(e - i);
            ++pos;
        }
    }
    __syncwarp();
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int j = lane; j < nd; j += 32) {
        const uint64_t key = dk[j];
        const uint32_t df = df_lookup(tab, key);
        const double v = w[j] * (tab.log_n - log(df > 1u ? (double)df : 1.0));
        w[j] = v;
        const int n = gram_n(key);
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[q] += q == n - 1 ? v * v : 0.0;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) norm[q] = sqrt(warp_sum(acc[q]));
    __syncwarp();
    *len_out = len;
    return nd;
}

__global__ void __launch_bounds__(kThreads) cider_d_kernel(Table tab, const int32_t* __restrict__ cand, int C, int T,
                                                          const int32_t* __restrict__ refs, int R, int T_ref, int eos,
                                                          int V, int PR, int PC, float* __restrict__ scores) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int ref_nd[kMaxRefs], ref_len[kMaxRefs];
    __shared__ double ref_norm[kMaxRefs][4];
    const int img = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int PS = PR > PC ? PR : PC;
    uint64_t* ref_dk = (uint64_t*)smem;                        // [R][PR]
    double* ref_w = (double*)(ref_dk + (size_t)R * PR);        // [R][PR]
    uint64_t* cand_dk = (uint64_t*)(ref_w + (size_t)R * PR);   // [kWarps][PC]
    double* cand_w = (double*)(cand_dk + kWarps * PC);         // [kWarps][PC]
    uint64_t* scratch = (uint64_t*)(cand_w + kWarps * PC) + (size_t)warp * PS;

    // phase 1: the references of this image, one warp each
    if (warp < R) {
        double nr[4];
        int len;
        const int nd = warp_ngrams(refs + ((size_t)img * R + warp) * T_ref, T_ref, eos, V, tab, scratch,
                                   ref_dk + (size_t)warp * PR, ref_w + (size_t)warp * PR, &len, nr);
        if (lane == 0) {
            ref_nd[warp] = nd;
            ref_len[warp] = len;
            for (int q = 0; q < 4; ++q) ref_norm[warp][q] = nr[q];
        }
    }
    __syncthreads();
    int n_refs = 0;
    for (int r = 0; r < R; ++r) n_refs += ref_len[r] > 0;

    // phase 2: one warp per candidate
    uint64_t* dk = cand_dk + (size_t)warp * PC;
    double* w = cand_w + (size_t)warp * PC;
    for (int c = warp; c < C; c += kWarps) {
        double nh[4];
        int len;
        const int nd = warp_ngrams(cand + ((size_t)img * C + c) * T, T, eos, V, tab, scratch, dk, w, &len, nh);
        double score[4] = {0.0, 0.0, 0.0, 0.0};
        const int lh = len > 1 ? len - 1 : 0;   // "length" = number of bigrams, as both reference scorers compute it
        for (int r = 0; r < R; ++r) {
            if (ref_len[r] == 0) continue;
            const uint64_t* rk = ref_dk + (size_t)r * PR;
            const double* rw = ref_w + (size_t)r * PR;
            const int rn = ref_nd[r];
            double acc[4] = {0.0, 0.0, 0.0, 0.0};
            for (int j = lane; j < nd; j += 32) {
                const uint64_t key = dk[j];
                int a = 0, b = rn;   // lower bound of key in rk[0, rn)
                while (a < b) {
                    const int m = (a + b) >> 1;
                    if (rk[m] < key) a = m + 1;
                    else b = m;
                }
                if (a < rn && rk[a] == key) {
                    const double vh = w[j], vr = rw[a];
                    const double s = fmin(vh, vr) * vr;
                    const int n = gram_n(key);
#pragma unroll
                    for (int q = 0; q < 4; ++q) acc[q] += q == n - 1 ? s : 0.0;
                }
            }
            const int lr = ref_len[r] > 1 ? ref_len[r] - 1 : 0;
            const double delta = (double)(lh - lr);
            const double pen = exp(-(delta * delta) / (2.0 * kSigma * kSigma));
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                double val = warp_sum(acc[q]);
                if (nh[q] != 0.0 && ref_norm[r][q] != 0.0) val /= nh[q] * ref_norm[r][q];
                score[q] += val * pen;
            }
        }
        if (lane == 0) {
            const double tot = ((score[0] + score[1]) + score[2]) + score[3];
            scores[(size_t)img * C + c] = n_refs ? (float)(tot / n_refs / 4.0 * 10.0) : 0.f;
        }
        __syncwarp();
    }
}

// restores the caller's current device on scope exit
struct DeviceScope {
    int prev = -1;
    ~DeviceScope() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

}  // namespace

struct sat_cider {
    int dev;
    int eos_id, vocabulary_size;
    Table tab;
    uint64_t* keys;
    uint32_t* df;
};

extern "C" void sat_cider_destroy(sat_cider* c) {
    if (!c) return;
    DeviceScope ds;
    if (cudaGetDevice(&ds.prev) == cudaSuccess) cudaSetDevice(c->dev);
    cudaFree(c->keys);
    cudaFree(c->df);
    delete c;
}

static int cider_create(const int32_t* refs_host, int64_t n_img, int32_t R, int32_t T_ref, int32_t eos_id, int32_t V,
                        sat_cider** out) {
    // every image's distinct n-grams (a set per image: df counts images, not occurrences)
    std::vector<uint64_t> all, img;
    for (int64_t i = 0; i < n_img; ++i) {
        img.clear();
        for (int r = 0; r < R; ++r) {
            const int32_t* row = refs_host + (i * R + r) * (int64_t)T_ref;
            int len = 0;
            while (len < T_ref && row[len] >= 0 && row[len] < V) {
                if (row[len++] == eos_id) break;
            }
            for (int n = 1; n <= 4; ++n)
                for (int s = 0; s + n <= len; ++s) {
                    uint64_t key = 0;
                    for (int m = 0; m < n; ++m) key |= (uint64_t)(uint32_t)(row[s + m] + 1) << (48 - 16 * m);
                    img.push_back(key);
                }
        }
        std::sort(img.begin(), img.end());
        img.erase(std::unique(img.begin(), img.end()), img.end());
        all.insert(all.end(), img.begin(), img.end());
    }
    std::sort(all.begin(), all.end());
    size_t distinct = 0;
    for (size_t i = 0; i < all.size(); ++i) distinct += i == 0 || all[i] != all[i - 1];
    size_t cap = 1024;
    while (cap < 2 * distinct) cap <<= 1;
    std::vector<uint64_t> keys(cap, 0);
    std::vector<uint32_t> df(cap, 0);
    for (size_t i = 0; i < all.size();) {
        size_t e = i + 1;
        while (e < all.size() && all[e] == all[i]) ++e;
        uint64_t s = mix64(all[i]) & (cap - 1);
        while (keys[s] != 0) s = (s + 1) & (cap - 1);
        keys[s] = all[i];
        df[s] = (uint32_t)(e - i);
        i = e;
    }
    std::vector<uint64_t>().swap(all);
    int dev = 0;
    CCK(cudaGetDevice(&dev));
    sat_cider* c = new sat_cider();
    c->dev = dev;
    c->eos_id = eos_id;
    c->vocabulary_size = V;
    c->keys = nullptr;
    c->df = nullptr;
    cudaError_t e = cudaMalloc(&c->keys, cap * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(&c->df, cap * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMemcpy(c->keys, keys.data(), cap * sizeof(uint64_t), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(c->df, df.data(), cap * sizeof(uint32_t), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        sat_cider_destroy(c);
        return sat_fail(e == cudaErrorMemoryAllocation ? SAT_ERR_NOMEM : SAT_ERR_CUDA, "sat_cider_create: %s",
                        cudaGetErrorString(e));
    }
    c->tab = Table{c->keys, c->df, (uint64_t)(cap - 1), log((double)n_img)};
    *out = c;
    return SAT_OK;
}

extern "C" int sat_cider_create(const int32_t* refs_host, int64_t n_img, int32_t R, int32_t T_ref, int32_t eos_id,
                                int32_t vocabulary_size, sat_cider** out) {
    if (!out) return sat_fail(SAT_ERR_INVALID, "sat_cider_create: null out");
    *out = nullptr;
    if (!refs_host || n_img < 1 || n_img > (int64_t)UINT32_MAX || R < 1 || T_ref < 1)
        return sat_fail(SAT_ERR_INVALID, "sat_cider_create: bad corpus (n_img=%lld, R=%d, T_ref=%d)", (long long)n_img,
                        R, T_ref);
    if (vocabulary_size < 2 || vocabulary_size > 65535)
        return sat_fail(SAT_ERR_INVALID, "sat_cider_create: vocabulary_size %d outside [2, 65535]", vocabulary_size);
    try {
        return cider_create(refs_host, n_img, R, T_ref, eos_id, vocabulary_size, out);
    } catch (const std::bad_alloc&) {
        return sat_fail(SAT_ERR_NOMEM, "sat_cider_create: out of host memory");
    }
}

extern "C" int sat_cider_d(const sat_cider* c, const int32_t* candidates, int32_t n_img, int32_t C, int32_t T,
                           const int32_t* refs, int32_t R, int32_t T_ref, float* scores, void* stream) {
    if (!c || !candidates || !refs || !scores || n_img < 0 || C < 1 || T < 1 || R < 1 || T_ref < 1)
        return sat_fail(SAT_ERR_INVALID, "sat_cider_d: bad argument (n_img=%d, C=%d, T=%d, R=%d, T_ref=%d)", n_img, C,
                        T, R, T_ref);
    if (R > kMaxRefs || T > kMaxLen || T_ref > kMaxLen)
        return sat_fail(SAT_ERR_UNSUPPORTED, "sat_cider_d: R=%d, T=%d, T_ref=%d (limits: R <= %d, T and T_ref <= %d)",
                        R, T, T_ref, kMaxRefs, kMaxLen);
    if (n_img == 0) return SAT_OK;
    DeviceScope ds;
    CCK(cudaGetDevice(&ds.prev));
    CCK(cudaSetDevice(c->dev));
    const int PR = pow2_at_least(gram_count(T_ref)), PC = pow2_at_least(gram_count(T));
    const size_t smem = (size_t)R * PR * 16 + (size_t)kWarps * PC * 16 + (size_t)kWarps * std::max(PR, PC) * 8;
    if (smem > 48 * 1024) CCK(cudaFuncSetAttribute(cider_d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cider_d_kernel<<<n_img, kThreads, smem, (cudaStream_t)stream>>>(c->tab, candidates, C, T, refs, R, T_ref, c->eos_id,
                                                                  c->vocabulary_size, PR, PC, scores);
    CCK(cudaGetLastError());
    return SAT_OK;
}
