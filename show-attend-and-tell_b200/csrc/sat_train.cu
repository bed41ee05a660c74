// sat_train.cu — the training step of the unrolled decoder (model.py:250-334 losses, :461-511 optimizer):
// forward with dropout and teacher forcing, backward through time, global-norm clip and Adam.
//
// First complete version: every op is a plain fp32 CUDA-core kernel (tiled SGEMM + element-wise kernels)
// working on explicit, stashed intermediates, written to mirror the reference graph node by node so that
// losses and every gradient can be checked against the autograd oracle (oracle/train_ref.py).  The
// tensor-core versions of the large GEMMs (attend/fc_1a forward and weight gradient: ~70 % of the FLOPs)
// are the next step; correctness comes first.
//
// Dropout masks come from a counter-based generator (splitmix64 of seed/stream/index, see
// oracle/train_ref.py) — the reference's TF ops are unseeded, so injected masks are the only way to
// compare a training step (SURVEY.md N4).
//
// Data parallelism: gradients are written into ONE flat fp32 buffer laid out like the parameters; the host
// all-reduces it (NCCL) between sat_train_forward_backward and sat_train_apply.  Losses use the global
// normalisers passed in (sum of masks, global batch), so the summed shard gradients equal the
// single-process gradient; the L2-regulariser gradient is added once, in sat_train_apply.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/sat_b200.h"
#include "sat_internal.h"
#include "sat_linear.cuh"

namespace {

#define TCK(x)                                                                                          \
    do {                                                                                                \
        cudaError_t e_ = (x);                                                                           \
        if (e_ != cudaSuccess) return sat_fail(SAT_ERR_CUDA, "%s failed: %s", #x, cudaGetErrorString(e_)); \
    } while (0)
#define TRET(x)                      \
    do {                             \
        int r_ = (x);                \
        if (r_ != SAT_OK) return r_; \
    } while (0)

// ------------------------------------------------------------------------------------------ RNG
// counter-based dropout masks: sat::rng_u24 / sat::drop_scale of sat_linear.cuh (shared with the packing kernels)
using sat::drop_gen;
using sat::drop_scale;
using sat::DropGen;
using sat::rng_u24;

// ------------------------------------------------------------------------------------------ launches
// Every kernel of this file starts with "wait for the predecessor grid, then let the successor launch"
// (griddepcontrol.wait ; griddepcontrol.launch_dependents) and is launched with the programmatic-serialization
// attribute: the next kernel's launch latency (a few microseconds, comparable to the run time of the many small
// element-wise kernels of a time step) overlaps this kernel's execution, while the data dependency stays a full
// one — nothing is read or written before the wait returns, and because the trigger comes after the kernel's own
// wait, a kernel never starts before the predecessor of its predecessor has completed (the convention of
// sat_common.cuh, which the dense kernel's early weight prefetch relies on).  SAT_TRAIN_PDL=0 turns the attribute off.
__device__ __forceinline__ void pdl_enter() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
static int train_pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("SAT_TRAIN_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v;
}
#define PDLK train_pdl_enabled()
template <typename... KA, typename... A>
static cudaError_t launch_k(void (*kernel)(KA...), dim3 grid, dim3 block, cudaStream_t st, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = train_pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KA>(args)...);
}

// ------------------------------------------------------------------------------------------ SGEMM
// C[M,N] = op(A)[M,K] * op(B)[K,N] (+ C if accumulate).  Row-major.  TA: A is stored [K,M]; TB: B is stored [N,K].
// 128x128x8 tiles, 256 threads x (8x8) outputs, double-buffered shared memory, float4 global loads where the
// operand is aligned.  gridDim.z > 1 splits K and accumulates with atomics (accumulate semantics on a pre-set C).
constexpr int GM = 128, GN = 128, GK = 8;

template <bool TRANS>   // TRANS: the tile's fast axis in memory is the M/N axis (A stored [K,M] / B stored [K,N])
__device__ __forceinline__ void gemm_load_tile(float (&reg)[4], const float* __restrict__ P, int ld, int mn0, int k0, int MN,
                                               int k_end, int tid) {
    // tile = 128 (mn) x 8 (k) = 256 float4; thread `tid` owns one float4
    if (TRANS) {
        const int k = tid >> 5, mn = (tid & 31) * 4;           // float4 along mn
        const int gk = k0 + k, gmn = mn0 + mn;
        const float* p = P + (size_t)gk * ld + gmn;
        if (gk < k_end && gmn + 3 < MN && ((((size_t)p) & 15) == 0)) {
            const float4 v = *reinterpret_cast<const float4*>(p);
            reg[0] = v.x; reg[1] = v.y; reg[2] = v.z; reg[3] = v.w;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) reg[i] = (gk < k_end && gmn + i < MN) ? p[i] : 0.f;
        }
    } else {
        const int mn = tid >> 1, k = (tid & 1) * 4;            // float4 along k
        const int gmn = mn0 + mn, gk = k0 + k;
        const float* p = P + (size_t)gmn * ld + gk;
        if (gmn < MN && gk + 3 < k_end && ((((size_t)p) & 15) == 0)) {
            const float4 v = *reinterpret_cast<const float4*>(p);
            reg[0] = v.x; reg[1] = v.y; reg[2] = v.z; reg[3] = v.w;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) reg[i] = (gmn < MN && gk + i < k_end) ? p[i] : 0.f;
        }
    }
}
template <bool TRANS>
__device__ __forceinline__ void gemm_store_tile(float (*sm)[GM + 4], const float (&reg)[4], int tid) {
    if (TRANS) {
        const int k = tid >> 5, mn = (tid & 31) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) sm[k][mn + i] = reg[i];
    } else {
        const int mn = tid >> 1, k = (tid & 1) * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) sm[k + i][mn] = reg[i];
    }
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(256) sgemm_kernel(int M, int N, int K, const float* __restrict__ A, int lda,
                                                    const float* __restrict__ B, int ldb, float* __restrict__ C, int ldc,
                                                    int accumulate, int kchunk) {
    pdl_enter();
    __shared__ float As[2][GK][GM + 4];
    __shared__ float Bs[2][GK][GN + 4];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;   // 16 x 16 threads; thread owns rows ty*4+{0..3}, 64+ty*4+{0..3}; cols likewise
    const int m0 = blockIdx.y * GM, n0 = blockIdx.x * GN;
    const int k_begin = blockIdx.z * kchunk, k_end = min(K, k_begin + kchunk);
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float ra[4], rb[4];
    // A tile: TA means memory is [K, M] (fast axis m) -> TRANS = TA.  B tile: memory [K, N] (fast axis n) unless TB.
    gemm_load_tile<TA>(ra, A, lda, m0, k_begin, M, k_end, tid);
    gemm_load_tile<!TB>(rb, B, ldb, n0, k_begin, N, k_end, tid);
    gemm_store_tile<TA>(As[0], ra, tid);
    gemm_store_tile<!TB>(Bs[0], rb, tid);
    __syncthreads();
    int buf = 0;
    for (int k0 = k_begin; k0 < k_end; k0 += GK) {
        const bool more = k0 + GK < k_end;
        if (more) {
            gemm_load_tile<TA>(ra, A, lda, m0, k0 + GK, M, k_end, tid);
            gemm_load_tile<!TB>(rb, B, ldb, n0, k0 + GK, N, k_end, tid);
        }
#pragma unroll
        for (int kk = 0; kk < GK; ++kk) {
            float a[8], b[8];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (more) {
            gemm_store_tile<TA>(As[buf ^ 1], ra, tid);
            gemm_store_tile<!TB>(Bs[buf ^ 1], rb, tid);
            __syncthreads();
            buf ^= 1;
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int gn = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + j - 4);
            if (gn >= N) continue;
            float* c = C + (size_t)gm * ldc + gn;
            if (gridDim.z > 1) atomicAdd(c, acc[i][j]);
            else *c = accumulate ? *c + acc[i][j] : acc[i][j];
        }
    }
}

cudaError_t sgemm(cudaStream_t st, bool ta, bool tb, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
                  float* C, int ldc, bool accumulate) {
    dim3 grid((N + GN - 1) / GN, (M + GM - 1) / GM, 1);
    int kchunk = K;
    const int tiles = grid.x * grid.y;
    if (tiles < sat::device_sm_count() && K >= 512) {
        // few output tiles (batch-sized M, or weight gradients with a huge K): split K over the SMs and sum
        // with atomics.  A non-accumulating product starts from a zeroed C (ldc == N: contiguous).
        int z = (2 * sat::device_sm_count() + tiles - 1) / tiles;
        if (z > K / 128) z = K / 128;
        if (z < 1) z = 1;
        kchunk = ((K + z - 1) / z + GK - 1) / GK * GK;
        grid.z = (K + kchunk - 1) / kchunk;
        if (grid.z > 1 && !accumulate) {
            if (ldc != N) { grid.z = 1; kchunk = K; }
            else {
                cudaError_t e = cudaMemsetAsync(C, 0, (size_t)M * N * sizeof(float), st);
                if (e != cudaSuccess) return e;
            }
        }
    }
    const int acc = accumulate ? 1 : 0;
    if (!ta && !tb) launch_k(sgemm_kernel<false, false>, grid, 256, st, M, N, K, A, lda, B, ldb, C, ldc, acc, kchunk);
    else if (ta && !tb) launch_k(sgemm_kernel<true, false>, grid, 256, st, M, N, K, A, lda, B, ldb, C, ldc, acc, kchunk);
    else if (!ta && tb) launch_k(sgemm_kernel<false, true>, grid, 256, st, M, N, K, A, lda, B, ldb, C, ldc, acc, kchunk);
    else launch_k(sgemm_kernel<true, true>, grid, 256, st, M, N, K, A, lda, B, ldb, C, ldc, acc, kchunk);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------ element-wise
#define GRID1D(n) dim3((unsigned)(((n) + 255) / 256 < 65535 * 16 ? ((n) + 255) / 256 : 65535 * 16))

// y[r, c] = x[r, c] * drop(seed, stream, r * cols + c) ; x / y may have different leading dimensions
__global__ void dropout2d_kernel(float* y, int ldy, const float* x, int ldx, int rows, int cols,
                                 const unsigned long long* seedp, unsigned long long stream, float keep, int accumulate) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const size_t n = (size_t)rows * cols;
    if (ldx == cols && ldy == cols && !accumulate && (n & 3) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
        // dense case (the [B*L, D] contexts): four elements per thread, no index arithmetic beyond the linear index
        // (the mask of element i depends on i only, exactly as in the general path)
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* y4 = reinterpret_cast<float4*>(y);
        for (size_t i4 = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i4 < (n >> 2); i4 += (size_t)gridDim.x * blockDim.x) {
            float4 v = x4[i4];
            if (seed) {
                const unsigned long long i = i4 << 2;
                v.x *= drop_scale(seed, stream, i, keep);
                v.y *= drop_scale(seed, stream, i + 1, keep);
                v.z *= drop_scale(seed, stream, i + 2, keep);
                v.w *= drop_scale(seed, stream, i + 3, keep);
            }
            y4[i4] = v;
        }
        return;
    }
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i - (size_t)r * cols);
        const float s = seed ? drop_scale(seed, stream, i, keep) : 1.0f;
        const float v = x[(size_t)r * ldx + c] * s;
        float* o = y + (size_t)r * ldy + c;
        *o = accumulate ? *o + v : v;
    }
}
// y = act(x + b[c]) in place ; act 0 none, 1 tanh
__global__ void bias_act_kernel(float* x, const float* b, int rows, int cols, int act) {
    pdl_enter();
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float v = x[i] + (b ? b[i % cols] : 0.f);
        x[i] = act ? tanhf(v) : v;
    }
}
// dx = drop(dy) * (1 - y^2) in place on dy (dense [rows, cols]: mask index = linear index): the backward of
// y = tanh(.) followed by dropout
__global__ void drop_tanh_bwd_kernel(float* dy, const float* y, size_t n, const unsigned long long* seedp, unsigned long long stream,
                                     float keep, size_t per_step) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t ts = per_step ? i / per_step : 0;   // (stacked time steps: see concat3_drop_kernel)
        const float d = seed ? dy[i] * drop_scale(seed, stream + 16ull * ts, i - ts * per_step, keep) : dy[i];
        dy[i] = d * (1.0f - y[i] * y[i]);
    }
}
// dx = dy * (1 - y^2) in place on dy
__global__ void tanh_bwd_kernel(float* dy, const float* y, size_t n) {
    pdl_enter();
    if ((n & 3) == 0 && ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
        float4* d4 = reinterpret_cast<float4*>(dy);
        const float4* y4 = reinterpret_cast<const float4*>(y);
        for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (n >> 2); i += (size_t)gridDim.x * blockDim.x) {
            float4 d = d4[i];
            const float4 t = y4[i];
            d.x *= 1.0f - t.x * t.x; d.y *= 1.0f - t.y * t.y; d.z *= 1.0f - t.z * t.z; d.w *= 1.0f - t.w * t.w;
            d4[i] = d;
        }
        return;
    }
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dy[i] *= 1.0f - y[i] * y[i];
}
// db[c] += sum_r dx[r, c] * (w ? w[r] : 1)   (column sums, optionally row-weighted: the weight gradient of a
// one-column dense layer is dw[c] = sum_r x[r, c] * dy[r]).  Eight rows in flight per thread.
__global__ void colsum_kernel(float* db, const float* dx, int rows, int cols, const float* w = nullptr) {
    pdl_enter();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    const int r0 = blockIdx.y * 256, r1 = min(rows, r0 + 256);
    float s0 = 0.f, s1 = 0.f;
    int r = r0;
    for (; r + 8 <= r1; r += 8) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = dx[(size_t)(r + j) * cols + c];
        if (w) {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] *= w[r + j];
        }
        s0 += (v[0] + v[1]) + (v[2] + v[3]);
        s1 += (v[4] + v[5]) + (v[6] + v[7]);
    }
    for (; r < r1; ++r) s0 += dx[(size_t)r * cols + c] * (w ? w[r] : 1.f);
    atomicAdd(db + c, s0 + s1);
}
// out[r, :] = concat(a[r, :na], b[r, :nb], c[r, :nc]) with dropout on the first `ndrop` columns, mask index
// r * ndrop + col (= a dropout2d over a dense [rows, ndrop] matrix: one launch instead of three copies + one dropout)
// rows_per_step > 0: the rows are T stacked time steps of rows_per_step rows each; step t draws its mask from stream
// `stream + 16 t` with the row index inside the step (what T per-step launches with ST(t, k) would have drawn)
__global__ void concat3_drop_kernel(float* out, int ldo, const float* a, int na, const float* b, int nb, const float* c, int nc,
                                    int ndrop, int rows, const unsigned long long* seedp, unsigned long long stream, float keep,
                                    int rows_per_step, uint8_t* pa, int pa_mode, int pa_row_tile) {
    // pa (optional): the row also goes out as a packed operand of the wgmma dense kernel (row tile pa_row_tile, width
    // = cols, a multiple of 64): the product that consumes it needs no packing launch of its own
    pdl_enter();
    const unsigned long long seed = *seedp;
    const int cols = na + nb + nc;
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), col = (int)(i - (size_t)r * cols);
        float v = col < na ? a[(size_t)r * na + col] : col < na + nb ? b[(size_t)r * nb + col - na] : c[(size_t)r * nc + col - na - nb];
        if (seed && col < ndrop) {
            const int ts = rows_per_step ? r / rows_per_step : 0, rl = r - ts * rows_per_step;
            v *= drop_scale(seed, stream + 16ull * ts, (unsigned long long)rl * ndrop + col, keep);
        }
        out[(size_t)r * ldo + col] = v;
        if (pa) sat::pa_store(pa, pa_mode, pa_row_tile, cols >> 6, r, col, v);
    }
}
// y = drop(x) for a dense [rows, cols] matrix, also written as a packed operand (see concat3_drop_kernel)
__global__ void dropout_pack_kernel(float* y, const float* x, int rows, int cols, const unsigned long long* seedp,
                                    unsigned long long stream, float keep, uint8_t* pa, int pa_mode, int pa_row_tile) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i - (size_t)r * cols);
        const float v = seed ? x[i] * drop_scale(seed, stream, i, keep) : x[i];
        y[i] = v;
        sat::pa_store(pa, pa_mode, pa_row_tile, cols >> 6, r, c, v);
    }
}
// dx = dy * (1 - y^2) in place on dy [rows, cols], also written as a packed operand
__global__ void tanh_bwd_pack_kernel(float* dy, const float* y, int rows, int cols, uint8_t* pa, int pa_mode, int pa_row_tile) {
    pdl_enter();
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i - (size_t)r * cols);
        const float v = dy[i] * (1.0f - y[i] * y[i]);
        dy[i] = v;
        sat::pa_store(pa, pa_mode, pa_row_tile, cols >> 6, r, c, v);
    }
}
// y = drop(x) for T stacked dense steps of `per_step` elements each (streams as above)
__global__ void dropout_steps_kernel(float* y, const float* x, size_t n, size_t per_step, const unsigned long long* seedp,
                                     unsigned long long stream, float keep) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t ts = i / per_step;
        y[i] = seed ? x[i] * drop_scale(seed, stream + 16ull * ts, i - ts * per_step, keep) : x[i];
    }
}
// the transpose of the above: src[r, :] (dropout on the first ndrop columns) is split into three destinations, each
// either assigned or accumulated
__global__ void split3_drop_kernel(const float* src, int lds, int rows, float* a, int na, int acc_a, float* b, int nb, int acc_b,
                                   float* c, int nc, int acc_c, int ndrop, const unsigned long long* seedp,
                                   unsigned long long stream, float keep) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const int cols = na + nb + nc;
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), col = (int)(i - (size_t)r * cols);
        float v = src[(size_t)r * lds + col];
        if (seed && col < ndrop) v *= drop_scale(seed, stream, (unsigned long long)r * ndrop + col, keep);
        float* o;
        int acc;
        if (col < na) { o = a + (size_t)r * na + col; acc = acc_a; }
        else if (col < na + nb) { o = b + (size_t)r * nb + col - na; acc = acc_b; }
        else { o = c + (size_t)r * nc + col - na - nb; acc = acc_c; }
        *o = acc ? *o + v : v;
    }
}
__global__ void copy2d_kernel(float* y, int ldy, const float* x, int ldx, int rows, int cols, int accumulate) {
    pdl_enter();
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i - (size_t)r * cols);
        float* o = y + (size_t)r * ldy + c;
        const float v = x[(size_t)r * ldx + c];
        *o = accumulate ? *o + v : v;
    }
}
// Word ids index the embedding table and its gradient: an id outside [0, V) (TF's embedding_lookup / sparse softmax
// raise InvalidArgument on those) reads as a zero row, contributes no gradient and is counted in *bad (reported by
// sat_get_info "train_bad_ids"; the facade raises), instead of reading / corrupting neighbouring memory.
// rows_per_step > 0: rows are T stacked time steps, row r = (step r / rows_per_step, batch row r % rows_per_step), and
// idx is the [B, T] sentence matrix itself: step t looks up word t-1 of its row (teacher forcing), step 0 word id 0
__device__ __forceinline__ int step_word(const int32_t* idx, int idx_ld, int r, int rows_per_step) {
    if (!idx) return 0;
    if (!rows_per_step) return idx[(size_t)r * idx_ld];
    const int ts = r / rows_per_step, b = r - ts * rows_per_step;
    return ts ? idx[(size_t)b * idx_ld + ts - 1] : 0;
}
__global__ void gather_rows_kernel(float* y, int ldy, const float* table, int E, const int32_t* idx, int idx_ld, int rows, int V,
                                   float* bad, int rows_per_step) {
    pdl_enter();
    const size_t n = (size_t)rows * E;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / E), c = (int)(i - (size_t)r * E);
        const int w = step_word(idx, idx_ld, r, rows_per_step);
        const bool ok = (unsigned)w < (unsigned)V;
        if (!ok && c == 0) atomicAdd(bad, 1.0f);
        y[(size_t)r * ldy + c] = ok ? table[(size_t)w * E + c] : 0.f;
    }
}
__global__ void scatter_add_rows_kernel(float* dtable, int E, const int32_t* idx, int idx_ld, const float* dx, int ldx, int rows,
                                        int V, int rows_per_step) {
    pdl_enter();
    const size_t n = (size_t)rows * E;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(i / E), c = (int)(i - (size_t)r * E);
        const int w = step_word(idx, idx_ld, r, rows_per_step);
        if ((unsigned)w < (unsigned)V) atomicAdd(dtable + (size_t)w * E + c, dx[(size_t)r * ldx + c]);
    }
}
// temp[b*L + l, a] = (T1[b*L + l, a] + q[b, a]) * drop(att_mid)
__global__ void att_temp_kernel(float* temp, const float* T1, const float* q, int B, int L, int A,
                                const unsigned long long* seedp, unsigned long long stream, float keep) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const size_t n = (size_t)B * L * A;
    if ((A & 3) == 0 && n < (1ull << 33) && ((reinterpret_cast<uintptr_t>(temp) | reinterpret_cast<uintptr_t>(T1) | reinterpret_cast<uintptr_t>(q)) & 15) == 0) {
        const unsigned A4 = (unsigned)A >> 2, n4 = (unsigned)(n >> 2);
        for (unsigned i4 = blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += gridDim.x * blockDim.x) {
            const unsigned row = i4 / A4, a4 = i4 - row * A4, b = row / (unsigned)L;
            const float4 t = reinterpret_cast<const float4*>(T1)[i4];
            const float4 qq = reinterpret_cast<const float4*>(q)[(size_t)b * A4 + a4];
            float4 v = make_float4(t.x + qq.x, t.y + qq.y, t.z + qq.z, t.w + qq.w);
            if (seed) {
                const unsigned long long i = (unsigned long long)i4 << 2;
                v.x *= drop_scale(seed, stream, i, keep);
                v.y *= drop_scale(seed, stream, i + 1, keep);
                v.z *= drop_scale(seed, stream, i + 2, keep);
                v.w *= drop_scale(seed, stream, i + 3, keep);
            }
            reinterpret_cast<float4*>(temp)[i4] = v;
        }
        return;
    }
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int a = (int)(i % A);
        const int b = (int)(i / ((size_t)L * A));
        const float s = seed ? drop_scale(seed, stream, i, keep) : 1.0f;
        temp[i] = (T1[i] + q[(size_t)b * A + a]) * s;
    }
}
// e[b*L + l] = sum_a (T1[b*L + l, a] + q[b, a]) * drop(att_mid) * w2[a]: att_temp + rowdot in one pass over T1 (temp is
// not stored; the backward pass rebuilds it from T1, q and the mask).  One warp per row, A % 4 == 0.
// group > 1: T1 holds one [L, A] block per image and batch row b reads the block of image b / group
__global__ void att_logits_kernel(float* __restrict__ e, const float* __restrict__ T1, const float* __restrict__ q,
                                  const float* __restrict__ w2, int B, int L, int A,
                                  const unsigned long long* seedp, unsigned long long stream, float keep, int group = 1) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const DropGen gen = drop_gen(seed, stream, keep);
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (row >= B * L) return;
    const int A4 = A >> 2, b = row / L;
    const int trow = group == 1 ? row : (b / group) * L + (row - b * L);
    const float4* t4 = reinterpret_cast<const float4*>(T1) + (size_t)trow * A4;
    const float4* q4 = reinterpret_cast<const float4*>(q) + (size_t)b * A4;
    const float4* w4 = reinterpret_cast<const float4*>(w2);
    float s = 0.f;
#pragma unroll 4
    for (int a4 = lane; a4 < A4; a4 += 32) {
        const float4 t = t4[a4], qq = q4[a4], w = w4[a4];
        float4 v = make_float4(t.x + qq.x, t.y + qq.y, t.z + qq.z, t.w + qq.w);
        if (seed) {
            const unsigned long long i = ((unsigned long long)row * A4 + a4) << 2;
            v.x *= gen.scale(i);
            v.y *= gen.scale(i + 1);
            v.z *= gen.scale(i + 2);
            v.w *= gen.scale(i + 3);
        }
        s = fmaf(v.x, w.x, fmaf(v.y, w.y, fmaf(v.z, w.z, fmaf(v.w, w.w, s))));
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) e[row] = s;
}
// The backward pass of the scorer in one pass over T1 (A % 4 == 0).  With m = drop(att_mid) and de the logit gradient:
//   dtemp[r, a] = de[r] * w2[a] * m[r, a] * (1 - T1[r, a]^2)        (written: the gradient at the fc_1a pre-activation)
//   dq[b, a]   += sum_l de[r] * w2[a] * m[r, a]                      (dq zeroed by the caller)
//   dw2[a]     += sum_r (T1[r, a] + q[b, a]) * m[r, a] * de[r]
//   db[a]      += sum_r dtemp[r, a]                                  (db may be null)
// grid (ceil(A/256), row chunks, B), 256 threads = 4 row groups x 64 float4 columns.
constexpr int kAbRG = 4, kAbCT = 64;
__device__ __forceinline__ void att_bwd_fused_body(float* __restrict__ dtemp, float* dq, float* dw2, float* db,
                                                   const float* __restrict__ T1, const float* __restrict__ q,
                                                   const float* __restrict__ de, const float* __restrict__ w2, int L, int A,
                                                   int chunk_rows, const unsigned long long* seedp,
                                                   unsigned long long stream, float keep, const float* __restrict__ alpha) {
    pdl_enter();
    __shared__ float4 red[3][kAbRG - 1][kAbCT];
    // alpha != nullptr: `de` still holds d loss / d alpha and the softmax backward de = alpha (dalpha - sum alpha dalpha)
    // is taken here (every CTA of image b recomputes the L-term dot product) instead of in a launch of its own
    float sdot = 0.f;
    if (alpha) {
        __shared__ float sd[kAbRG * kAbCT / 32];
        float p = 0.f;
        for (int l = threadIdx.x; l < L; l += kAbRG * kAbCT) p = fmaf(alpha[(size_t)blockIdx.z * L + l], de[(size_t)blockIdx.z * L + l], p);
        for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
        if ((threadIdx.x & 31) == 0) sd[threadIdx.x >> 5] = p;
        __syncthreads();
        for (int w = 0; w < kAbRG * kAbCT / 32; ++w) sdot += sd[w];
    }
    const unsigned long long seed = *seedp;
    const DropGen gen = drop_gen(seed, stream, keep);
    const int ct = threadIdx.x % kAbCT, rg = threadIdx.x / kAbCT;
    const int A4 = A >> 2, c4 = blockIdx.x * kAbCT + ct, b = blockIdx.z;
    const int l0 = blockIdx.y * chunk_rows, l1 = min(L, l0 + chunk_rows);
    const bool on = c4 < A4;
    float4 aq = make_float4(0.f, 0.f, 0.f, 0.f), aw = aq, ab = aq;
    if (on) {
        const float4 w = reinterpret_cast<const float4*>(w2)[c4];
        const float4 qq = reinterpret_cast<const float4*>(q)[(size_t)b * A4 + c4];
#pragma unroll 4
        for (int l = l0 + rg; l < l1; l += kAbRG) {
            const size_t r = (size_t)b * L + l;
            const float4 t = reinterpret_cast<const float4*>(T1)[r * A4 + c4];
            const float d = alpha ? alpha[r] * (de[r] - sdot) : de[r];
            float4 m = make_float4(1.f, 1.f, 1.f, 1.f);
            if (seed) {
                const unsigned long long i = (r * A4 + c4) << 2;
                m.x = gen.scale(i);
                m.y = gen.scale(i + 1);
                m.z = gen.scale(i + 2);
                m.w = gen.scale(i + 3);
            }
            const float4 dm = make_float4(d * m.x, d * m.y, d * m.z, d * m.w);          // de * mask
            const float4 g = make_float4(dm.x * w.x, dm.y * w.y, dm.z * w.z, dm.w * w.w);  // d temp (before the mask: d (T1 + q))
            aq.x += g.x; aq.y += g.y; aq.z += g.z; aq.w += g.w;
            aw.x = fmaf(t.x + qq.x, dm.x, aw.x); aw.y = fmaf(t.y + qq.y, dm.y, aw.y);
            aw.z = fmaf(t.z + qq.z, dm.z, aw.z); aw.w = fmaf(t.w + qq.w, dm.w, aw.w);
            const float4 o = make_float4(g.x * (1.0f - t.x * t.x), g.y * (1.0f - t.y * t.y), g.z * (1.0f - t.z * t.z), g.w * (1.0f - t.w * t.w));
            ab.x += o.x; ab.y += o.y; ab.z += o.z; ab.w += o.w;
            reinterpret_cast<float4*>(dtemp)[r * A4 + c4] = o;
        }
    }
    if (rg > 0) { red[0][rg - 1][ct] = aq; red[1][rg - 1][ct] = aw; red[2][rg - 1][ct] = ab; }
    __syncthreads();
    if (rg == 0 && on) {
#pragma unroll
        for (int g = 0; g < kAbRG - 1; ++g) {
            const float4 x = red[0][g][ct], y = red[1][g][ct], z = red[2][g][ct];
            aq.x += x.x; aq.y += x.y; aq.z += x.z; aq.w += x.w;
            aw.x += y.x; aw.y += y.y; aw.z += y.z; aw.w += y.w;
            ab.x += z.x; ab.y += z.y; ab.z += z.z; ab.w += z.w;
        }
        float* pq = dq + ((size_t)b * A4 + c4) * 4;
        float* pw = dw2 + (size_t)c4 * 4;
        atomicAdd(pq, aq.x); atomicAdd(pq + 1, aq.y); atomicAdd(pq + 2, aq.z); atomicAdd(pq + 3, aq.w);
        atomicAdd(pw, aw.x); atomicAdd(pw + 1, aw.y); atomicAdd(pw + 2, aw.z); atomicAdd(pw + 3, aw.w);
        if (db) {
            float* pb = db + (size_t)c4 * 4;
            atomicAdd(pb, ab.x); atomicAdd(pb + 1, ab.y); atomicAdd(pb + 2, ab.z); atomicAdd(pb + 3, ab.w);
        }
    }
}
#define ATT_BWD_ARGS                                                                                                      \
    float *__restrict__ dtemp, float *dq, float *dw2, float *db, const float *__restrict__ T1, const float *__restrict__ q, \
        const float *__restrict__ de, const float *__restrict__ w2, int L, int A, int chunk_rows,                         \
        const unsigned long long *seedp, unsigned long long stream, float keep, const float *__restrict__ alpha
__global__ void __launch_bounds__(kAbRG* kAbCT) att_bwd_fused_kernel(ATT_BWD_ARGS) {
    att_bwd_fused_body(dtemp, dq, dw2, db, T1, q, de, w2, L, A, chunk_rows, seedp, stream, keep, alpha);
}
// the same held to 64 registers (4 CTAs per SM), for the one-resident-wave experiment (SAT_TRAIN_ATTBWD_WAVE=1)
__global__ void __launch_bounds__(kAbRG* kAbCT, 4) att_bwd_fused_wave_kernel(ATT_BWD_ARGS) {
    att_bwd_fused_body(dtemp, dq, dw2, db, T1, q, de, w2, L, A, chunk_rows, seedp, stream, keep, alpha);
}
#undef ATT_BWD_ARGS
// The same backward pass when the rows of an image share its T1 block (rows b = img * group + k, k < group; T1 and
// dtemp hold one [L, A] block per image).  Each (l, column) of the image's T1 chunk is read once per tile of kAbGT rows:
//   dtemp[img, l, a] = sum_k de[b, l] * w2[a] * m[b, l, a] * (1 - T1[img, l, a]^2)     (summed over the group)
//   dq[b, a] += sum_l de[b, l] * w2[a] * m[b, l, a]  per row; dw2 and db as above
// grid (ceil(A/256), row chunks, n_img); att_mid masks stay per row (index (b * L + l) * A + a, as in att_logits_kernel).
constexpr int kAbGT = kAbRG * kAbCT / 32;   // rows per tile: one warp computes the softmax dot product of one row
__global__ void __launch_bounds__(kAbRG* kAbCT) att_bwd_grouped_kernel(
    float* __restrict__ dtemp, float* dq, float* dw2, float* db, const float* __restrict__ T1, const float* __restrict__ q,
    const float* __restrict__ de, const float* __restrict__ w2, int L, int A, int chunk_rows, int group,
    const unsigned long long* seedp, unsigned long long stream, float keep, const float* __restrict__ alpha) {
    pdl_enter();
    __shared__ float4 red[kAbRG - 1][kAbCT];
    __shared__ float sd[kAbGT];
    const unsigned long long seed = *seedp;
    const DropGen gen = drop_gen(seed, stream, keep);
    const int ct = threadIdx.x % kAbCT, rg = threadIdx.x / kAbCT, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int A4 = A >> 2, c4 = blockIdx.x * kAbCT + ct, img = blockIdx.z;
    const int l0 = blockIdx.y * chunk_rows, l1 = min(L, l0 + chunk_rows);
    const bool on = c4 < A4;
    const float4 w = on ? reinterpret_cast<const float4*>(w2)[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 aw = make_float4(0.f, 0.f, 0.f, 0.f), ab = aw;
    // sum of a float4 over the kAbRG row groups, left in row group 0
    auto reduce_rg = [&](float4 v) -> float4 {
        __syncthreads();
        if (rg > 0) red[rg - 1][ct] = v;
        __syncthreads();
        if (rg == 0) {
#pragma unroll
            for (int g = 0; g < kAbRG - 1; ++g) {
                const float4 x = red[g][ct];
                v.x += x.x; v.y += x.y; v.z += x.z; v.w += x.w;
            }
        }
        return v;
    };
    for (int k0 = 0; k0 < group; k0 += kAbGT) {
        const int kn = min(kAbGT, group - k0);
        const size_t b0 = (size_t)img * group + k0;   // first batch row of this tile
        if (alpha) {   // softmax backward folded in: sd[j] = sum_l alpha[b, l] * dalpha[b, l] of row b0 + j
            __syncthreads();
            if (warp < kn) {
                float p = 0.f;
                for (int l = lane; l < L; l += 32) p = fmaf(alpha[(b0 + warp) * L + l], de[(b0 + warp) * L + l], p);
                for (int o = 16; o > 0; o >>= 1) p += __shfl_xor_sync(0xffffffffu, p, o);
                if (lane == 0) sd[warp] = p;
            }
            __syncthreads();
        }
        float4 aq[kAbGT];
#pragma unroll
        for (int j = 0; j < kAbGT; ++j) aq[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (on) {
            for (int l = l0 + rg; l < l1; l += kAbRG) {
                const size_t ti = ((size_t)img * L + l) * A4 + c4;
                const float4 t = reinterpret_cast<const float4*>(T1)[ti];
                float4 gs = make_float4(0.f, 0.f, 0.f, 0.f);   // sum over the tile's rows of d temp
#pragma unroll
                for (int j = 0; j < kAbGT; ++j) {
                    if (j < kn) {
                        const size_t r = (b0 + j) * L + l;
                        const float d = alpha ? alpha[r] * (de[r] - sd[j]) : de[r];
                        const float4 qq = reinterpret_cast<const float4*>(q)[(b0 + j) * A4 + c4];
                        float4 m = make_float4(1.f, 1.f, 1.f, 1.f);
                        if (seed) {
                            const unsigned long long i = (r * A4 + c4) << 2;
                            m.x = gen.scale(i);
                            m.y = gen.scale(i + 1);
                            m.z = gen.scale(i + 2);
                            m.w = gen.scale(i + 3);
                        }
                        const float4 dm = make_float4(d * m.x, d * m.y, d * m.z, d * m.w);
                        const float4 g = make_float4(dm.x * w.x, dm.y * w.y, dm.z * w.z, dm.w * w.w);
                        aq[j].x += g.x; aq[j].y += g.y; aq[j].z += g.z; aq[j].w += g.w;
                        gs.x += g.x; gs.y += g.y; gs.z += g.z; gs.w += g.w;
                        aw.x = fmaf(t.x + qq.x, dm.x, aw.x); aw.y = fmaf(t.y + qq.y, dm.y, aw.y);
                        aw.z = fmaf(t.z + qq.z, dm.z, aw.z); aw.w = fmaf(t.w + qq.w, dm.w, aw.w);
                    }
                }
                float4 o = make_float4(gs.x * (1.0f - t.x * t.x), gs.y * (1.0f - t.y * t.y), gs.z * (1.0f - t.z * t.z),
                                       gs.w * (1.0f - t.w * t.w));
                ab.x += o.x; ab.y += o.y; ab.z += o.z; ab.w += o.w;
                float4* pd = reinterpret_cast<float4*>(dtemp) + ti;
                if (k0) {   // (the same thread wrote this element for the previous tile)
                    const float4 p = *pd;
                    o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
                }
                *pd = o;
            }
        }
#pragma unroll
        for (int j = 0; j < kAbGT; ++j) {
            if (j < kn) {
                const float4 v = reduce_rg(aq[j]);
                if (rg == 0 && on) {
                    float* pq = dq + ((b0 + j) * A4 + c4) * 4;
                    atomicAdd(pq, v.x); atomicAdd(pq + 1, v.y); atomicAdd(pq + 2, v.z); atomicAdd(pq + 3, v.w);
                }
            }
        }
    }
    aw = reduce_rg(aw);
    ab = reduce_rg(ab);
    if (rg == 0 && on) {
        float* pw = dw2 + (size_t)c4 * 4;
        atomicAdd(pw, aw.x); atomicAdd(pw + 1, aw.y); atomicAdd(pw + 2, aw.z); atomicAdd(pw + 3, aw.w);
        if (db) {
            float* pb = db + (size_t)c4 * 4;
            atomicAdd(pb, ab.x); atomicAdd(pb + 1, ab.y); atomicAdd(pb + 2, ab.z); atomicAdd(pb + 3, ab.w);
        }
    }
}
// y[r, c] = x[r / group, c] for r < rows: image-level rows copied to each of the image's batch rows
__global__ void expand_rows_kernel(float* __restrict__ y, const float* __restrict__ x, int rows, int cols, int group) {
    pdl_enter();
    const size_t n = (size_t)rows * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / cols, c = i - r * cols;
        y[i] = x[(r / group) * cols + c];
    }
}
// y[i, c] = sum_k x[i * group + k, c] for i < n_img: the transpose of expand_rows_kernel
__global__ void group_sum_kernel(float* __restrict__ y, const float* __restrict__ x, int n_img, int cols, int group) {
    pdl_enter();
    const size_t n = (size_t)n_img * cols;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / cols, c = i - r * cols;
        const float* p = x + r * group * cols + c;
        float s = 0.f;
        for (int k = 0; k < group; ++k) s += p[(size_t)k * cols];
        y[i] = s;
    }
}
// e[r] = sum_a temp[r, a] * w2[a]       (one warp per row)
__global__ void rowdot_kernel(float* e, const float* temp, const float* w2, int rows, int A) {
    pdl_enter();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    float s = 0.f;
    for (int a = lane; a < A; a += 32) s = fmaf(temp[(size_t)warp * A + a], w2[a], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) e[warp] = s;
}
// softmax over L per row (one warp per row)
// and the attention coverage accumulator att[b, l] += alpha[b, l] * mask[b, t] (att == nullptr: skipped)
__global__ void softmax_rows_kernel(float* alpha, const float* e, int rows, int L, float* att, const float* masks, int mld, int t) {
    pdl_enter();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float* x = e + (size_t)warp * L;
    float m = -INFINITY;
    for (int l = lane; l < L; l += 32) m = fmaxf(m, x[l]);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int l = lane; l < L; l += 32) s += expf(x[l] - m);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mk = att ? masks[(size_t)warp * mld + t] : 0.f;
    for (int l = lane; l < L; l += 32) {
        const float a = expf(x[l] - m) / s;
        alpha[(size_t)warp * L + l] = a;
        if (att) att[(size_t)warp * L + l] += a * mk;
    }
}
// de = alpha * (dalpha - sum_l alpha*dalpha)   (one warp per row), written over dalpha
__global__ void softmax_bwd_kernel(float* dalpha, const float* alpha, int rows, int L) {
    pdl_enter();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    float s = 0.f;
    for (int l = lane; l < L; l += 32) s = fmaf(alpha[(size_t)warp * L + l], dalpha[(size_t)warp * L + l], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    for (int l = lane; l < L; l += 32) {
        const size_t i = (size_t)warp * L + l;
        dalpha[i] = alpha[i] * (dalpha[i] - s);
    }
}
// z[b, d] = sum_l alpha[b, l] * ctx[b / group, l, d]  (group > 1: the rows of an image share its contexts; likewise below)
__global__ void context_fwd_kernel(float* z, const float* alpha, const float* ctx, int B, int L, int D, int group = 1) {
    pdl_enter();
    const int b = blockIdx.y, d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    const float* c = ctx + (size_t)(b / group) * L * D + d;
    float s = 0.f;
    for (int l = 0; l < L; ++l) s = fmaf(alpha[(size_t)b * L + l], c[(size_t)l * D], s);
    z[(size_t)b * D + d] = s;
}
// the same on float4 columns with eight rows in flight per column: grid (ceil(D / 128), B), 256 threads =
// 8 row groups x 32 float4 columns, row groups summed through shared memory (D % 4 == 0, 16-byte aligned)
__global__ void __launch_bounds__(256) context_fwd4_kernel(float* __restrict__ z, const float* __restrict__ alpha,
                                                            const float* __restrict__ ctx, int L, int D, int group = 1) {
    pdl_enter();
    __shared__ float4 red[7][32];
    const int ct = threadIdx.x & 31, rg = threadIdx.x >> 5, b = blockIdx.y;
    const int D4 = D >> 2, c4 = blockIdx.x * 32 + ct;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < D4) {
        const float4* c = reinterpret_cast<const float4*>(ctx) + (size_t)(b / group) * L * D4 + c4;
        const float* al = alpha + (size_t)b * L;
#pragma unroll 4
        for (int l = rg; l < L; l += 8) {
            const float4 v = c[(size_t)l * D4];
            const float w = al[l];
            a.x = fmaf(w, v.x, a.x); a.y = fmaf(w, v.y, a.y); a.z = fmaf(w, v.z, a.z); a.w = fmaf(w, v.w, a.w);
        }
    }
    if (rg > 0) red[rg - 1][ct] = a;
    __syncthreads();
    if (rg == 0 && c4 < D4) {
#pragma unroll
        for (int g = 0; g < 7; ++g) {
            const float4 v = red[g][ct];
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        reinterpret_cast<float4*>(z)[(size_t)b * D4 + c4] = a;
    }
}
// softmax over the L scores of image b, then the context vector, in one launch: every CTA of the image (one per 128
// columns) recomputes the L-term softmax in shared memory (L <= kSmL) and the first one records alpha and the
// coverage accumulator att[b, l] += alpha[b, l] * mask[b, t] — what softmax_rows_kernel + context_fwd4_kernel do in
// two dependent launches, of which the first keeps 8 CTAs busy
constexpr int kSmL = 1024;
__global__ void __launch_bounds__(256) softmax_context_fwd4_kernel(float* __restrict__ z, float* __restrict__ alpha,
                                                                    const float* __restrict__ e, const float* __restrict__ ctx,
                                                                    int L, int D, float* att, const float* masks, int mld, int t,
                                                                    int group = 1) {
    pdl_enter();
    __shared__ float4 red[7][32];
    __shared__ float al_s[kSmL];
    __shared__ float rs[8];
    const int ct = threadIdx.x & 31, rg = threadIdx.x >> 5, b = blockIdx.y;
    const float* x = e + (size_t)b * L;
    float m = -INFINITY;
    for (int l = threadIdx.x; l < L; l += 256) m = fmaxf(m, x[l]);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (ct == 0) rs[rg] = m;
    __syncthreads();
    m = rs[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, rs[w]);
    __syncthreads();
    float sum = 0.f;
    for (int l = threadIdx.x; l < L; l += 256) {
        const float v = expf(x[l] - m);
        al_s[l] = v;
        sum += v;
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (ct == 0) rs[rg] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += rs[w];
    const float mk = att ? masks[(size_t)b * mld + t] : 0.f;
    for (int l = threadIdx.x; l < L; l += 256) {
        const float a = al_s[l] / sum;
        al_s[l] = a;
        if (blockIdx.x == 0) {
            alpha[(size_t)b * L + l] = a;
            if (att) att[(size_t)b * L + l] += a * mk;
        }
    }
    __syncthreads();
    const int D4 = D >> 2, c4 = blockIdx.x * 32 + ct;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < D4) {
        const float4* c = reinterpret_cast<const float4*>(ctx) + (size_t)(b / group) * L * D4 + c4;
#pragma unroll 4
        for (int l = rg; l < L; l += 8) {
            const float4 v = c[(size_t)l * D4];
            const float w = al_s[l];
            a.x = fmaf(w, v.x, a.x); a.y = fmaf(w, v.y, a.y); a.z = fmaf(w, v.z, a.z); a.w = fmaf(w, v.w, a.w);
        }
    }
    if (rg > 0) red[rg - 1][ct] = a;
    __syncthreads();
    if (rg == 0 && c4 < D4) {
#pragma unroll
        for (int g = 0; g < 7; ++g) {
            const float4 v = red[g][ct];
            a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
        }
        reinterpret_cast<float4*>(z)[(size_t)b * D4 + c4] = a;
    }
}
// dalpha[b, l] = sum_d dz[b, d] * ctx[b, l, d]  (+ extra[b, l] * mask[b, t] if given)   (one warp per (b, l))
__global__ void context_bwd_kernel(float* dalpha, const float* dz, const float* ctx, const float* extra, int B, int L, int D,
                                   const float* masks, int mld, int t, int group = 1) {
    pdl_enter();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B * L) return;
    const int b = warp / L;
    const size_t crow = group == 1 ? (size_t)warp : (size_t)(b / group) * L + (warp - b * L);
    float s = 0.f;
    for (int d = lane; d < D; d += 32) s = fmaf(dz[(size_t)b * D + d], ctx[crow * D + d], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    // extra = d coverage loss / d att (datt); it reaches alpha[b, l] of step t through att += alpha * mask[b, t]
    if (lane == 0) dalpha[warp] = s + (extra ? extra[warp] * masks[(size_t)b * mld + t] : 0.f);
}
// dtemp[r, a] = de[r] * w2[a] * drop(att_mid)   and  (1 - T1^2) applied later
__global__ void att_dtemp_kernel(float* dtemp, const float* de, const float* w2, int rows, int A,
                                 const unsigned long long* seedp, unsigned long long stream, float keep) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const size_t n = (size_t)rows * A;
    if ((A & 3) == 0 && n < (1ull << 33) && ((reinterpret_cast<uintptr_t>(dtemp) | reinterpret_cast<uintptr_t>(w2)) & 15) == 0) {
        const unsigned A4 = (unsigned)A >> 2, n4 = (unsigned)(n >> 2);
        for (unsigned i4 = blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += gridDim.x * blockDim.x) {
            const unsigned row = i4 / A4, a4 = i4 - row * A4;
            const float d = de[row];
            const float4 w = reinterpret_cast<const float4*>(w2)[a4];
            float4 v = make_float4(d * w.x, d * w.y, d * w.z, d * w.w);
            if (seed) {
                const unsigned long long i = (unsigned long long)i4 << 2;
                v.x *= drop_scale(seed, stream, i, keep);
                v.y *= drop_scale(seed, stream, i + 1, keep);
                v.z *= drop_scale(seed, stream, i + 2, keep);
                v.w *= drop_scale(seed, stream, i + 3, keep);
            }
            reinterpret_cast<float4*>(dtemp)[i4] = v;
        }
        return;
    }
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int a = (int)(i % A);
        const float s = seed ? drop_scale(seed, stream, i, keep) : 1.0f;
        dtemp[i] = de[i / A] * w2[a] * s;
    }
}
// dq[b, a] = sum_l dtemp[b*L + l, a]
__global__ void segsum_kernel(float* dq, const float* dtemp, int B, int L, int A) {
    pdl_enter();
    const int b = blockIdx.y, a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    float s = 0.f;
    for (int l = 0; l < L; ++l) s += dtemp[((size_t)b * L + l) * A + a];
    dq[(size_t)b * A + a] = s;
}
__device__ inline float sigm(float x) { return 1.0f / (1.0f + expf(-x)); }
// gates G [B, 4H] (blocks i, j, f, o) -> activated gates (in place), c, and the two dropped copies of
// h_raw = o * tanh(c): h_out = drop_out(h_raw) (mask stream st_out), h_state = drop_state(h_raw) (st_state)
__global__ void lstm_fwd_kernel(float* G, const float* bias, const float* c_prev, float* c, float* h_out, float* h_state, int B, int H,
                                const unsigned long long* seedp, unsigned long long st_out, unsigned long long st_state, float keep) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const size_t n = (size_t)B * H;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / H), u = (int)(i - (size_t)b * H);
        float* g = G + (size_t)b * 4 * H;
        const float gi = sigm(g[u] + bias[u]);
        const float gj = tanhf(g[H + u] + bias[H + u]);
        const float gf = sigm(g[2 * H + u] + bias[2 * H + u] + 1.0f);
        const float go = sigm(g[3 * H + u] + bias[3 * H + u]);
        const float cc = gf * c_prev[i] + gi * gj;
        g[u] = gi; g[H + u] = gj; g[2 * H + u] = gf; g[3 * H + u] = go;
        c[i] = cc;
        const float hr = go * tanhf(cc);
        h_out[i] = seed ? hr * drop_scale(seed, st_out, i, keep) : hr;
        h_state[i] = seed ? hr * drop_scale(seed, st_state, i, keep) : hr;
    }
}
// dh_raw = drop_out(dh_out) + drop_state(dh_state) (the masks of the forward pass), dc (in/out: on entry dc = gradient
// flowing into c_t from step t+1) -> dG (pre-activation), dc_prev
__global__ void lstm_bwd_kernel(float* dG, float* dc, const float* dh_out, const float* dh_state, const float* acts, const float* c,
                                const float* c_prev, int B, int H, const unsigned long long* seedp, unsigned long long st_out,
                                unsigned long long st_state, float keep, uint8_t* pa, int pa_mode, int pa_row_tile) {
    pdl_enter();
    const unsigned long long seed = *seedp;
    const size_t n = (size_t)B * H;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / H), u = (int)(i - (size_t)b * H);
        const float* a = acts + (size_t)b * 4 * H;
        const float gi = a[u], gj = a[H + u], gf = a[2 * H + u], go = a[3 * H + u];
        const float tc = tanhf(c[i]);
        const float dh = seed ? dh_out[i] * drop_scale(seed, st_out, i, keep) + dh_state[i] * drop_scale(seed, st_state, i, keep)
                              : dh_out[i] + dh_state[i];
        const float dcc = dh * go * (1.0f - tc * tc) + dc[i];
        float* d = dG + (size_t)b * 4 * H;
        const float di = dcc * gj * gi * (1.0f - gi), dj = dcc * gi * (1.0f - gj * gj), df = dcc * c_prev[i] * gf * (1.0f - gf),
                    d_o = dh * tc * go * (1.0f - go);
        d[u] = di;
        d[H + u] = dj;
        d[2 * H + u] = df;
        d[3 * H + u] = d_o;
        if (pa) {   // d G as the packed operand of the input-gradient product (see concat3_drop_kernel)
            const int kb = (4 * H) >> 6;
            sat::pa_store(pa, pa_mode, pa_row_tile, kb, b, u, di);
            sat::pa_store(pa, pa_mode, pa_row_tile, kb, b, H + u, dj);
            sat::pa_store(pa, pa_mode, pa_row_tile, kb, b, 2 * H + u, df);
            sat::pa_store(pa, pa_mode, pa_row_tile, kb, b, 3 * H + u, d_o);
        }
        dc[i] = dcc * gf;
    }
}
// masked cross entropy of one time step + its gradient; one block per row
constexpr int kCeThreads = 1024;   // one CTA per batch row: the three passes over the V logits are latency bound
// (rows_per_step > 0: block r is row r % rows_per_step of time step t + r / rows_per_step — all T steps in one launch)
// kWeighted: the gradient and the cross entropy of row b are scaled by row_w[b] (a policy-gradient advantage, any sign);
// the accuracy is not
template <bool kWeighted>
__global__ void __launch_bounds__(kCeThreads) ce_kernel(const float* logits, float* dlogits, const int32_t* sent, int sent_ld, int t,
                                                        const float* masks, int V, const float* inv_msum_p, float* loss_acc,
                                                        int rows_per_step, const float* row_w) {
    pdl_enter();
    constexpr int NW = kCeThreads / 32;
    const float inv_msum = *inv_msum_p;
    __shared__ float red[NW];
    __shared__ int redi[NW];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int b = blockIdx.x;
    if (rows_per_step) { t += b / rows_per_step; b = b % rows_per_step; }
    const float* x = logits + (size_t)blockIdx.x * V;
    float* d = dlogits + (size_t)blockIdx.x * V;
    float m = -INFINITY;
    int mi = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += kCeThreads) {
        const float v = x[i];
        if (v > m || (v == m && i < mi)) { m = v; mi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, m, o);
        const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        if (ov > m || (ov == m && oi < mi)) { m = ov; mi = oi; }
    }
    if (lane == 0) { red[warp] = m; redi[warp] = mi; }
    __syncthreads();
    m = red[0]; mi = redi[0];
    for (int w = 1; w < NW; ++w)
        if (red[w] > m || (red[w] == m && redi[w] < mi)) { m = red[w]; mi = redi[w]; }
    __syncthreads();
    float s = 0.f;
    for (int i = threadIdx.x; i < V; i += kCeThreads) {   // e^{x - m} is kept in dlogits for the last pass (same thread, same i)
        const float e = expf(x[i] - m);
        d[i] = e;
        s += e;
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    s = 0.f;
    for (int w = 0; w < NW; ++w) s += red[w];
    const int y_raw = sent[(size_t)b * sent_ld + t];
    const bool y_ok = (unsigned)y_raw < (unsigned)V;      // (an id outside the vocabulary: no target, counted as bad)
    const int y = y_ok ? y_raw : 0;
    const float mk = y_ok ? masks[(size_t)b * sent_ld + t] : 0.f;
    const float scale = kWeighted ? mk * inv_msum * row_w[b] : mk * inv_msum;
    for (int i = threadIdx.x; i < V; i += kCeThreads) {
        const float p = d[i] / s;
        d[i] = (p - (i == y ? 1.0f : 0.0f)) * scale;
    }
    if (threadIdx.x == 0) {
        if (!y_ok) atomicAdd(loss_acc + 5, 1.0f);
        const float ce = logf(s) + m - x[y];
        atomicAdd(loss_acc + 0, ce * scale);                       // cross entropy (already / sum of masks)
        atomicAdd(loss_acc + 1, (mi == y ? mk : 0.0f) * inv_msum);  // accuracy
    }
}
// loss = factor * sum (1 - att)^2 / 2 / (GB * L);  datt = -factor * (1 - att) / (GB * L)
__global__ void coverage_loss_kernel(float* datt, const float* att, int n, float factor, float inv_gbl, float* loss_acc) {
    pdl_enter();
    __shared__ float red[8];
    float s = 0.f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float d = 1.0f - att[i];
        s += d * d;
        datt[i] = -factor * d * inv_gbl;
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < (int)blockDim.x / 32; ++w) t += red[w];
        atomicAdd(loss_acc + 2, t * 0.5f * factor * inv_gbl);
    }
}
__global__ void mean_L_kernel(float* out, const float* ctx, int L, int D) {
    pdl_enter();
    const int b = blockIdx.y, d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= D) return;
    float s = 0.f;
    for (int l = 0; l < L; ++l) s += ctx[((size_t)b * L + l) * D + d];
    out[(size_t)b * D + d] = s / (float)L;
}
// out[0] += scale * sum x^2
__global__ void sumsq_kernel(const float* x, size_t n, float scale, float* out) {
    pdl_enter();
    __shared__ float red[8];
    float s = 0.f;
    const size_t tid = blockIdx.x * (size_t)blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
    size_t head = 0;   // elements covered by the float4 loop
    if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
        const float4* x4 = reinterpret_cast<const float4*>(x);
        const size_t n4 = n >> 2;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
        for (size_t i = tid; i < n4; i += nth) {
            const float4 v = x4[i];
            a.x = fmaf(v.x, v.x, a.x); a.y = fmaf(v.y, v.y, a.y); a.z = fmaf(v.z, v.z, a.z); a.w = fmaf(v.w, v.w, a.w);
        }
        s = (a.x + a.y) + (a.z + a.w);
        head = n4 << 2;
    }
    for (size_t i = head + tid; i < n; i += nth) s = fmaf(x[i], x[i], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < (int)blockDim.x / 32; ++w) t += red[w];
        atomicAdd(out, t * scale);
    }
}
__global__ void axpy_kernel(float* y, const float* x, float a, size_t n) {
    pdl_enter();
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) y[i] = fmaf(a, x[i], y[i]);
}
// clip_by_global_norm + TF Adam.  norm2 = sum of squares of the (already reduced, regularised) gradient
__global__ void adam_kernel(float* w, const float* g, float* m, float* v, size_t n, const float* norm2, float clip, float lr_t,
                            float b1, float b2, float eps) {
    pdl_enter();
    const float norm = sqrtf(*norm2);
    const float scale = clip > 0.f ? clip / fmaxf(norm, clip) : 1.0f;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float gi = g[i] * scale;
        const float mi = b1 * m[i] + (1.0f - b1) * gi;
        const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        w[i] -= lr_t * mi / (sqrtf(vi) + eps);
    }
}

// The other optimizers of model.py:486-503 (TF 1.x update rules), after the same global-norm clip:
//   RMSProp   ms = decay ms + (1-decay) g^2 ; [centered: mg = decay mg + (1-decay) g] ;
//             mom = momentum mom + lr g / sqrt(ms [- mg^2] + eps) ; w -= mom            (slots: ms starts at ONE)
//   Momentum  acc = momentum acc + g ; w -= nesterov ? lr (g + momentum acc) : lr acc
//   SGD       w -= lr g
__global__ void rmsprop_kernel(float* w, const float* g, float* ms, float* mg, float* mom, size_t n, const float* norm2, float clip,
                               float lr, float decay, float momentum, float eps, int centered) {
    pdl_enter();
    const float norm = sqrtf(*norm2);
    const float scale = clip > 0.f ? clip / fmaxf(norm, clip) : 1.0f;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float gi = g[i] * scale;
        const float msi = decay * ms[i] + (1.0f - decay) * gi * gi;
        ms[i] = msi;
        float denom = msi;
        if (centered) {
            const float mgi = decay * mg[i] + (1.0f - decay) * gi;
            mg[i] = mgi;
            denom = msi - mgi * mgi;
        }
        const float mi = momentum * mom[i] + lr * gi / sqrtf(denom + eps);
        mom[i] = mi;
        w[i] -= mi;
    }
}
__global__ void momentum_kernel(float* w, const float* g, float* acc, size_t n, const float* norm2, float clip, float lr, float momentum,
                                int nesterov, int plain_sgd) {
    pdl_enter();
    const float norm = sqrtf(*norm2);
    const float scale = clip > 0.f ? clip / fmaxf(norm, clip) : 1.0f;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float gi = g[i] * scale;
        if (plain_sgd) { w[i] -= lr * gi; continue; }
        const float a = momentum * acc[i] + gi;
        acc[i] = a;
        w[i] -= nesterov ? lr * gi + lr * momentum * a : lr * a;
    }
}
__global__ void fill_kernel(float* x, float v, size_t n) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) x[i] = v;
}

// ------------------------------------------------------------------------------------------ state
enum Var { vEmb = 0, vIa1W, vIa1B, vIa2W, vIa2B, vIb1W, vIb1B, vIb2W, vIb2B, vA1aW, vA1aB, vA1bW, vA1bB, vA2W, vLW, vLB,
           vD1W, vD1B, vD2W, vD2B, kNumVars };
// names of the 2-layer graph; the 1-layer variants of initialize / attend / decode (model.py:362-371, 401-414, 442-447)
// reuse the first-layer slots under the reference's names for them and leave the second-layer slots empty (fill_layout)
const char* kVarNames[kNumVars] = {
    "word_embedding/weights", "initialize/fc_a1/kernel", "initialize/fc_a1/bias", "initialize/fc_a2/kernel",
    "initialize/fc_a2/bias", "initialize/fc_b1/kernel", "initialize/fc_b1/bias", "initialize/fc_b2/kernel",
    "initialize/fc_b2/bias", "attend/fc_1a/kernel", "attend/fc_1a/bias", "attend/fc_1b/kernel", "attend/fc_1b/bias",
    "attend/fc_2/kernel", "lstm/lstm_cell/kernel", "lstm/lstm_cell/bias", "decode/fc_1/kernel", "decode/fc_1/bias",
    "decode/fc_2/kernel", "decode/fc_2/bias"};

struct TrainState {
    sat_dims d;
    int B = 0, T = 0;
    // B = n_img * group batch rows; row r is a caption of image r / group.  What depends on the image alone (context
    // mean, initialize, attend/fc_1a and its T1 stash) is computed on n_img rows, the rest on B rows.
    int n_img = 0, group = 1;
    float *c0i = nullptr, *h0i = nullptr, *dci = nullptr, *dhi = nullptr;   // group > 1: image-level c0 / h0 and gradients
    float *e_img = nullptr, *dtemp_g = nullptr;   // group > 1: 1-layer image scores / group-summed d temp (non-fused scorer)
    float keep_fc = 0.5f, keep_lstm = 0.7f, att_factor = 0.01f, reg_scale = 1e-4f;
    size_t off[kNumVars + 1];
    int rows[kNumVars], cols[kNumVars];
    bool regularised[kNumVars];
    const char* names[kNumVars];
    int present[kNumVars], num_present = 0;   // slots in use, in enumeration order (sat_train_var)
    // stashes (index [t])
    std::vector<float*> T1, q, hd, alpha, z, lstm_in, acts, c, h_out, h_state, expd, t1, td, dlogits, emb;
    float *ctxd = nullptr, *temp = nullptr, *e = nullptr, *G = nullptr, *logits = nullptr;
    float *mean = nullptr, *meand = nullptr, *ia1 = nullptr, *ia1d = nullptr, *ib1 = nullptr, *ib1d = nullptr, *c0 = nullptr,
          *h0 = nullptr;
    float *att = nullptr, *datt = nullptr;
    // backward scratch
    float *dtd = nullptr, *dexp = nullptr, *dh_out = nullptr, *dh_state = nullptr, *dc = nullptr, *dG = nullptr,
          *dlin = nullptr, *dz = nullptr, *demb = nullptr, *dalpha = nullptr, *dtemp = nullptr, *dq = nullptr, *dhd = nullptr,
          *dbuf = nullptr;
    // tensor-core path of attend/fc_1a (forward + weight gradient: ~25 % of the step's time on CUDA cores): the
    // operands in the packed layouts of the wgmma dense kernel
    uint8_t *tc_xpa = nullptr, *tc_wbig = nullptr, *tc_w1a = nullptr;   // packed rows / packed [BL x A] "weight" / packed W1a
    float* tc_b1a = nullptr;
    bool tc_ok = false;
    // batch-row products (rows = B) of the step: y = x W (+ b) forward and dx = dy W^T backward, with this step's
    // weights packed once (W as the kernel's weight operand, W^T likewise through the row packer)
    struct TcLayer {
        int var_w = -1, var_b = -1, K = 0, N = 0;
        uint8_t *w = nullptr, *wT = nullptr;
        float* b = nullptr;
        bool fwd = false, dx = false;
    } tcl[4];   // 0 attend/fc_1b, 1 lstm, 2 decode/fc_1, 3 decode/fc_2
    uint8_t* tc_xs = nullptr;   // packed batch rows (scratch)
    int tc_rt = 0;              // their row tile
    // weight gradients of those layers: dW = sum_t x_t^T dy_t = X_all^T dY_all with the T steps stacked ([T*B, .]
    // matrices: the per-step stashes are contiguous), one tensor-core product per layer after the time loop
    // input gradient of decode/fc_2: K = V is not a multiple of the 64-wide K block; its two operands get buffers of
    // their own, zeroed once, so that the unwritten tail of the last K block stays zero
    uint8_t *tc_vx = nullptr, *tc_vw = nullptr;
    int tc_vk = 0;                         // V rounded up to K blocks (0 = path off)
    std::vector<float*> dys[4];            // [t] slices of dY_all per layer (decode/fc_2 uses dlogits)
    uint8_t *tc_sx = nullptr, *tc_sw = nullptr;   // packed X_all^T / packed dY_all
    bool tc_stack = false;
    // decode layers of all T steps at once (teacher forcing: nothing in the recurrence consumes the logits, so the two
    // layers and their input gradients are [T*B]-row products after / before the time loops instead of 4 T products
    // of B rows that each stream the whole weight matrix)
    bool dec_all = false;
    int all_rt = 0, all_rows = 0;                 // row tile of the stacked rows, rows rounded up to it
    float *logits_all = nullptr, *dexp_all = nullptr;
    float* demb_all = nullptr;                    // d emb of every step: ONE scatter into the embedding gradient after the loop
    uint8_t* tc_vx_all = nullptr;
    // the [B*L]-row products of attend/fc_1a are outside the recurrence (forward: T1[t] needs only ctx and the mask of
    // step t; backward: nothing waits for dW1a): they run on a second, low-priority stream beside the batch-row work
    // of the time loops, joined through events (graph edges once the step is captured)
    cudaStream_t side = nullptr;
    std::vector<cudaEvent_t> ev;          // [0] fork, [1] join, then T x {T1 ready, scorer backward done, dtemp packed}
    float* dtemp2 = nullptr;              // second d temp buffer: the scorer backward of step t-1 beside the product of step t
    sat_handle* handle = nullptr;
    float* loss_acc = nullptr;   // [0] ce, [1] accuracy, [2] attention, [3] reg, [4] grad norm^2, [5] out-of-vocabulary ids seen
                                 // by the last forward pass ([6] the same, accumulated since sat_train_init)
    // per-call scalars live in device cells (fed by small stream-ordered copies before each launch), so that the
    // ~3500 launches of a step are captured once into a CUDA graph and replayed
    unsigned long long* seed_d = nullptr;
    float* inv_msum_d = nullptr;
    struct GEntry { std::vector<long long> key; int seen = 0; cudaGraphExec_t exec = nullptr; };
    std::vector<GEntry> graphs;
    std::vector<void*> all;
};

int talloc(TrainState* s, float** p, size_t n) {
    cudaError_t e = cudaMalloc((void**)p, (n ? n : 1) * sizeof(float));
    if (e != cudaSuccess) return sat_fail(SAT_ERR_NOMEM, "training buffer of %zu floats: %s", n, cudaGetErrorString(e));
    s->all.push_back(*p);
    return SAT_OK;
}

void train_free(void* p) {
    TrainState* s = (TrainState*)p;
    if (!s) return;
    for (void* b : s->all) cudaFree(b);
    for (auto& g : s->graphs)
        if (g.exec) cudaGraphExecDestroy(g.exec);
    for (cudaEvent_t e : s->ev) cudaEventDestroy(e);
    if (s->side) cudaStreamDestroy(s->side);
    delete s;
}

}  // namespace

// =========================================================================================== C ABI
// the dropout generator on the host: lets a CPU test pin it against the numpy copy in oracle/train_ref.py
extern "C" float sat_train_rng_uniform(uint64_t seed, uint64_t stream, uint64_t index) { return rng_u24(seed, stream, index); }

static void fill_layout(TrainState* s) {
    const sat_dims& d = s->d;
    const int D = d.dim_ctx, E = d.dim_embedding, H = d.num_lstm_units, A = d.dim_attend_layer, Dd = d.dim_decode_layer,
              I = d.dim_initalize_layer, V = d.vocabulary_size, L = d.num_ctx;
    int shp[kNumVars][2] = {{V, E}, {D, I}, {1, I}, {I, H}, {1, H}, {D, I}, {1, I}, {I, H}, {1, H}, {D, A}, {1, A}, {H, A},
                            {1, A}, {A, 1}, {D + E + H, 4 * H}, {1, 4 * H}, {H + D + E, Dd}, {1, Dd}, {Dd, V}, {1, V}};
    for (int i = 0; i < kNumVars; ++i) s->names[i] = kVarNames[i];
    auto set = [&](int v, const char* name, int r, int c) { s->names[v] = name; shp[v][0] = r; shp[v][1] = c; };
    if (d.num_initalize_layers == 1) {        // memory = fc_a(mean), output = fc_b(mean)                 model.py:362-371
        set(vIa1W, "initialize/fc_a/kernel", D, H); set(vIa1B, "initialize/fc_a/bias", 1, H);
        set(vIb1W, "initialize/fc_b/kernel", D, H); set(vIb1B, "initialize/fc_b/bias", 1, H);
        set(vIa2W, nullptr, 0, 0); set(vIa2B, nullptr, 0, 0); set(vIb2W, nullptr, 0, 0); set(vIb2B, nullptr, 0, 0);
    }
    if (d.num_attend_layers == 1) {           // logits = fc_a(ctx)[BL,1] + fc_b(h)[B,L], both without bias model.py:401-414
        set(vA1aW, "attend/fc_a/kernel", D, 1); set(vA1bW, "attend/fc_b/kernel", H, L);
        set(vA1aB, nullptr, 0, 0); set(vA1bB, nullptr, 0, 0); set(vA2W, nullptr, 0, 0);
    }
    if (d.num_decode_layers == 1) {           // logits = fc(expanded)                                    model.py:442-447
        set(vD1W, "decode/fc/kernel", H + D + E, V); set(vD1B, "decode/fc/bias", 1, V);
        set(vD2W, nullptr, 0, 0); set(vD2B, nullptr, 0, 0);
    }
    size_t o = 0;
    s->num_present = 0;
    for (int i = 0; i < kNumVars; ++i) {
        s->off[i] = o;
        s->rows[i] = shp[i][0];
        s->cols[i] = shp[i][1];
        o += ((size_t)shp[i][0] * shp[i][1] + 31) / 32 * 32;
        if (s->names[i]) s->present[s->num_present++] = i;
        // L2-regularised: embedding + every dense kernel, not the LSTM kernel, not biases (nn.py:33-37)
        s->regularised[i] = s->names[i] && ((i == vEmb) || (shp[i][0] > 1 && i != vLW));
    }
    s->off[kNumVars] = o;
}

extern "C" int sat_train_num_vars(sat_handle* h) {
    if (!h) return kNumVars;
    TrainState tmp;
    tmp.d = *sat_handle_dims(h);
    fill_layout(&tmp);
    return tmp.num_present;
}

extern "C" int sat_train_init_grouped(sat_handle* h, int32_t n_img, int32_t group, int32_t T, float fc_drop_rate,
                                      float lstm_drop_rate, float attention_loss_factor, float fc_kernel_regularizer_scale) {
    if (!h) return sat_fail(SAT_ERR_INVALID, "null handle");
    const sat_dims* dp = sat_handle_dims(h);
    for (int nl : {dp->num_attend_layers, dp->num_decode_layers, dp->num_initalize_layers})
        if (nl != 1 && nl != 2) return sat_fail(SAT_ERR_UNSUPPORTED, "attend/decode/initialize have 1 or 2 layers (got %d)", nl);
    if (n_img < 1 || group < 1 || T < 1 || (int64_t)n_img * group > INT32_MAX) return sat_fail(SAT_ERR_INVALID, "bad B/T");
    const int32_t B = n_img * group;
    TCK(cudaSetDevice(sat_handle_device(h)));
    void** slot = sat_handle_train_slot(h);
    if (*slot) { train_free(*slot); *slot = nullptr; }
    TrainState* s = new TrainState();
    s->d = *dp;
    s->B = B;
    s->T = T;
    s->n_img = n_img;
    s->group = group;
    s->keep_fc = (float)(1.0 - (double)fc_drop_rate);      // same value as numpy's float32(1 - rate)
    s->keep_lstm = (float)(1.0 - (double)lstm_drop_rate);
    s->att_factor = attention_loss_factor;
    s->reg_scale = fc_kernel_regularizer_scale;
    fill_layout(s);
    const sat_dims& d = s->d;
    const size_t BL = (size_t)B * d.num_ctx, D = d.dim_ctx, E = d.dim_embedding, H = d.num_lstm_units, A = d.dim_attend_layer,
                 Dd = d.dim_decode_layer, I = d.dim_initalize_layer, V = d.vocabulary_size, L = d.num_ctx;
    int rc = SAT_OK;
    auto A1 = [&](float** p, size_t n) { if (rc == SAT_OK) rc = talloc(s, p, n); };
    auto AT = [&](std::vector<float*>& v, size_t n) {   // one block, [t] = slice t: the T slices also form a [T*B, .] matrix
        v.assign(T, nullptr);
        float* base = nullptr;
        A1(&base, n * T);
        for (int t = 0; t < T && base; ++t) v[t] = base + (size_t)t * n;
    };
    const size_t NI = (size_t)n_img, BLi = NI * L;   // image-level rows
    AT(s->T1, BLi * A); AT(s->q, B * A); AT(s->hd, B * H); AT(s->alpha, B * L); AT(s->z, B * D); AT(s->lstm_in, B * (D + E + H));
    AT(s->acts, B * 4 * H); AT(s->c, B * H); AT(s->h_out, B * H); AT(s->h_state, B * H); AT(s->expd, B * (H + D + E));
    AT(s->t1, B * Dd); AT(s->td, B * Dd); AT(s->dlogits, B * V); AT(s->emb, B * E);
    A1(&s->ctxd, BLi * D); A1(&s->temp, BL * A); A1(&s->e, BL); A1(&s->G, B * 4 * H); A1(&s->logits, B * V);
    A1(&s->mean, NI * D); A1(&s->meand, NI * D); A1(&s->ia1, NI * I); A1(&s->ia1d, NI * I); A1(&s->ib1, NI * I); A1(&s->ib1d, NI * I);
    A1(&s->c0, B * H); A1(&s->h0, B * H); A1(&s->att, BL); A1(&s->datt, BL);
    if (group > 1) {
        A1(&s->c0i, NI * H); A1(&s->h0i, NI * H); A1(&s->dci, NI * H); A1(&s->dhi, NI * H);
        A1(&s->e_img, BLi); A1(&s->dtemp_g, BLi * A);
    }
    A1(&s->dtd, B * Dd); A1(&s->dexp, B * (H + D + E)); A1(&s->dh_out, B * H); A1(&s->dh_state, B * H);
    A1(&s->dc, B * H); A1(&s->dG, B * 4 * H); A1(&s->dlin, B * (D + E + H)); A1(&s->dz, B * D); A1(&s->demb, B * E);
    A1(&s->dalpha, BL); A1(&s->dtemp, BL * A); A1(&s->dq, B * A); A1(&s->dhd, B * H); A1(&s->dbuf, B * (D + E + I + H));
    A1(&s->loss_acc, 8);
    A1(&s->demb_all, (size_t)T * B * E);
    s->handle = h;
    const bool att2 = d.num_attend_layers == 2, dec2 = d.num_decode_layers == 2;
    s->tc_ok = att2 && (D % 128 == 0) && (A % 128 == 0) && (BLi % 128 == 0);
    if (s->tc_ok) {
        float* f = nullptr;   // (sizes in floats: a packed operand takes 4 bytes per element, like fp32)
        A1(&f, BLi * D); s->tc_xpa = reinterpret_cast<uint8_t*>(f);
        A1(&f, BLi * (A > D ? A : D)); s->tc_wbig = reinterpret_cast<uint8_t*>(f);
        A1(&f, D * A); s->tc_w1a = reinterpret_cast<uint8_t*>(f);
        A1(&s->tc_b1a, A);
        A1(&s->dtemp2, BLi * A);   // (used by the fused scorer only, which writes image-level d temp)
        int lo_pri = 0, hi_pri = 0;
        cudaDeviceGetStreamPriorityRange(&lo_pri, &hi_pri);
        if (rc == SAT_OK && cudaStreamCreateWithPriority(&s->side, cudaStreamNonBlocking, lo_pri) == cudaSuccess) {
            s->ev.assign(2 + 3 * (size_t)T, nullptr);
            for (auto& e : s->ev)
                if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) rc = sat_fail(SAT_ERR_CUDA, "event creation failed");
        } else {
            s->side = nullptr;
        }
    }
    {
        const size_t XLs = D + E + H, XDs = H + D + E;
        const int vw[4] = {vA1bW, vLW, vD1W, vD2W}, vb[4] = {vA1bB, vLB, vD1B, vD2B};
        const size_t Ks[4] = {H, XLs, XDs, Dd}, Ns[4] = {A, 4 * H, Dd, V};
        size_t kmax = 0;
        s->tc_rt = (int)((B + 15) / 16 * 16);
        for (int i = 0; i < 4; ++i) {
            TrainState::TcLayer& l = s->tcl[i];
            l.var_w = vw[i]; l.var_b = vb[i]; l.K = (int)Ks[i]; l.N = (int)Ns[i];
            // (the 1-layer variants of attend / decode stay on the CUDA-core products: they are not the shipped graph)
            const bool used = i == 1 || (i == 0 ? att2 : dec2);
            l.fwd = used && (Ks[i] % 64 == 0) && s->tc_rt <= sat::kMaxRowTile;
            l.dx = l.fwd && (Ns[i] % 64 == 0);
            float* f = nullptr;
            const size_t npad = (Ns[i] + 127) / 128 * 128, kpad = (Ks[i] + 127) / 128 * 128;
            if (l.fwd) { A1(&f, Ks[i] * npad); l.w = reinterpret_cast<uint8_t*>(f); A1(&l.b, npad); }
            if (l.dx) { A1(&f, Ns[i] * kpad); l.wT = reinterpret_cast<uint8_t*>(f); }
            kmax = Ks[i] > kmax ? Ks[i] : kmax;
            kmax = (l.dx && Ns[i] > kmax) ? Ns[i] : kmax;
        }
        float* f = nullptr;
        A1(&f, (size_t)(s->tc_rt + 16) * kmax);
        s->tc_xs = reinterpret_cast<uint8_t*>(f);
        // (producers that write their rows here directly never touch the padding rows of the tile: zero once)
        if (rc == SAT_OK) cudaMemset(s->tc_xs, 0, (size_t)(s->tc_rt + 16) * kmax * 4);
        if (s->tcl[3].fwd && V % 8 == 0) {
            s->tc_vk = (int)((V + 63) / 64 * 64);
            const size_t ddp = (Dd + 127) / 128 * 128;
            A1(&f, (size_t)(s->tc_rt + 16) * s->tc_vk); s->tc_vx = reinterpret_cast<uint8_t*>(f);
            A1(&f, ddp * s->tc_vk); s->tc_vw = reinterpret_cast<uint8_t*>(f);
            if (rc == SAT_OK) {
                cudaMemset(s->tc_vx, 0, (size_t)(s->tc_rt + 16) * s->tc_vk * 4);
                cudaMemset(s->tc_vw, 0, ddp * s->tc_vk * 4);
            }
        }
        // stacked weight gradients: T*B rows must fill whole K blocks
        const size_t TB = (size_t)T * B;
        s->tc_stack = (TB % 64 == 0);
        for (int i = 0; i < 4 && s->tc_stack; ++i) s->tc_stack = s->tcl[i].fwd && (i == 3 || s->tcl[i].dx);
        if (s->tc_stack) {
            AT(s->dys[0], B * A); AT(s->dys[1], B * 4 * H); AT(s->dys[2], B * Dd);
            size_t xmax = 0, wmax = 0;
            for (int i = 0; i < 4; ++i) {
                const size_t kp = (Ks[i] + 127) / 128 * 128, np = (Ns[i] + 127) / 128 * 128;
                xmax = TB * kp > xmax ? TB * kp : xmax;
                wmax = TB * np > wmax ? TB * np : wmax;
            }
            s->dec_all = dec2 && s->tc_vk > 0;
            s->all_rt = TB >= 128 ? 128 : (int)TB;
            s->all_rows = (int)((TB + s->all_rt - 1) / s->all_rt * s->all_rt);
            if (s->dec_all)   // packed rows of expanded / td / d td, all T steps
                for (int i = 2; i < 4; ++i) {
                    const size_t kp = (Ks[i] + 127) / 128 * 128;
                    xmax = (size_t)s->all_rows * kp > xmax ? (size_t)s->all_rows * kp : xmax;
                }
            A1(&f, xmax); s->tc_sx = reinterpret_cast<uint8_t*>(f);
            A1(&f, wmax); s->tc_sw = reinterpret_cast<uint8_t*>(f);
            if (s->dec_all) {
                A1(&s->logits_all, TB * V);
                A1(&s->dexp_all, TB * XDs);
                A1(&f, (size_t)(s->all_rows + 16) * s->tc_vk); s->tc_vx_all = reinterpret_cast<uint8_t*>(f);
                if (rc == SAT_OK) cudaMemset(s->tc_vx_all, 0, (size_t)(s->all_rows + 16) * s->tc_vk * 4);
            }
        }
    }
    float* cells = nullptr;
    A1(&cells, 8);
    if (rc == SAT_OK) {
        s->seed_d = reinterpret_cast<unsigned long long*>(cells);
        s->inv_msum_d = cells + 2;
    }
    if (rc != SAT_OK) { train_free(s); return rc; }
    *slot = s;
    sat_handle_set_train_free(h, train_free);
    return SAT_OK;
}

extern "C" int sat_train_init(sat_handle* h, int32_t B, int32_t T, float fc_drop_rate, float lstm_drop_rate,
                              float attention_loss_factor, float fc_kernel_regularizer_scale) {
    return sat_train_init_grouped(h, B, 1, T, fc_drop_rate, lstm_drop_rate, attention_loss_factor, fc_kernel_regularizer_scale);
}

int sat_train_info(sat_handle* h, const char* key, int64_t* value, int* rc) {
    if (strcmp(key, "train_bad_ids") != 0) return 0;
    TrainState* s = (TrainState*)*sat_handle_train_slot(h);
    *value = 0;
    *rc = SAT_OK;
    if (!s) return 1;
    float v = 0.f;
    cudaError_t e = cudaMemcpy(&v, s->loss_acc + 5, sizeof(float), cudaMemcpyDeviceToHost);   // (synchronises)
    if (e != cudaSuccess) { *rc = sat_fail(SAT_ERR_CUDA, "train_bad_ids: %s", cudaGetErrorString(e)); return 1; }
    *value = (int64_t)v;
    return 1;
}

extern "C" int sat_train_var(sat_handle* h, int32_t i, const char** name, int64_t* offset, int64_t* rows, int64_t* cols,
                             int32_t* regularised, int64_t* total) {
    if (!h) return sat_fail(SAT_ERR_INVALID, "null handle");
    TrainState tmp;
    TrainState* s = (TrainState*)*sat_handle_train_slot(h);
    if (!s) { tmp.d = *sat_handle_dims(h); fill_layout(&tmp); s = &tmp; }
    if (total) *total = (int64_t)s->off[kNumVars];
    if (i < 0 || i >= s->num_present) return i == -1 ? SAT_OK : sat_fail(SAT_ERR_INVALID, "variable index %d", i);
    i = s->present[i];
    if (name) *name = s->names[i];
    if (offset) *offset = (int64_t)s->off[i];
    if (rows) *rows = s->rows[i];
    if (cols) *cols = s->cols[i];
    if (regularised) *regularised = s->regularised[i] ? 1 : 0;
    return SAT_OK;
}

// y = act(dropout?(x) W + b)
static int dense_fwd(cudaStream_t st, const float* x, int rows, int K, const float* W, const float* b, int N, float* y, int act) {
    TCK(sgemm(st, false, false, rows, N, K, x, K, W, N, y, N, false));
    if (b || act) launch_k(bias_act_kernel, GRID1D((size_t)rows * N), 256, st, y, b, rows, N, act);
    return SAT_OK;
}
// given dy (w.r.t. pre-activation): dW += x^T dy, db += colsum(dy), dx = dy W^T (if dx)
static int dense_bwd(cudaStream_t st, const float* x, int rows, int K, const float* W, int N, const float* dy, float* dW,
                     float* db, float* dx) {
    TCK(sgemm(st, true, false, K, N, rows, x, K, dy, N, dW, N, true));
    if (db) launch_k(colsum_kernel, dim3((N + 127) / 128, (rows + 255) / 256), 128, st, db, dy, rows, N, nullptr);
    if (dx) TCK(sgemm(st, false, true, rows, K, N, dy, N, W, N, dx, K, false));
    return SAT_OK;
}

static int train_enqueue(TrainState* s, const float* params, float* grads, const float* contexts,
                         const int32_t* sentences, const float* masks, const float* row_w, int32_t B, int32_t T,
                         int32_t global_batch, float* losses, cudaStream_t st) {
    const sat_dims& d = s->d;
    const int L = d.num_ctx, D = d.dim_ctx, E = d.dim_embedding, H = d.num_lstm_units, A = d.dim_attend_layer,
              Dd = d.dim_decode_layer, I = d.dim_initalize_layer, V = d.vocabulary_size;
    const int BL = B * L, XL = D + E + H, XD = H + D + E;
    // image-level rows: NI images of G batch rows each (G == 1: NI == B, and every launch below is the ungrouped one)
    const int G = s->group, NI = s->n_img, BLi = NI * L;
    const float kf = s->keep_fc, kl = s->keep_lstm;   // 1 - fc_drop_rate, 1 - lstm_drop_rate (config.py:25-26)
    auto P = [&](int v) { return params + s->off[v]; };
    auto Gd = [&](int v) { return grads + s->off[v]; };
    auto ST = [&](int t, int k) { return (unsigned long long)(t * 16 + k); };
    const unsigned long long INIT = 0xFFFF0ull;
    const unsigned long long* seed = s->seed_d;
    const float* inv_msum = s->inv_msum_d;
    const float inv_gbl = 1.0f / ((float)global_batch * (float)L);

    TCK(cudaMemsetAsync(grads, 0, s->off[kNumVars] * sizeof(float), st));
    TCK(cudaMemsetAsync(s->loss_acc, 0, 8 * sizeof(float), st));
    TCK(cudaMemsetAsync(s->att, 0, (size_t)BL * sizeof(float), st));

    // ------------------------------------------------------------ initialize (model.py:239-242, 358-393)
    // (per image; the init_* masks are drawn for NI rows)
    float* const c0i = G > 1 ? s->c0i : s->c0;
    float* const h0i = G > 1 ? s->h0i : s->h0;
    launch_k(mean_L_kernel, dim3((D + 127) / 128, NI), 128, st, s->mean, contexts, L, D);
    launch_k(dropout2d_kernel, GRID1D((size_t)NI * D), 256, st, s->meand, D, s->mean, D, NI, D, seed, INIT + 0, kf, 0);
    const bool init2 = d.num_initalize_layers == 2, att2 = d.num_attend_layers == 2, dec2 = d.num_decode_layers == 2;
    if (init2) {
        TRET(dense_fwd(st, s->meand, NI, D, P(vIa1W), P(vIa1B), I, s->ia1, 1));
        launch_k(dropout2d_kernel, GRID1D((size_t)NI * I), 256, st, s->ia1d, I, s->ia1, I, NI, I, seed, INIT + 1, kf, 0);
        TRET(dense_fwd(st, s->ia1d, NI, I, P(vIa2W), P(vIa2B), H, c0i, 0));
        TRET(dense_fwd(st, s->meand, NI, D, P(vIb1W), P(vIb1B), I, s->ib1, 1));
        launch_k(dropout2d_kernel, GRID1D((size_t)NI * I), 256, st, s->ib1d, I, s->ib1, I, NI, I, seed, INIT + 2, kf, 0);
        TRET(dense_fwd(st, s->ib1d, NI, I, P(vIb2W), P(vIb2B), H, h0i, 0));
    } else {   // one layer each, no activation (model.py:362-371)
        TRET(dense_fwd(st, s->meand, NI, D, P(vIa1W), P(vIa1B), H, c0i, 0));
        TRET(dense_fwd(st, s->meand, NI, D, P(vIb1W), P(vIb1B), H, h0i, 0));
    }
    if (G > 1) {   // every caption of an image starts from the image's state
        launch_k(expand_rows_kernel, GRID1D((size_t)B * H), 256, st, s->c0, (const float*)c0i, B, H, G);
        launch_k(expand_rows_kernel, GRID1D((size_t)B * H), 256, st, s->h0, (const float*)h0i, B, H, G);
    }

    const bool tc = s->tc_ok && sat_handle_train_tc(s->handle);
    const int lmode = sat_handle_layout_mode(s->handle);
    if (tc) {   // this step's attend/fc_1a weights in the packed layout (they change with every optimizer step)
        TCK(sat::lin_repack_weight(P(vA1aW), D, A, 0, s->tc_w1a, lmode, st, nullptr, PDLK));
        TCK(sat::lin_repack_bias(P(vA1aB), A, 0, s->tc_b1a, st));
    }
    const bool tcb = sat_handle_train_tc(s->handle) != 0;
    if (tcb) {
        for (int i = 0; i < 4; ++i) {
            TrainState::TcLayer& l = s->tcl[i];
            if (l.fwd) {
                TCK(sat::lin_repack_weight(P(l.var_w), l.K, l.N, 0, l.w, lmode, st, nullptr, PDLK));
                TCK(sat::lin_repack_bias(P(l.var_b), l.N, 0, l.b, st));
            }
            if (l.dx) {   // W^T as a weight operand: row n of the operand = row k of W ... i.e. W's rows are its K-major rows
                sat::PackJob job{P(l.var_w), nullptr, l.N, l.N, l.K, 128, l.wT};
                TCK(sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK));
            }
        }
    }
    const bool tcv = tcb && dec2 && s->tc_vk > 0;
    if (tcv) {   // decode/fc_2's W^T (rows Dd, K = V rounded up) for its input gradient
        sat::PackJob job{P(vD2W), nullptr, V, V, Dd, 128, s->tc_vw, s->tc_vk / 64};
        TCK(sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK));
    }
    auto tc_splits = [&](int n_out, int K) {
        const int tiles = (n_out + 127) / 128;
        int sp = 1;
        while (sp * 2 <= 8 && tiles * sp * 2 <= sat::device_sm_count() && sp * 2 <= K / 64) sp *= 2;
        return sp;
    };
    // y[B, N] = epi(x[B, K] W + b) on the wgmma kernel; false if this layer / shape stays on the CUDA-core path
    auto tc_fwd = [&](int li, const float* x, int epi, float* y, int* rc) -> bool {
        TrainState::TcLayer& l = s->tcl[li];
        if (!tcb || !l.fwd) return false;
        sat::PackJob job{x, nullptr, l.K, l.K, B, s->tc_rt, s->tc_xs};
        cudaError_t ce = sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK);
        if (ce != cudaSuccess) { *rc = sat_fail(SAT_ERR_CUDA, "pack: %s", cudaGetErrorString(ce)); return true; }
        *rc = sat_dense_packed(s->handle, s->tc_xs, B, s->tc_rt, l.K, l.w, l.b, l.N, epi, y, l.N, 0, tc_splits(l.N, l.K), st);
        return true;
    };
    // dx[B, K] = dy[B, N] W^T
    auto tc_dx = [&](int li, const float* dy, float* dx, int* rc) -> bool {
        TrainState::TcLayer& l = s->tcl[li];
        if (!tcb || !l.dx) return false;
        sat::PackJob job{dy, nullptr, l.N, l.N, B, s->tc_rt, s->tc_xs};
        cudaError_t ce = sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK);
        if (ce != cudaSuccess) { *rc = sat_fail(SAT_ERR_CUDA, "pack: %s", cudaGetErrorString(ce)); return true; }
        *rc = sat_dense_packed(s->handle, s->tc_xs, B, s->tc_rt, l.N, l.wT, nullptr, l.K, sat::kEpiNone, dx, l.K, 0, tc_splits(l.K, l.N), st);
        return true;
    };
    // the same two products when the producer of x / dy has already written the packed operand into tc_xs
    static const int fuse_pack_env = []() { const char* e = getenv("SAT_TRAIN_FUSE_PACK"); return (e && e[0] == '0') ? 0 : 1; }();
    auto pk_fwd_ok = [&](int li) { return tcb && fuse_pack_env && s->tcl[li].fwd; };
    auto pk_dx_ok = [&](int li) { return tcb && fuse_pack_env && s->tcl[li].dx; };
    auto tc_fwd_packed = [&](int li, int epi, float* y) -> int {
        TrainState::TcLayer& l = s->tcl[li];
        return sat_dense_packed(s->handle, s->tc_xs, B, s->tc_rt, l.K, l.w, l.b, l.N, epi, y, l.N, 0, tc_splits(l.N, l.K), st);
    };
    auto tc_dx_packed = [&](int li, float* dx) -> int {
        TrainState::TcLayer& l = s->tcl[li];
        return sat_dense_packed(s->handle, s->tc_xs, B, s->tc_rt, l.N, l.wT, nullptr, l.K, sat::kEpiNone, dx, l.K, 0, tc_splits(l.K, l.N), st);
    };
    int trc = SAT_OK;
    // second stream for the fc_1a products (SAT_TRAIN_SIDE=0: everything in order on the caller's stream)
    // (2 / 3: only the forward / only the backward products)
    static const int side_env = []() { const char* e = getenv("SAT_TRAIN_SIDE"); return e ? atoi(e) : 1; }();
    auto hand = [&](cudaStream_t from, cudaStream_t to, cudaEvent_t e) -> cudaError_t {   // `to` continues after `from`'s work so far
        cudaError_t ce = cudaEventRecord(e, from);
        return ce != cudaSuccess ? ce : cudaStreamWaitEvent(to, e, 0);
    };
    auto evT1 = [&](int t) { return s->ev[2 + 3 * t]; };
    auto evAb = [&](int t) { return s->ev[3 + 3 * t]; };
    auto evRp = [&](int t) { return s->ev[4 + 3 * t]; };
    // SAT_TRAIN_FUSE_SOFTMAX: 0 = separate softmax kernels, 2 = only the forward one folded in, 1 / unset = both directions
    static const int fuse_env = []() { const char* e = getenv("SAT_TRAIN_FUSE_SOFTMAX"); return e ? atoi(e) : 1; }();
    const bool fuse_sm = fuse_env != 0;
    const bool stack = tcb && s->tc_stack;   // weight gradients of the four batch-row layers after the time loop
    static const int dec_all_env = []() { const char* e = getenv("SAT_TRAIN_DEC_ALL"); return (e && e[0] == '0') ? 0 : 1; }();
    const bool dec_all = stack && tcv && s->dec_all && dec_all_env;   // decode layers of all T steps as [T*B]-row products
    const int TBr = T * B;
    auto all_splits = [&](int n_out, int K) {
        const int tiles = ((n_out + 127) / 128) * (s->all_rows / (s->all_rt > 0 ? s->all_rt : 1));
        int sp = 1;
        while (sp * 2 <= 8 && tiles * sp * 2 <= sat::device_sm_count() && sp * 2 <= K / 64) sp *= 2;
        return sp;
    };
    // scorer: fused one-pass kernels when the rows are float4-addressable (every buffer involved is a cudaMalloc'd
    // [rows, A] matrix or an A-vector, so A % 4 == 0 gives 16-byte alignment)
    const bool att_fused = att2 && (A & 3) == 0 && ((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads)) & 15) == 0;
    const bool side_any = tc && att_fused && s->side && side_env;
    const bool side_f = side_any && side_env != 3, side_b = side_any && side_env != 2;
    cudaStream_t sd = side_f ? s->side : st;
    int ab_chunks = 1, ab_rows = L, ab_wave = 0;
    {
        const int gx = (A / 4 + kAbCT - 1) / kAbCT;
        // about four CTAs per SM (grouped: one CTA covers the rows of an image)
        ab_chunks = (sat::device_sm_count() * 4 + NI * gx - 1) / (NI * gx > 0 ? NI * gx : 1);
        if (ab_chunks > (L + 15) / 16) ab_chunks = (L + 15) / 16;
        if (ab_chunks < 1) ab_chunks = 1;
        // SAT_TRAIN_ATTBWD_WAVE=1 (experiment, off by default): the 64-register build of the kernel and as many row
        // chunks as fit ONE resident wave, which trades registers per thread for the absence of a partly filled tail wave
        static const int one_wave = []() { const char* e = getenv("SAT_TRAIN_ATTBWD_WAVE"); return (e && e[0] == '1') ? 1 : 0; }();
        ab_wave = one_wave;
        if (one_wave) {
            int occ = 0, sms = sat::device_sm_count(), dev = 0;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, att_bwd_fused_wave_kernel, kAbRG * kAbCT, 0) != cudaSuccess || occ < 1) occ = 1;
            ab_chunks = (occ * sms) / (NI * gx > 0 ? NI * gx : 1);
            if (ab_chunks > (L + 7) / 8) ab_chunks = (L + 7) / 8;
            if (ab_chunks < 1) ab_chunks = 1;
        }
        ab_rows = (L + ab_chunks - 1) / ab_chunks;
        ab_chunks = (L + ab_rows - 1) / ab_rows;
    }
    // attend/fc_1a runs on the NI * L image-level rows: the att_ctx mask of step t is drawn for those rows
    if (side_f) {   // T1[t] = tanh(drop_t(ctx) W1a + b1a) for every step, queued ahead on the second stream
        TCK(hand(st, sd, s->ev[0]));
        for (int t = 0; t < T; ++t) {
            sat::PackJob job{contexts, nullptr, D, D, BLi, 128, s->tc_xpa};
            const sat::DropSpec drop{seed, ST(t, 0), kf};
            TCK(sat::pack_rows_launch(&job, 1, lmode, sd, &drop, PDLK));
            TRET(sat_dense_packed(s->handle, s->tc_xpa, BLi, 128, D, s->tc_w1a, s->tc_b1a, A, sat::kEpiBiasTanh, s->T1[t], A, 0, 1, sd));
            TCK(cudaEventRecord(evT1(t), sd));
        }
    }
    // the non-fused scorer reads T1 per batch row: grouped, the image blocks of step t are first copied to the rows
    // (into temp, which att_temp_kernel then updates in place)
    auto att_t1_rows = [&](int t) -> const float* {
        if (G == 1) return s->T1[t];
        launch_k(expand_rows_kernel, GRID1D((size_t)BL * A), 256, st, s->temp, (const float*)s->T1[t], B, L * A, G);
        return s->temp;
    };
    auto launch_ce = [&](int blocks, const float* logits, float* dlogits, int t, int rows_per_step) {
        if (row_w)
            launch_k(ce_kernel<true>, blocks, kCeThreads, st, logits, dlogits, sentences, T, t, masks, V, inv_msum, s->loss_acc, rows_per_step, row_w);
        else
            launch_k(ce_kernel<false>, blocks, kCeThreads, st, logits, dlogits, sentences, T, t, masks, V, inv_msum, s->loss_acc, rows_per_step,
                     (const float*)nullptr);
    };
    // ------------------------------------------------------------ forward through time (model.py:258-312)
    for (int t = 0; t < T; ++t) {
        const float* h_out_prev = t ? s->h_out[t - 1] : s->h0;
        const float* h_state_prev = t ? s->h_state[t - 1] : s->h0;
        const float* c_prev = t ? s->c[t - 1] : s->c0;
        // attend (model.py:395-436)
        if (!att2) {   // one layer: e = drop(ctx) wa [BL] + drop(h) Wb [B, L]  (the first term per image)
            launch_k(dropout2d_kernel, GRID1D((size_t)BLi * D), 256, st, s->ctxd, D, contexts, D, BLi, D, seed, ST(t, 0), kf, 0);
            launch_k(rowdot_kernel, (BLi * 32 + 255) / 256, 256, st, G > 1 ? s->e_img : s->e, s->ctxd, P(vA1aW), BLi, D);
            if (G > 1) launch_k(expand_rows_kernel, GRID1D((size_t)BL), 256, st, s->e, (const float*)s->e_img, B, L, G);
        } else if (side_f) {
        } else if (tc) {   // T1 = tanh(drop(ctx) W1a + b1a) on the wgmma dense kernel: the context dropout is applied while the
                    // rows are packed (no fp32 dropped copy), bias + tanh fused in the epilogue
            sat::PackJob job{contexts, nullptr, D, D, BLi, 128, s->tc_xpa};
            const sat::DropSpec drop{seed, ST(t, 0), kf};
            TCK(sat::pack_rows_launch(&job, 1, lmode, st, &drop, PDLK));
            TRET(sat_dense_packed(s->handle, s->tc_xpa, BLi, 128, D, s->tc_w1a, s->tc_b1a, A, sat::kEpiBiasTanh, s->T1[t], A, 0, 1, st));
        } else {
            launch_k(dropout2d_kernel, GRID1D((size_t)BLi * D), 256, st, s->ctxd, D, contexts, D, BLi, D, seed, ST(t, 0), kf, 0);
            TRET(dense_fwd(st, s->ctxd, BLi, D, P(vA1aW), P(vA1aB), A, s->T1[t], 1));
        }
        const bool hd_packed = att2 && pk_fwd_ok(0);
        if (hd_packed)
            launch_k(dropout_pack_kernel, GRID1D((size_t)B * H), 256, st, s->hd[t], h_out_prev, B, H, seed, ST(t, 1), kf, s->tc_xs, lmode, s->tc_rt);
        else
            launch_k(dropout2d_kernel, GRID1D((size_t)B * H), 256, st, s->hd[t], H, h_out_prev, H, B, H, seed, ST(t, 1), kf, 0);
        if (!att2) {
            TRET(dense_fwd(st, s->hd[t], B, H, P(vA1bW), nullptr, L, s->dalpha, 0));   // (dalpha: backward scratch, free here)
            launch_k(copy2d_kernel, GRID1D((size_t)BL), 256, st, s->e, L, s->dalpha, L, B, L, 1);
        } else if (hd_packed) { TRET(tc_fwd_packed(0, sat::kEpiBiasTanh, s->q[t]));
        } else if (tc_fwd(0, s->hd[t], sat::kEpiBiasTanh, s->q[t], &trc)) { TRET(trc); }
        else TRET(dense_fwd(st, s->hd[t], B, H, P(vA1bW), P(vA1bB), A, s->q[t], 1));
        if (side_f) TCK(cudaStreamWaitEvent(st, evT1(t), 0));
        if (!att2) {   // (the 1-layer scores are complete: e = drop(ctx) wa + drop(h) Wb above)
        } else if (att_fused) {
            launch_k(att_logits_kernel, (BL * 32 + 255) / 256, 256, st, s->e, s->T1[t], s->q[t], P(vA2W), B, L, A, seed, ST(t, 2), kf, G);
        } else {
            launch_k(att_temp_kernel, GRID1D((size_t)BL * A), 256, st, s->temp, att_t1_rows(t), s->q[t], B, L, A, seed, ST(t, 2), kf);
            launch_k(rowdot_kernel, (BL * 32 + 255) / 256, 256, st, s->e, s->temp, P(vA2W), BL, A);
        }
        const bool ctx4 = (D & 3) == 0 && (reinterpret_cast<uintptr_t>(contexts) & 15) == 0;
        if (ctx4 && L <= kSmL && fuse_sm) {   // softmax + coverage + context vector in one launch
            launch_k(softmax_context_fwd4_kernel, dim3((D / 4 + 31) / 32, B), 256, st, s->z[t], s->alpha[t], s->e, contexts, L, D, s->att, masks, T, t, G);
        } else {
            launch_k(softmax_rows_kernel, (B * 32 + 255) / 256, 256, st, s->alpha[t], s->e, B, L, s->att, masks, T, t);   // + coverage
            if (ctx4)   // un-dropped ctx
                launch_k(context_fwd4_kernel, dim3((D / 4 + 31) / 32, B), 256, st, s->z[t], s->alpha[t], contexts, L, D, G);
            else
                launch_k(context_fwd_kernel, dim3((D + 127) / 128, B), 128, st, s->z[t], s->alpha[t], contexts, B, L, D, G);
        }
        // embedding of the previous word: 0 at t = 0, then teacher forcing (model.py:254, 310)
        if (t == 0)   // every step's rows at once (teacher forcing: the words are inputs)
            launch_k(gather_rows_kernel, GRID1D((size_t)T * B * E), 256, st, s->emb[0], E, P(vEmb), E, sentences, T, T * B, V,
                     s->loss_acc + 5, B);
        // LSTM with DropoutWrapper (model.py:228-236, 276-279)
        // lstm_in = [ drop_in(concat(z, emb)) | h_state_prev ]
        launch_k(concat3_drop_kernel, GRID1D((size_t)B * XL), 256, st, s->lstm_in[t], XL, s->z[t], D, s->emb[t], E, h_state_prev, H, D + E, B,
                                                                    seed, ST(t, 3), kl, 0, pk_fwd_ok(1) ? s->tc_xs : nullptr, lmode, s->tc_rt);
        if (pk_fwd_ok(1)) { TRET(tc_fwd_packed(1, sat::kEpiNone, s->acts[t])); }
        else if (tc_fwd(1, s->lstm_in[t], sat::kEpiNone, s->acts[t], &trc)) { TRET(trc); }   // (bias and gates: next kernel)
        else TCK(sgemm(st, false, false, B, 4 * H, XL, s->lstm_in[t], XL, P(vLW), 4 * H, s->acts[t], 4 * H, false));
        launch_k(lstm_fwd_kernel, GRID1D((size_t)B * H), 256, st, s->acts[t], P(vLB), c_prev, s->c[t], s->h_out[t], s->h_state[t], B, H, seed,
                 ST(t, 5), ST(t, 4), kl);
        // decode (model.py:282-287, 438-459)
        if (dec_all) continue;   // (the decode layers of every step follow the loop)
        launch_k(concat3_drop_kernel, GRID1D((size_t)B * XD), 256, st, s->expd[t], XD, s->h_out[t], H, s->z[t], D, s->emb[t], E, XD, B,
                                                                    seed, ST(t, 6), kf, 0, (uint8_t*)nullptr, 0, 0);
        if (!dec2) {
            TRET(dense_fwd(st, s->expd[t], B, XD, P(vD1W), P(vD1B), V, s->logits, 0));
        } else {
            if (tc_fwd(2, s->expd[t], sat::kEpiBiasTanh, s->t1[t], &trc)) { TRET(trc); }
            else TRET(dense_fwd(st, s->expd[t], B, XD, P(vD1W), P(vD1B), Dd, s->t1[t], 1));
            launch_k(dropout2d_kernel, GRID1D((size_t)B * Dd), 256, st, s->td[t], Dd, s->t1[t], Dd, B, Dd, seed, ST(t, 7), kf, 0);
            if (tc_fwd(3, s->td[t], sat::kEpiBias, s->logits, &trc)) { TRET(trc); }
            else TRET(dense_fwd(st, s->td[t], B, Dd, P(vD2W), P(vD2B), V, s->logits, 0));
        }
        // masked cross entropy + accuracy, and d loss / d logits (model.py:292-305, 316-318, 332-334)
        launch_ce(B, s->logits, s->dlogits[t], t, 0);
    }
    if (dec_all) {   // decode of all T steps (model.py:282-305): the per-step stashes are contiguous = [T*B, .] matrices
        launch_k(concat3_drop_kernel, GRID1D((size_t)TBr * XD), 256, st, s->expd[0], XD, s->h_out[0], H, s->z[0], D, s->emb[0], E, XD, TBr,
                                                                      seed, ST(0, 6), kf, B, (uint8_t*)nullptr, 0, 0);
        {
            sat::PackJob job{s->expd[0], nullptr, XD, XD, TBr, s->all_rt, s->tc_sx};
            TCK(sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK));
            TRET(sat_dense_packed(s->handle, s->tc_sx, TBr, s->all_rt, XD, s->tcl[2].w, s->tcl[2].b, Dd, sat::kEpiBiasTanh, s->t1[0], Dd, 0,
                                  all_splits(Dd, XD), st));
        }
        launch_k(dropout_steps_kernel, GRID1D((size_t)TBr * Dd), 256, st, s->td[0], s->t1[0], (size_t)TBr * Dd, (size_t)B * Dd, seed, ST(0, 7), kf);
        {
            sat::PackJob job{s->td[0], nullptr, Dd, Dd, TBr, s->all_rt, s->tc_sx};
            TCK(sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK));
            TRET(sat_dense_packed(s->handle, s->tc_sx, TBr, s->all_rt, Dd, s->tcl[3].w, s->tcl[3].b, V, sat::kEpiBias, s->logits_all, V, 0,
                                  all_splits(V, Dd), st));
        }
        launch_ce(TBr, s->logits_all, s->dlogits[0], 0, B);
    }
    // attention coverage loss (model.py:320-326) and L2 regulariser (model.py:328)
    launch_k(coverage_loss_kernel, 64, 256, st, s->datt, s->att, BL, s->att_factor, inv_gbl, s->loss_acc);
    for (int v = 0; v < kNumVars; ++v)
        if (s->regularised[v]) {
            const size_t n = (size_t)s->rows[v] * s->cols[v];
            const int g = (int)((n / 4 + 1023) / 1024);   // about four float4 per thread
            launch_k(sumsq_kernel, g < 1 ? 1 : (g > sat::device_sm_count() * 8 ? sat::device_sm_count() * 8 : g), 256, st, P(v), n, 0.5f * s->reg_scale, s->loss_acc + 3);
        }

    // ------------------------------------------------------------ backward through time
    TCK(cudaMemsetAsync(s->dh_out, 0, (size_t)B * H * sizeof(float), st));    // d loss / d h_out[t] from step t+1's attend
    TCK(cudaMemsetAsync(s->dh_state, 0, (size_t)B * H * sizeof(float), st));  // d loss / d h_state[t] from step t+1's LSTM
    TCK(cudaMemsetAsync(s->dc, 0, (size_t)B * H * sizeof(float), st));
    sd = side_b ? s->side : st;
    if (side_b && !side_f) TCK(hand(st, sd, s->ev[0]));   // (the second stream joins the step here)
    if (stack && att_fused) TCK(cudaMemsetAsync(s->dys[0][0], 0, (size_t)T * B * A * sizeof(float), st));   // d q of every step
    if (dec_all) {   // d logits -> d td (x tanh', dropout) -> d expanded, for all T steps
        sat::PackJob job{s->dlogits[0], nullptr, V, V, TBr, s->all_rt, s->tc_vx_all, s->tc_vk / 64};
        TCK(sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK));
        TRET(sat_dense_packed(s->handle, s->tc_vx_all, TBr, s->all_rt, s->tc_vk, s->tc_vw, nullptr, Dd, sat::kEpiNone, s->dys[2][0], Dd, 0,
                              all_splits(Dd, s->tc_vk), st));
        launch_k(drop_tanh_bwd_kernel, GRID1D((size_t)TBr * Dd), 256, st, s->dys[2][0], s->t1[0], (size_t)TBr * Dd, seed, ST(0, 7), kf,
                 (size_t)B * Dd);
        sat::PackJob job2{s->dys[2][0], nullptr, Dd, Dd, TBr, s->all_rt, s->tc_sx};
        TCK(sat::pack_rows_launch(&job2, 1, lmode, st, nullptr, PDLK));
        TRET(sat_dense_packed(s->handle, s->tc_sx, TBr, s->all_rt, Dd, s->tcl[2].wT, nullptr, XD, sat::kEpiNone, s->dexp_all, XD, 0,
                              all_splits(XD, Dd), st));
    }
    for (int t = T - 1; t >= 0; --t) {
        const float* h_state_prev = t ? s->h_state[t - 1] : s->h0;
        const float* c_prev = t ? s->c[t - 1] : s->c0;
        (void)h_state_prev;
        // decode fc_2, fc_1
        float* dtd = stack ? s->dys[2][t] : s->dtd;
        float* dG = stack ? s->dys[1][t] : s->dG;
        float* dq = stack ? s->dys[0][t] : s->dq;
        bool vdx = false;
        const float* dexp = dec_all ? s->dexp_all + (size_t)t * B * XD : s->dexp;
        float* const demb = s->demb_all + (size_t)t * B * E;
        if (dec_all) {
        } else if (!dec2) {
            TRET(dense_bwd(st, s->expd[t], B, XD, P(vD1W), V, s->dlogits[t], Gd(vD1W), Gd(vD1B), s->dexp));
        } else {
            if (tcv) {   // dtd = dlogits W2^T on the tensor cores (ragged K = V: zero-padded last K block)
                sat::PackJob job{s->dlogits[t], nullptr, V, V, B, s->tc_rt, s->tc_vx, s->tc_vk / 64};
                TCK(sat::pack_rows_launch(&job, 1, lmode, st, nullptr, PDLK));
                TRET(sat_dense_packed(s->handle, s->tc_vx, B, s->tc_rt, s->tc_vk, s->tc_vw, nullptr, Dd, sat::kEpiNone, dtd, Dd, 0,
                                      tc_splits(Dd, s->tc_vk), st));
                vdx = true;
            }
            if (stack) { if (!vdx) TCK(sgemm(st, false, true, B, Dd, V, s->dlogits[t], V, P(vD2W), V, dtd, Dd, false)); }
            else if (vdx) TRET(dense_bwd(st, s->td[t], B, Dd, P(vD2W), V, s->dlogits[t], Gd(vD2W), Gd(vD2B), nullptr));
            else TRET(dense_bwd(st, s->td[t], B, Dd, P(vD2W), V, s->dlogits[t], Gd(vD2W), Gd(vD2B), dtd));
            launch_k(drop_tanh_bwd_kernel, GRID1D((size_t)B * Dd), 256, st, dtd, s->t1[t], (size_t)B * Dd, seed, ST(t, 7), kf, (size_t)0);
            if (tc_dx(2, dtd, s->dexp, &trc)) { TRET(trc); if (!stack) TRET(dense_bwd(st, s->expd[t], B, XD, P(vD1W), Dd, dtd, Gd(vD1W), Gd(vD1B), nullptr)); }
            else TRET(dense_bwd(st, s->expd[t], B, XD, P(vD1W), Dd, dtd, Gd(vD1W), Gd(vD1B), s->dexp));
        }
        // drop(dexp) = [dh_out (+=) | dz (=) | demb (=)]
        launch_k(split3_drop_kernel, GRID1D((size_t)B * XD), 256, st, dexp, XD, B, s->dh_out, H, 1, s->dz, D, 0, demb, E, 0, XD, seed,
                                                                   ST(t, 6), kf);
        // h_out = drop_out(h_raw), h_state = drop_state(h_raw)
        launch_k(lstm_bwd_kernel, GRID1D((size_t)B * H), 256, st, dG, s->dc, s->dh_out, s->dh_state, s->acts[t], s->c[t], c_prev, B, H, seed,
                 ST(t, 5), ST(t, 4), kl, pk_dx_ok(1) ? s->tc_xs : (uint8_t*)nullptr, lmode, s->tc_rt);
        if (pk_dx_ok(1)) {
            TRET(tc_dx_packed(1, s->dlin));
            if (!stack) TRET(dense_bwd(st, s->lstm_in[t], B, XL, P(vLW), 4 * H, dG, Gd(vLW), Gd(vLB), nullptr));
        } else if (tc_dx(1, dG, s->dlin, &trc)) { TRET(trc); if (!stack) TRET(dense_bwd(st, s->lstm_in[t], B, XL, P(vLW), 4 * H, dG, Gd(vLW), Gd(vLB), nullptr)); }
        else TRET(dense_bwd(st, s->lstm_in[t], B, XL, P(vLW), 4 * H, dG, Gd(vLW), Gd(vLB), s->dlin));
        // dlin = [d xd (D+E) | dh_state_prev]
        launch_k(split3_drop_kernel, GRID1D((size_t)B * XL), 256, st, s->dlin, XL, B, s->dz, D, 1, demb, E, 1, s->dh_state, H, 0, D + E, seed,
                                                                   ST(t, 3), kl);
        // attention: context vector, softmax, scorer
        launch_k(context_bwd_kernel, (BL * 32 + 255) / 256, 256, st, s->dalpha, s->dz, contexts, s->datt, B, L, D, masks, T, t, G);
        const bool sm_in_ab = att2 && att_fused && fuse_env == 1;   // (the fused scorer backward takes the softmax backward itself)
        if (!sm_in_ab) launch_k(softmax_bwd_kernel, (B * 32 + 255) / 256, 256, st, s->dalpha, s->alpha[t], B, L);   // dalpha now holds de
        if (!att2) {   // de = dalpha [B, L]: dwa += drop(ctx)^T de, dWb += drop(h)^T de, d drop(h) = de Wb^T
            launch_k(dropout2d_kernel, GRID1D((size_t)BLi * D), 256, st, s->ctxd, D, contexts, D, BLi, D, seed, ST(t, 0), kf, 0);
            if (G > 1) launch_k(group_sum_kernel, GRID1D((size_t)BLi), 256, st, s->e_img, (const float*)s->dalpha, NI, L, G);   // de per image
            launch_k(colsum_kernel, dim3((D + 127) / 128, (BLi + 255) / 256), 128, st, Gd(vA1aW), s->ctxd, BLi, D,
                     G > 1 ? s->e_img : s->dalpha);
            TRET(dense_bwd(st, s->hd[t], B, H, P(vA1bW), L, s->dalpha, Gd(vA1bW), nullptr, s->dhd));
        } else {
            float* const dtemp = (side_b && (t & 1)) ? s->dtemp2 : s->dtemp;
            float* dtemp_w = dtemp;   // d temp of the NI * L image-level rows: the fc_1a weight gradient's operand
            if (att_fused) {   // temp, dw2, dtemp, dq, tanh' and (tensor-core path) db1a in one pass over T1
                if (!stack) TCK(cudaMemsetAsync(dq, 0, (size_t)B * A * sizeof(float), st));   // (stacked: zeroed once before the loop)
                if (side_b && t + 2 < T) TCK(cudaStreamWaitEvent(st, evRp(t + 2), 0));   // this d temp buffer has been packed
                if (G == 1)
                    launch_k(ab_wave ? att_bwd_fused_wave_kernel : att_bwd_fused_kernel, dim3((A / 4 + kAbCT - 1) / kAbCT, ab_chunks, B),
                             kAbRG * kAbCT, st, dtemp, dq, Gd(vA2W), tc ? Gd(vA1aB) : nullptr, s->T1[t], s->q[t], s->dalpha, P(vA2W), L, A,
                             ab_rows, seed, ST(t, 2), kf, sm_in_ab ? s->alpha[t] : nullptr);
                else   // one pass over each image's T1 block for all of its rows; d temp summed over the group
                    launch_k(att_bwd_grouped_kernel, dim3((A / 4 + kAbCT - 1) / kAbCT, ab_chunks, NI), kAbRG * kAbCT, st, dtemp, dq, Gd(vA2W),
                             tc ? Gd(vA1aB) : nullptr, s->T1[t], s->q[t], s->dalpha, P(vA2W), L, A, ab_rows, G, seed, ST(t, 2), kf,
                             sm_in_ab ? s->alpha[t] : nullptr);
            } else {
                launch_k(att_temp_kernel, GRID1D((size_t)BL * A), 256, st, s->temp, att_t1_rows(t), s->q[t], B, L, A, seed, ST(t, 2), kf);
                launch_k(colsum_kernel, dim3((A + 127) / 128, (BL + 255) / 256), 128, st, Gd(vA2W), s->temp, BL, A, s->dalpha);   // dw2 += temp^T de
                launch_k(att_dtemp_kernel, GRID1D((size_t)BL * A), 256, st, s->dtemp, s->dalpha, P(vA2W), BL, A, seed, ST(t, 2), kf);
                launch_k(segsum_kernel, dim3((A + 127) / 128, B), 128, st, dq, s->dtemp, B, L, A);
                if (G > 1) {   // sum over each image's rows, then tanh' of the image's T1
                    launch_k(group_sum_kernel, GRID1D((size_t)BLi * A), 256, st, s->dtemp_g, (const float*)s->dtemp, NI, L * A, G);
                    dtemp_w = s->dtemp_g;
                }
                launch_k(tanh_bwd_kernel, GRID1D((size_t)BLi * A), 256, st, dtemp_w, s->T1[t], (size_t)BLi * A);
            }
            if (tc) {
                // dW1a[D, A] += ctxd^T[D, BL] * dtemp[BL, A]: the weight repack kernel transposes, so ctxd [BL x D] read
                // as a "[K x n_out] weight" IS the packed activation ctxd^T (row tile 128), and dtemp [BL x A] is the
                // packed weight; split-K over an 8-CTA cluster, accumulated into the gradient in the epilogue
                // (the context dropout mask is re-applied while ctx is packed: mask index row * D + column, as in the forward pass)
                const sat::DropSpec drop{seed, ST(t, 0), kf};
                TCK(sat::lin_repack_weight(contexts, BLi, D, 0, s->tc_xpa, lmode, sd, &drop, PDLK));   // (needs nothing of this step)
                if (side_b) TCK(hand(st, sd, evAb(t)));
                TCK(sat::lin_repack_weight(dtemp_w, BLi, A, 0, s->tc_wbig, lmode, sd, nullptr, PDLK));
                if (side_b) TCK(cudaEventRecord(evRp(t), sd));
                TRET(sat_dense_packed(s->handle, s->tc_xpa, D, 128, BLi, s->tc_wbig, nullptr, A, sat::kEpiNone, Gd(vA1aW), A, 1, 8, sd, 1));
                if (!att_fused) launch_k(colsum_kernel, dim3((A + 127) / 128, (BLi + 255) / 256), 128, st, Gd(vA1aB), dtemp_w, BLi, A, nullptr);
            } else {
                launch_k(dropout2d_kernel, GRID1D((size_t)BLi * D), 256, st, s->ctxd, D, contexts, D, BLi, D, seed, ST(t, 0), kf, 0);
                TRET(dense_bwd(st, s->ctxd, BLi, D, P(vA1aW), A, dtemp_w, Gd(vA1aW), Gd(vA1aB), nullptr));       // contexts are inputs
            }
            if (pk_dx_ok(0)) {
                launch_k(tanh_bwd_pack_kernel, GRID1D((size_t)B * A), 256, st, dq, s->q[t], B, A, s->tc_xs, lmode, s->tc_rt);
                TRET(tc_dx_packed(0, s->dhd));
                if (!stack) TRET(dense_bwd(st, s->hd[t], B, H, P(vA1bW), A, dq, Gd(vA1bW), Gd(vA1bB), nullptr));
            } else {
                launch_k(tanh_bwd_kernel, GRID1D((size_t)B * A), 256, st, dq, s->q[t], (size_t)B * A);
                if (tc_dx(0, dq, s->dhd, &trc)) { TRET(trc); if (!stack) TRET(dense_bwd(st, s->hd[t], B, H, P(vA1bW), A, dq, Gd(vA1bW), Gd(vA1bB), nullptr)); }
                else TRET(dense_bwd(st, s->hd[t], B, H, P(vA1bW), A, dq, Gd(vA1bW), Gd(vA1bB), s->dhd));
            }
        }
        // attend consumed drop(h_out[t-1]): this becomes d h_out[t-1] (the decode part is added next iteration)
        launch_k(dropout2d_kernel, GRID1D((size_t)B * H), 256, st, s->dh_out, H, s->dhd, H, B, H, seed, ST(t, 1), kf, 0);
    }
    launch_k(scatter_add_rows_kernel, GRID1D((size_t)T * B * E), 256, st, Gd(vEmb), E, sentences, T, s->demb_all, E, T * B, V, B);
    if (side_b) TCK(hand(sd, st, s->ev[1]));   // join: every fc_1a weight-gradient product has been accumulated
    if (stack) {
        // dW += X_all^T dY_all, db += colsum(dY_all) for attend/fc_1b, lstm, decode/fc_1, decode/fc_2 (the repack kernel
        // transposes: X_all [T*B, K] read as a "[K' x n_out'] weight" is the packed operand X_all^T, row tile 128)
        const int TB = T * B;
        const float* xs[4] = {s->hd[0], s->lstm_in[0], s->expd[0], s->td[0]};
        const float* dy[4] = {s->dys[0][0], s->dys[1][0], s->dys[2][0], s->dlogits[0]};
        for (int i = 0; i < 4; ++i) {
            TrainState::TcLayer& l = s->tcl[i];
            TCK(sat::lin_repack_weight(xs[i], TB, l.K, 0, s->tc_sx, lmode, st, nullptr, PDLK));
            TCK(sat::lin_repack_weight(dy[i], TB, l.N, 0, s->tc_sw, lmode, st, nullptr, PDLK));
            int sp = 1;
            const int tiles = ((l.N + 127) / 128) * ((l.K + 127) / 128);
            while (sp * 2 <= 8 && tiles * sp * 2 <= sat::device_sm_count()) sp *= 2;
            TRET(sat_dense_packed(s->handle, s->tc_sx, l.K, 128, TB, s->tc_sw, nullptr, l.N, sat::kEpiNone, Gd(l.var_w), l.N, 1, sp, st, 1));
            launch_k(colsum_kernel, dim3((l.N + 127) / 128, (TB + 255) / 256), 128, st, Gd(l.var_b), dy[i], TB, l.N, nullptr);
        }
    }
    // ------------------------------------------------------------ initialize backward
    // h0 is both h_out[-1] (attend of step 0) and h_state[-1] (LSTM of step 0); c0 receives dc
    launch_k(copy2d_kernel, GRID1D((size_t)B * H), 256, st, s->dh_out, H, s->dh_state, H, B, H, 1);
    float* dh0 = s->dh_out;
    float* dc0 = s->dc;
    if (G > 1) {   // the image's state fed each of its rows: sum their gradients, then initialize backward per image
        launch_k(group_sum_kernel, GRID1D((size_t)NI * H), 256, st, s->dhi, (const float*)s->dh_out, NI, H, G);
        launch_k(group_sum_kernel, GRID1D((size_t)NI * H), 256, st, s->dci, (const float*)s->dc, NI, H, G);
        dh0 = s->dhi;
        dc0 = s->dci;
    }
    float* dmid = s->dbuf + (size_t)B * D;  // [NI, I]
    if (!init2) {
        TRET(dense_bwd(st, s->meand, NI, D, P(vIb1W), H, dh0, Gd(vIb1W), Gd(vIb1B), nullptr));
        TRET(dense_bwd(st, s->meand, NI, D, P(vIa1W), H, dc0, Gd(vIa1W), Gd(vIa1B), nullptr));
    } else {
        TRET(dense_bwd(st, s->ib1d, NI, I, P(vIb2W), H, dh0, Gd(vIb2W), Gd(vIb2B), dmid));
        launch_k(drop_tanh_bwd_kernel, GRID1D((size_t)NI * I), 256, st, dmid, s->ib1, (size_t)NI * I, seed, INIT + 2, kf, (size_t)0);
        TRET(dense_bwd(st, s->meand, NI, D, P(vIb1W), I, dmid, Gd(vIb1W), Gd(vIb1B), nullptr));
        TRET(dense_bwd(st, s->ia1d, NI, I, P(vIa2W), H, dc0, Gd(vIa2W), Gd(vIa2B), dmid));
        launch_k(drop_tanh_bwd_kernel, GRID1D((size_t)NI * I), 256, st, dmid, s->ia1, (size_t)NI * I, seed, INIT + 1, kf, (size_t)0);
        TRET(dense_bwd(st, s->meand, NI, D, P(vIa1W), I, dmid, Gd(vIa1W), Gd(vIa1B), nullptr));
    }
    TCK(cudaGetLastError());
    TCK(cudaMemcpyAsync(losses, s->loss_acc, 4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return SAT_OK;
}

namespace {
__global__ void reciprocal_kernel(float* out, const double* in) { *out = (float)(1.0 / *in); }

// masks[r, t] = 1 up to and including the first eos of row r (every t if there is none), 0 after it; *sum = their total
// (one CTA: a deterministic sum, and the rows x T of a sampling round are few)
__global__ void __launch_bounds__(256) caption_masks_kernel(const int32_t* __restrict__ tokens, int rows, int T, int eos,
                                                            float* __restrict__ masks, double* sum) {
    __shared__ double red[8];
    double s = 0.0;
    for (int r = threadIdx.x; r < rows; r += blockDim.x) {
        const int32_t* tk = tokens + (size_t)r * T;
        int end = T;   // number of words kept
        for (int t = 0; t < T; ++t)
            if (tk[t] == eos) { end = t + 1; break; }
        float* m = masks + (size_t)r * T;
        for (int t = 0; t < T; ++t) m[t] = t < end ? 1.f : 0.f;
        s += end;
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0 && sum) {
        double tot = 0.0;
        for (int w = 0; w < (int)blockDim.x / 32; ++w) tot += red[w];
        *sum = tot;
    }
}
}  // namespace

extern "C" int sat_caption_masks(const int32_t* tokens, int32_t rows, int32_t T, int32_t eos_id, float* masks, double* mask_sum,
                                 void* stream) {
    if (!tokens || !masks || rows < 0 || T < 1) return sat_fail(SAT_ERR_INVALID, "sat_caption_masks: bad argument");
    caption_masks_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(tokens, rows, T, eos_id, masks, mask_sum);
    TCK(cudaGetLastError());
    return SAT_OK;
}

static int train_forward_backward(sat_handle* h, const float* params, float* grads, const float* contexts,
                                  const int32_t* sentences, const float* masks, const float* row_w, int32_t n_img,
                                  int32_t group, int32_t T, uint64_t seed, double global_mask_sum, const double* global_mask_sum_dev,
                                  int32_t global_batch, float* losses, void* stream) {
    if (!h || !params || !grads || !contexts || !sentences || !masks || !losses)
        return sat_fail(SAT_ERR_INVALID, "sat_train_forward_backward: null argument");
    // the packing kernels read W^T of the batch-row layers (params) and the contexts as float4, the fused scorer the
    // gradient rows (grads): a buffer off by a few floats is refused here, not met as a misaligned load on the device
    if (((reinterpret_cast<uintptr_t>(params) | reinterpret_cast<uintptr_t>(grads) | reinterpret_cast<uintptr_t>(contexts)) & 15) != 0)
        return sat_fail(SAT_ERR_INVALID, "sat_train_forward_backward: params, grads and contexts must be 16-byte aligned");
    TrainState* s = (TrainState*)*sat_handle_train_slot(h);
    const int32_t B = n_img * group;
    if (!s || s->n_img * s->group != B || s->T != T) return sat_fail(SAT_ERR_STATE, "call sat_train_init(B=%d, T=%d) first", B, T);
    TCK(cudaSetDevice(sat_handle_device(h)));
    cudaStream_t st = (cudaStream_t)stream;
    // per-call scalars -> device cells, in stream order.  The sources are ordinary (pageable) host variables: such a
    // copy is staged by the driver before the call returns, so no stream synchronisation is needed to reuse them
    // and the host can queue the next step while this one runs.
    unsigned long long seed_v = seed;
    float inv = (float)(1.0 / global_mask_sum);
    TCK(cudaMemcpyAsync(s->seed_d, &seed_v, 8, cudaMemcpyHostToDevice, st));
    if (global_mask_sum_dev) reciprocal_kernel<<<1, 1, 0, st>>>(s->inv_msum_d, global_mask_sum_dev);   // the sum never visits the host
    else TCK(cudaMemcpyAsync(s->inv_msum_d, &inv, 4, cudaMemcpyHostToDevice, st));
    auto enqueue = [&]() { return train_enqueue(s, params, grads, contexts, sentences, masks, row_w, B, T, global_batch, losses, st); };
    if (st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread) return enqueue();
    // (row weights are read on the device: new values in the same buffer replay the graph)
    std::vector<long long> key = {(long long)params, (long long)grads, (long long)contexts, (long long)sentences,
                                  (long long)masks, (long long)losses, B, T, global_batch,
                                  sat_handle_train_tc(h), sat_handle_layout_mode(h), group, (long long)row_w};
    TrainState::GEntry* ent = nullptr;
    for (auto& g : s->graphs)
        if (g.key == key) ent = &g;
    if (!ent) {
        if (s->graphs.size() >= 8) {
            if (s->graphs.front().exec) cudaGraphExecDestroy(s->graphs.front().exec);
            s->graphs.erase(s->graphs.begin());
        }
        s->graphs.emplace_back();
        ent = &s->graphs.back();
        ent->key = key;
    }
    if (ent->exec) { TCK(cudaGraphLaunch(ent->exec, st)); return SAT_OK; }
    if (ent->seen++ == 0) return enqueue();           // first call eager
    TCK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue();
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc != SAT_OK) { if (graph) cudaGraphDestroy(graph); return rc; }
    if (ce != cudaSuccess) return sat_fail(SAT_ERR_CUDA, "training graph capture failed: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&ent->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) { ent->exec = nullptr; return sat_fail(SAT_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ce)); }
    TCK(cudaGraphLaunch(ent->exec, st));
    return SAT_OK;
}

extern "C" int sat_train_forward_backward(sat_handle* h, const float* params, float* grads, const float* contexts,
                                          const int32_t* sentences, const float* masks, int32_t B, int32_t T,
                                          uint64_t seed, double global_mask_sum, int32_t global_batch, float* losses,
                                          void* stream) {
    TrainState* s = h ? (TrainState*)*sat_handle_train_slot(h) : nullptr;
    if (s && s->group != 1 && s->B == B && s->T == T)
        return sat_fail(SAT_ERR_STATE, "the training state is grouped (%d x %d): use sat_train_forward_backward_grouped", s->n_img, s->group);
    return train_forward_backward(h, params, grads, contexts, sentences, masks, nullptr, B, 1, T, seed, global_mask_sum, nullptr,
                                  global_batch, losses, stream);
}
// the same with the global mask sum in device memory (one double, e.g. the result of an all-reduce still in flight
// on `stream`): a data-parallel loop then has no host synchronisation per step
extern "C" int sat_train_forward_backward_dsum(sat_handle* h, const float* params, float* grads, const float* contexts,
                                               const int32_t* sentences, const float* masks, int32_t B, int32_t T,
                                               uint64_t seed, const double* global_mask_sum_dev, int32_t global_batch,
                                               float* losses, void* stream) {
    if (!global_mask_sum_dev) return sat_fail(SAT_ERR_INVALID, "sat_train_forward_backward_dsum: null mask sum");
    TrainState* s = h ? (TrainState*)*sat_handle_train_slot(h) : nullptr;
    if (s && s->group != 1 && s->B == B && s->T == T)
        return sat_fail(SAT_ERR_STATE, "the training state is grouped (%d x %d): use sat_train_forward_backward_grouped", s->n_img, s->group);
    return train_forward_backward(h, params, grads, contexts, sentences, masks, nullptr, B, 1, T, seed, 1.0, global_mask_sum_dev,
                                  global_batch, losses, stream);
}
// rows = n_img * group captions, row r of image r / group; contexts [n_img, L, D]; row_w [rows] or NULL (= 1)
extern "C" int sat_train_forward_backward_grouped(sat_handle* h, const float* params, float* grads, const float* contexts,
                                                  int32_t n_img, int32_t group, const int32_t* sentences, const float* masks,
                                                  const float* row_weights, int32_t T, uint64_t seed,
                                                  const double* global_mask_sum_dev, int32_t global_batch, float* losses,
                                                  void* stream) {
    if (!h || !params || !grads || !contexts || !sentences || !masks || !losses || !global_mask_sum_dev)
        return sat_fail(SAT_ERR_INVALID, "sat_train_forward_backward_grouped: null argument");
    if (group < 1 || n_img < 1 || T < 1) return sat_fail(SAT_ERR_INVALID, "sat_train_forward_backward_grouped: bad n_img/group/T");
    TrainState* s = (TrainState*)*sat_handle_train_slot(h);
    if (!s) return sat_fail(SAT_ERR_STATE, "call sat_train_init_grouped first");
    if (s->n_img != n_img || s->group != group || s->T != T)
        return sat_fail(SAT_ERR_INVALID, "sat_train_forward_backward_grouped: (n_img, group, T) = (%d, %d, %d), the state has (%d, %d, %d)",
                        n_img, group, T, s->n_img, s->group, s->T);
    return train_forward_backward(h, params, grads, contexts, sentences, masks, row_weights, n_img, group, T, seed, 1.0,
                                  global_mask_sum_dev, global_batch, losses, stream);
}

// grads: the (all-reduced) sum over data-parallel shards.  Adds the L2-regulariser gradient once, clips by the
// global norm (clip_gradients = 5.0, model.py:505-510) and applies the optimizer (model.py:479-503).  step counts from 1.
extern "C" int sat_train_apply_opt(sat_handle* h, float* params, float* grads, float* slot0, float* slot1, float* slot2,
                                   int64_t step, const sat_optimizer* opt, float* grad_norm, void* stream) {
    if (!h || !params || !grads || !opt) return sat_fail(SAT_ERR_INVALID, "sat_train_apply_opt: null argument");
    TrainState* s = (TrainState*)*sat_handle_train_slot(h);
    if (!s) return sat_fail(SAT_ERR_STATE, "call sat_train_init first");
    if (step < 1) return sat_fail(SAT_ERR_INVALID, "step counts from 1");
    const int kind = opt->kind;
    if (kind < SAT_OPT_ADAM || kind > SAT_OPT_SGD) return sat_fail(SAT_ERR_INVALID, "unknown optimizer kind %d", kind);
    if ((kind == SAT_OPT_ADAM && (!slot0 || !slot1)) || (kind == SAT_OPT_RMSPROP && (!slot0 || !slot2 || (opt->centered && !slot1))) ||
        (kind == SAT_OPT_MOMENTUM && !slot0))
        return sat_fail(SAT_ERR_INVALID, "sat_train_apply_opt: optimizer slot buffer missing");
    TCK(cudaSetDevice(sat_handle_device(h)));
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = s->off[kNumVars];
    for (int v = 0; v < kNumVars; ++v)
        if (s->regularised[v]) {
            const size_t nv = (size_t)s->rows[v] * s->cols[v];
            launch_k(axpy_kernel, GRID1D(nv), 256, st, grads + s->off[v], params + s->off[v], s->reg_scale, nv);
        }
    TCK(cudaMemsetAsync(s->loss_acc + 4, 0, sizeof(float), st));
    launch_k(sumsq_kernel, sat::device_sm_count() * 8, 256, st, grads, n, 1.0f, s->loss_acc + 4);   // padding entries are zero
    const float clip = opt->clip_gradients, lr = opt->learning_rate;
    if (kind == SAT_OPT_ADAM) {
        const double lr_t = (double)lr * sqrt(1.0 - pow((double)opt->beta2, (double)step)) / (1.0 - pow((double)opt->beta1, (double)step));
        launch_k(adam_kernel, GRID1D(n), 256, st, params, grads, slot0, slot1, n, s->loss_acc + 4, clip, (float)lr_t, opt->beta1, opt->beta2,
                 opt->epsilon);
    } else if (kind == SAT_OPT_RMSPROP) {
        launch_k(rmsprop_kernel, GRID1D(n), 256, st, params, grads, slot0, slot1, slot2, n, s->loss_acc + 4, clip, lr, opt->decay,
                 opt->momentum, opt->epsilon, opt->centered ? 1 : 0);
    } else {
        launch_k(momentum_kernel, GRID1D(n), 256, st, params, grads, slot0, n, s->loss_acc + 4, clip, lr, opt->momentum,
                 opt->use_nesterov ? 1 : 0, kind == SAT_OPT_SGD ? 1 : 0);
    }
    TCK(cudaGetLastError());
    if (grad_norm) TCK(cudaMemcpyAsync(grad_norm, s->loss_acc + 4, sizeof(float), cudaMemcpyDeviceToDevice, st));  // norm^2
    return SAT_OK;
}

// TF's RMSProp starts its `rms` slot at one (the other slots of every optimizer start at zero)
extern "C" int sat_train_fill(sat_handle* h, float* buf, float value, int64_t n, void* stream) {
    if (!h || !buf || n < 0) return sat_fail(SAT_ERR_INVALID, "sat_train_fill: bad argument");
    TCK(cudaSetDevice(sat_handle_device(h)));
    fill_kernel<<<sat::device_sm_count() * 4, 256, 0, (cudaStream_t)stream>>>(buf, value, (size_t)n);
    TCK(cudaGetLastError());
    return SAT_OK;
}

extern "C" int sat_train_apply(sat_handle* h, float* params, float* grads, float* adam_m, float* adam_v, int64_t step, float lr,
                               float beta1, float beta2, float epsilon, float clip, float* grad_norm, void* stream) {
    if (!adam_m || !adam_v) return sat_fail(SAT_ERR_INVALID, "sat_train_apply: null argument");
    sat_optimizer o;
    memset(&o, 0, sizeof(o));
    o.kind = SAT_OPT_ADAM; o.learning_rate = lr; o.beta1 = beta1; o.beta2 = beta2; o.epsilon = epsilon; o.clip_gradients = clip;
    return sat_train_apply_opt(h, params, grads, adam_m, adam_v, nullptr, step, &o, grad_norm, stream);
}
