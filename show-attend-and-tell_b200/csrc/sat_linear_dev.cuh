// sat_linear_dev.cuh — device helpers shared by the dense kernels (sat_linear.cu: one launch per layer;
// sat_chain.cu: the three dense layers of a decode step in one persistent launch).  Include after sat_common.cuh
// and sat_linear.cuh.
#pragma once
#include "sat_common.cuh"
#include "sat_linear.cuh"

namespace sat {

// ---------------------------------------------------------------- helpers
__device__ __forceinline__ void split_bf16x8(const float4& a, const float4& b, uint4& hi, uint4& lo) {
    float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        __nv_bfloat16 h0 = __float2bfloat16_rn(x[2 * i]);
        __nv_bfloat16 h1 = __float2bfloat16_rn(x[2 * i + 1]);
        __nv_bfloat16 l0 = __float2bfloat16_rn(x[2 * i] - __bfloat162float(h0));
        __nv_bfloat16 l1 = __float2bfloat16_rn(x[2 * i + 1] - __bfloat162float(h1));
        h[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
        l[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// TF LSTMCell (un-vendored TF 1.7 dependency; gate order i, j, f, o and forget_bias 1.0
// confirmed on the reference's recorded GraphDef, tests/golden/graph_fixture.json):
//   c = sigmoid(f + 1) * c_prev + sigmoid(i) * tanh(j);  h = sigmoid(o) * tanh(c)
__device__ __forceinline__ void lstm_gates(const LinProblem& P, float4 g, float cp, int b, int unit, int mode, bool dry) {
    const float c = act_sigmoid(g.z + 1.0f) * cp + act_sigmoid(g.x) * act_tanh(g.y);
    const float h = act_sigmoid(g.w) * act_tanh(c);
    if (dry) return;   // instruction-cache warm-up pass: no side effects
    P.c_out[(size_t)b * P.H + unit] = c;
    P.h_out[(size_t)b * P.H + unit] = h;
    if (P.out_pa) pa_store(P.out_pa, mode, P.row_tile, P.H >> 6, b, unit, h);   // h feeds the next dense layers
}

// ---------------------------------------------------------------- tensor-core tile
// The 128 x N accumulator tile of a dense CTA (128 outputs x N batch rows, N <= 16 * NT <= kMaxRowTile) is held in the
// registers of the eight consumer warps 0..7: warpgroup g = threadIdx.x / 128 owns outputs [64g, 64g + 64) as NT
// register fragment of one 64 x 16NT wgmma (v[j] = its columns [16j, 16j + 16)).  NT is a compile-time constant: the
// MMA width is part of the instruction.
template <int NT>
struct AccTile {
    float v[NT][8];
};

// acc += W * X^T over the K block in the pipeline stage at shared address `wb` (W hi | W lo | X hi | X lo):
// per 16-wide K step the three split-precision products Whi*Xhi, Wlo*Xhi, Whi*Xlo (N = 16 NT batch rows).  Returns when the MMAs are complete, i.e. the stage may be refilled.  Every consumer warp calls it.
template <int NT>
__device__ __forceinline__ void mma_kblock(AccTile<NT>& acc, uint32_t wb, uint32_t x_half_bytes, int mode, bool first) {
    const uint32_t lbo = mode == 0 ? 128u : 16u;
    const uint32_t layout = mode == 0 ? 0u : 1u;
    const uint32_t kstep16 = (mode == 0 ? 256u : 32u) >> 4;   // descriptor address units (16 B) per K step of 16
    const uint64_t dzero = gmma_smem_desc(0u, lbo, 1024, layout);
    const uint32_t wrow = (threadIdx.x >> 7) * 8192u;         // this warpgroup's 64 rows of W: eight 1024-byte row groups
    // (14-bit start-address field: in a cluster launch a shared-memory address may carry the CTA's rank in its high
    // bits, which must not leak into the descriptor's other fields)
    uint64_t a_hi = dzero + (uint64_t)(((wb + wrow) >> 4) & 0x3FFFu);
    uint64_t a_lo = dzero + (uint64_t)(((wb + kWHalfBytes + wrow) >> 4) & 0x3FFFu);
    uint64_t b_hi = dzero + (uint64_t)(((wb + kWStageBytes) >> 4) & 0x3FFFu);
    uint64_t b_lo = dzero + (uint64_t)(((wb + kWStageBytes + x_half_bytes) >> 4) & 0x3FFFu);
    float* const d = &acc.v[0][0];
    wgmma_fence_operand(d, 8 * NT);
    wgmma_fence();
    uint32_t scale = first ? 0u : 1u;                         // the first product of a tile starts the sum
    // (fully unrolled: in a rolled loop ptxas serialises the MMAs; the empty asm at the end of a step keeps it from
    // precomputing the descriptors of all four steps into registers)
#pragma unroll
    for (int kk = 0; kk < kBK / 16; ++kk) {
        Wgmma<16 * NT>::mma(d, a_hi, b_hi, scale);
        Wgmma<16 * NT>::mma(d, a_lo, b_hi, 1u);
        Wgmma<16 * NT>::mma(d, a_hi, b_lo, 1u);
        scale = 1u;
        a_hi += kstep16; a_lo += kstep16; b_hi += kstep16; b_lo += kstep16;
        asm volatile("" : "+l"(a_hi), "+l"(a_lo), "+l"(b_hi), "+l"(b_lo));
    }
    wgmma_commit();
    wgmma_wait_all();
    wgmma_fence_operand(d, 8 * NT);
}

// f(m, n, value) for every accumulator element this thread holds: output m in [0, 128) of the tile, batch row n < N
template <int NT, typename F>
__device__ __forceinline__ void acc_for_each(const AccTile<NT>& acc, int N, F&& f) {
    const int l = threadIdx.x & 31;
    const int m0 = (threadIdx.x >> 7) * 64 + ((threadIdx.x >> 5) & 3) * 16 + (l >> 2);
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        if (16 * j < N) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int e = 0; e < 2; ++e) f(m0 + 8 * h, 16 * j + 8 * i + 2 * (l & 3) + e, acc.v[j][4 * i + 2 * h + e]);
        }
    }
}

}  // namespace sat
