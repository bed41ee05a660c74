// sat_attention.cu — fused soft attention of one decode step:
//   e[b,l]   = sum_a w2[a] * (T1[img(b),l,a] + q[b,a])        (attend, model.py:427-434)
//   alpha    = softmax_l(e)                                    (model.py:435)
//   z[b,:]   = sum_l alpha[b,l] * ctx[img(b),l,:]              (model.py:263-264)
// in ONE kernel.  T1 = tanh(ctx*W1a + b1a) is the step-invariant feature branch
// (model.py:417-420) produced once per image batch by sat_prepare_contexts;
// q = tanh(h*W1b + b1b) is the state branch (model.py:421-424).  The 1-layer scorer
// (model.py:401-414) runs through the same kernel with T = ctx, vec = fc_a kernel,
// q = null and eadd = h*fc_b.
//
// The kernel is HBM-bound (it streams T1 and ctx once: 4*[B*L*(D+A)] bytes) and is cut
// so that every SM pulls the same number of CONTIGUOUS bytes: the NI*L locations are
// split into equal contiguous row ranges, one per CTA (<= #SMs CTAs).  For each image
// segment of its range a CTA
//   1. streams the T1 rows (1-D bulk TMA chunks into a shared-memory ring), one warp per
//      row, warp-shuffle reduction -> logits e (kept in smem, also written to global);
//   2. takes the segment-local max m and weights w_l = exp(e_l - m), s = sum w_l;
//   3. streams the ctx rows of the SAME range through the same ring and accumulates the
//      un-normalised partial context  zp[d] = sum_l w_l * ctx[l, d]  (thread per d);
//   4. publishes (m, s, zp); the LAST CTA to finish an image (atomic counter) merges the
//      partials in fixed CTA order:  M = max m_c,  S = sum s_c e^{m_c-M},
//      z = sum zp_c e^{m_c-M} / S,  alpha_l = e^{e_l-M} / S     (softmax, split over L).
// There is no grid-wide dependency inside the kernel: a single producer thread keeps the
// ring full across the T1 -> ctx boundary, so the SM never waits on another SM.
// G rows (beams) of one image share the image's T1/ctx traffic.
//
// Two kernels implement this: att_wpc_kernel (further down; rows of exactly 512 floats, the reference's sizes:
// a TMA chunk of 8 rows belongs to ONE consumer warp, row sums by a transposing butterfly, whole-image CTAs
// normalise in place) and att_fused_kernel (below; any width, all warps on every chunk) as the general path.
#include "sat_common.cuh"
#include "sat_attention.cuh"
#include "sat_linear.cuh"

namespace sat {

// consumer warps per CTA: 8 (all G) or 16 (G == 1: twice the warps hide the shared-memory / shuffle latency
// of the two passes; needs <= 112 registers per thread)
constexpr int kAttMaxDPerThread = 8;   // D <= 2048

__device__ __forceinline__ int att_rbegin(long long NR, int P, int c) { return (int)(NR * c / P); }

// side job of the attention kernels: embedding rows of the words fed to this step -> packed operand tiles
// (a few 16-byte groups per thread)
__device__ __forceinline__ void att_pack_embedding(const AttParams& p, int first, int stride, int G) {
    const int groups = p.emb_E >> 3;
    const int total = p.NI * G * groups;
    const size_t half = (size_t)p.pa_row_tile * kBK * 2;
    for (int u = first; u < total; u += stride) {
        const int b = u / groups, gi = u - b * groups;
        const int w = p.emb_word[b];
        const float4* src = reinterpret_cast<const float4*>(p.emb + (size_t)w * p.emb_E + gi * 8);
        const float4 a = __ldg(src), a2 = __ldg(src + 1);
        const float x[8] = {a.x, a.y, a.z, a.w, a2.x, a2.y, a2.z, a2.w};
        uint32_t hh[4], ll[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const __nv_bfloat16 h0 = __float2bfloat16_rn(x[2 * i]), h1 = __float2bfloat16_rn(x[2 * i + 1]);
            const __nv_bfloat16 l0 = __float2bfloat16_rn(x[2 * i] - __bfloat162float(h0));
            const __nv_bfloat16 l1 = __float2bfloat16_rn(x[2 * i + 1] - __bfloat162float(h1));
            hh[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
            ll[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
        }
        const int rt = b / p.pa_row_tile, r = b - rt * p.pa_row_tile;
        uint8_t* dst = p.emb_pa + ((size_t)rt * (p.emb_E >> 6) + (gi >> 3)) * 2 * half + mma_tile_off(p.pa_mode, r, gi & 7);
        *reinterpret_cast<uint4*>(dst) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
        *reinterpret_cast<uint4*>(dst + half) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
    }
}

template <int G, int RV, int OCC, int NW>
__global__ void __launch_bounds__((NW + 1) * 32, OCC) att_fused_kernel(const __grid_constant__ AttParams p) {
    constexpr int kAttConsumerWarps = NW;
    extern __shared__ __align__(1024) uint8_t smem[];
    // layout: [slots][barriers 2*nslots*8][vec RL][q G*RL][w G*Lp][misc 64]
    uint8_t* slots = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.nslots * p.slot_bytes);
    uint64_t* empty = full + p.nslots;
    float* vec_s = reinterpret_cast<float*>(empty + p.nslots);
    float* q_s = vec_s + p.RL;
    const int Lp = (p.L + 3) & ~3;
    float* w_s = q_s + (size_t)G * p.RL;          // logits, then softmax weights of the current segment
    float* misc = w_s + (size_t)G * Lp;            // [G] max, [G] sum, flag

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int P = gridDim.x, c = blockIdx.x;
    const int L = p.L, RL = p.RL, D = p.D;
    const long long NR = (long long)p.NI * L;
    const int r_begin = att_rbegin(NR, P, c), r_end = att_rbegin(NR, P, c + 1);

    if (threadIdx.x == 0) {
        trace_stamp(p.dbg, 0);
        tl_begin(p.tl);
        for (int s = 0; s < p.nslots; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], kAttConsumerWarps);
        }
        fence_mbar_init();
    }
    __syncthreads();
    if (p.pdl) { pdl_wait(); pdl_launch_dependents(); }   // q / word of this step come from the predecessor
    if (threadIdx.x == 0) tl_go(p.tl);

    if (warp == kAttConsumerWarps) {
        // ============================ producer ============================
        if (lane == 0) {
            const uint64_t pol_t = l2_policy(p.l2_t), pol_c = l2_policy(p.l2_ctx);
            int idx = 0;
            for (int seg0 = r_begin; seg0 < r_end;) {
                const int img = seg0 / L;
                const int seg1 = min(r_end, (img + 1) * L);
                for (int pass = 0; pass < 2; ++pass) {
                    const float* src = pass == 0 ? p.T : p.ctx;
                    const int rl = pass == 0 ? RL : D;
                    const int rch = pass == 0 ? p.rch : p.cch;
                    const int pol_k = pass == 0 ? p.l2_t : p.l2_ctx;
                    const uint64_t pol = pass == 0 ? pol_t : pol_c;
                    for (int r = seg0; r < seg1; r += rch, ++idx) {
                        const int n = min(rch, seg1 - r);
                        const int s = idx % p.nslots;
                        const uint32_t ph = (uint32_t)(idx / p.nslots) & 1u;
                        mbar_wait(&empty[s], ph ^ 1u);
                        const uint32_t bytes = (uint32_t)n * rl * 4u;
                        mbar_arrive_expect_tx(&full[s], bytes);
                        tma_bulk_g2s_hint(slots + (size_t)s * p.slot_bytes, src + (size_t)r * rl, bytes, &full[s], pol_k,
                                          pol);
                    }
                }
                seg0 = seg1;
            }
        }
        return;
    }

    // ============================== consumers ==============================
    const int ct = threadIdx.x;  // 0..255
    constexpr int NT = kAttConsumerWarps * 32;
    for (int j = ct; j < RL; j += NT) vec_s[j] = p.vec[j];
    named_bar_sync(1, NT);
    float4 wreg[RV > 0 ? RV : 1];
    float4 qreg[G][RV > 0 ? RV : 1];
    if (RV > 0) {
#pragma unroll
        for (int k = 0; k < (RV > 0 ? RV : 1); ++k) wreg[k] = reinterpret_cast<const float4*>(vec_s)[lane + 32 * k];
    }
    const int nper = (D + NT - 1) / NT;   // context features per thread (d = ct + NT*k)
    int idx = 0;
    bool first_seg = true;
    long long wait1 = 0, wait2 = 0;   // cycles thread 0 spent blocked on "chunk landed" in pass 1 / pass 2 (trace)
    long long ph_a = 0, ph_b = 0, ph_c = 0, ph_d = 0;   // trace: pass-1 cycles in loads+FMA / reduction / stores+arrive, pass-2 compute
    if (p.emb_pa) att_pack_embedding(p, c * NT + ct, P * NT, G);
    if (ct == 0) trace_stamp(p.dbg, 1);

    for (int seg0 = r_begin; seg0 < r_end;) {
        const int img = seg0 / L;
        const int seg1 = min(r_end, (img + 1) * L);
        const int nseg = seg1 - seg0;
        // ---- state branch of this image
        if (RV > 0) {
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
                for (int k = 0; k < (RV > 0 ? RV : 1); ++k)
                    qreg[g][k] = p.q ? __ldg(reinterpret_cast<const float4*>(p.q + ((size_t)img * G + g) * RL) + lane + 32 * k)
                                     : make_float4(0.f, 0.f, 0.f, 0.f);
            if (!first_seg) named_bar_sync(1, NT);      // previous segment's w_s fully consumed
        } else {
            if (!first_seg) named_bar_sync(1, NT);
            if (p.q) {
                const float4* src = reinterpret_cast<const float4*>(p.q + (size_t)img * G * RL);
                float4* dst = reinterpret_cast<float4*>(q_s);
                for (int j = ct; j < G * RL / 4; j += NT) dst[j] = src[j];
            }
            named_bar_sync(1, NT);
        }
        first_seg = false;

        // ---- pass 1: logits of the segment's locations
        for (int r = seg0; r < seg1; r += p.rch, ++idx) {
            const int n = min(p.rch, seg1 - r);
            const int s = idx % p.nslots;
            const long long tw = p.dbg ? clock64() : 0;
            mbar_wait(&full[s], (uint32_t)(idx / p.nslots) & 1u);
            if (p.dbg) wait1 += clock64() - tw;
            if (ct == 0 && r == r_begin) trace_stamp(p.dbg, 2);
            const float* buf = reinterpret_cast<const float*>(slots + (size_t)s * p.slot_bytes);
            // two rows per warp at a time (rows `row` and `row + 8`), two independent partial sums per row and
            // per g: four FMA chains in flight instead of one 16-deep dependent chain, and the two warp
            // reductions interleave
            long long tq0 = p.dbg ? clock64() : 0, tq1 = 0, tq2 = 0;
            for (int row = warp; row < n; row += 2 * kAttConsumerWarps) {
                const int rowB = row + kAttConsumerWarps;
                const bool hasB = rowB < n;
                float accA[G][2], accB[G][2];
#pragma unroll
                for (int g = 0; g < G; ++g) { accA[g][0] = accA[g][1] = accB[g][0] = accB[g][1] = 0.f; }
                const float4* trA = reinterpret_cast<const float4*>(buf + (size_t)row * RL);
                const float4* trB = reinterpret_cast<const float4*>(buf + (size_t)(hasB ? rowB : row) * RL);
                if (RV > 0) {
                    float4 tA[RV > 0 ? RV : 1], tB[RV > 0 ? RV : 1];
#pragma unroll
                    for (int k = 0; k < (RV > 0 ? RV : 1); ++k) { tA[k] = trA[lane + 32 * k]; tB[k] = trB[lane + 32 * k]; }
#pragma unroll
                    for (int k = 0; k < (RV > 0 ? RV : 1); ++k) {
                        const float4 w = wreg[k];
#pragma unroll
                        for (int g = 0; g < G; ++g) {
                            const float4 qq = qreg[g][k];
                            accA[g][0] = fmaf(w.x, tA[k].x + qq.x, accA[g][0]);
                            accA[g][1] = fmaf(w.y, tA[k].y + qq.y, accA[g][1]);
                            accA[g][0] = fmaf(w.z, tA[k].z + qq.z, accA[g][0]);
                            accA[g][1] = fmaf(w.w, tA[k].w + qq.w, accA[g][1]);
                            accB[g][0] = fmaf(w.x, tB[k].x + qq.x, accB[g][0]);
                            accB[g][1] = fmaf(w.y, tB[k].y + qq.y, accB[g][1]);
                            accB[g][0] = fmaf(w.z, tB[k].z + qq.z, accB[g][0]);
                            accB[g][1] = fmaf(w.w, tB[k].w + qq.w, accB[g][1]);
                        }
                    }
                } else {
                    for (int j = lane; j < RL / 4; j += 32) {
                        const float4 ta = trA[j], tb = trB[j];
                        const float4 w = reinterpret_cast<const float4*>(vec_s)[j];
#pragma unroll
                        for (int g = 0; g < G; ++g) {
                            float4 qq = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (p.q) qq = reinterpret_cast<const float4*>(q_s + (size_t)g * RL)[j];
                            accA[g][0] = fmaf(w.x, ta.x + qq.x, accA[g][0]);
                            accA[g][1] = fmaf(w.y, ta.y + qq.y, accA[g][1]);
                            accA[g][0] = fmaf(w.z, ta.z + qq.z, accA[g][0]);
                            accA[g][1] = fmaf(w.w, ta.w + qq.w, accA[g][1]);
                            accB[g][0] = fmaf(w.x, tb.x + qq.x, accB[g][0]);
                            accB[g][1] = fmaf(w.y, tb.y + qq.y, accB[g][1]);
                            accB[g][0] = fmaf(w.z, tb.z + qq.z, accB[g][0]);
                            accB[g][1] = fmaf(w.w, tb.w + qq.w, accB[g][1]);
                        }
                    }
                }
                if (p.dbg) { float sink = accA[0][0] + accB[0][1]; if (sink == 12345.678f) tq1 = 1; tq1 = clock64(); }
#pragma unroll
                for (int g = 0; g < G; ++g) {
                    float sa = accA[g][0] + accA[g][1], sb = accB[g][0] + accB[g][1];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        sa += __shfl_xor_sync(0xffffffffu, sa, o);
                        sb += __shfl_xor_sync(0xffffffffu, sb, o);
                    }
                    if (p.dbg) { if (sa == 12345.678f) tq2 = 1; tq2 = clock64(); }
                    if (lane < 2 && (lane == 0 || hasB)) {
                        const int rr = lane == 0 ? row : rowB;
                        float sum = lane == 0 ? sa : sb;
                        const int ll = r + rr - seg0;            // location index within the segment
                        const int l = r + rr - img * L;          // location index within the image
                        const size_t o = ((size_t)img * G + g) * L + l;
                        if (p.eadd) sum += p.eadd[o];
                        p.e[o] = sum;
                        w_s[g * Lp + ll] = sum;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
            if (p.dbg) { const long long tq3 = clock64(); ph_a += tq1 - tq0; ph_b += tq2 - tq1; ph_c += tq3 - tq2; }
        }
        named_bar_sync(1, NT);
        if (ct == 0 && seg0 == r_begin) trace_stamp(p.dbg, 3);

        // ---- segment-local softmax statistics: m = max e, w = exp(e - m), s = sum w
        for (int g = warp; g < G; g += kAttConsumerWarps) {
            float m = -INFINITY;
            for (int l = lane; l < nseg; l += 32) m = fmaxf(m, w_s[g * Lp + l]);
            m = warp_max(m);
            float sum = 0.f;
            for (int l = lane; l < nseg; l += 32) {
                const float ex = expf(w_s[g * Lp + l] - m);
                w_s[g * Lp + l] = ex;
                sum += ex;
            }
            sum = warp_sum(sum);
            if (lane == 0) { misc[g] = m; misc[G + g] = sum; }
        }
        named_bar_sync(1, NT);

        // ---- pass 2: un-normalised partial context over the SAME rows.  Thread ct owns the features
        // d = 2*ct + 512*k (+1) when D % 512 == 0 (float2 per 512 features), else d = ct + 256*k.
        float zacc[G][kAttMaxDPerThread];
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int k = 0; k < kAttMaxDPerThread; ++k) zacc[g][k] = 0.f;
        const bool vec2 = (D % (2 * NT)) == 0;
        const int nk2 = D / (2 * NT);
        const bool vec1 = !vec2 && (D % NT) == 0;      // one float per NT features (16 warps, D = 512)
        const int nk1 = D / NT;
        for (int r = seg0; r < seg1; r += p.cch, ++idx) {
            const int n = min(p.cch, seg1 - r);
            const int s = idx % p.nslots;
            const long long tw = p.dbg ? clock64() : 0;
            mbar_wait(&full[s], (uint32_t)(idx / p.nslots) & 1u);
            if (p.dbg) wait2 += clock64() - tw;
            if (ct == 0 && r == r_begin) trace_stamp(p.dbg, 4);
            const long long tp0 = p.dbg ? clock64() : 0;
            const float* buf = reinterpret_cast<const float*>(slots + (size_t)s * p.slot_bytes);
            if (vec2) {
                const float2* b2 = reinterpret_cast<const float2*>(buf) + ct;
                const int rowstride = D / 2;   // float2 per row
                int row = 0;
                for (; row + 8 <= n; row += 8) {
                    const int ll = r + row - seg0;      // chunks start at multiples of cch (a multiple of 4): aligned
                    float wv[G][8];
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        if (((g * Lp + ll) & 3) == 0) {
                            const float4 w0 = *reinterpret_cast<const float4*>(w_s + g * Lp + ll);
                            const float4 w1 = *reinterpret_cast<const float4*>(w_s + g * Lp + ll + 4);
                            wv[g][0] = w0.x; wv[g][1] = w0.y; wv[g][2] = w0.z; wv[g][3] = w0.w;
                            wv[g][4] = w1.x; wv[g][5] = w1.y; wv[g][6] = w1.z; wv[g][7] = w1.w;
                        } else {
#pragma unroll
                            for (int j = 0; j < 8; ++j) wv[g][j] = w_s[g * Lp + ll + j];
                        }
                    }
#pragma unroll
                    for (int k = 0; k < kAttMaxDPerThread / 2; ++k) {
                        if (k < nk2) {
                            float2 x[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) x[j] = b2[(size_t)(row + j) * rowstride + NT * k];
#pragma unroll
                            for (int g = 0; g < G; ++g) {
                                float s0 = 0.f, s1 = 0.f, t0 = 0.f, t1 = 0.f;   // two chains per feature
#pragma unroll
                                for (int j = 0; j < 8; j += 2) {
                                    s0 = fmaf(wv[g][j], x[j].x, s0);
                                    s1 = fmaf(wv[g][j], x[j].y, s1);
                                    t0 = fmaf(wv[g][j + 1], x[j + 1].x, t0);
                                    t1 = fmaf(wv[g][j + 1], x[j + 1].y, t1);
                                }
                                zacc[g][2 * k] += s0 + t0;
                                zacc[g][2 * k + 1] += s1 + t1;
                            }
                        }
                    }
                }
                for (; row < n; ++row) {
                    const int ll = r + row - seg0;
#pragma unroll
                    for (int k = 0; k < kAttMaxDPerThread / 2; ++k) {
                        if (k < nk2) {
                            const float2 x = b2[(size_t)row * rowstride + NT * k];
#pragma unroll
                            for (int g = 0; g < G; ++g) {
                                const float wv = w_s[g * Lp + ll];
                                zacc[g][2 * k] = fmaf(wv, x.x, zacc[g][2 * k]);
                                zacc[g][2 * k + 1] = fmaf(wv, x.y, zacc[g][2 * k + 1]);
                            }
                        }
                    }
                }
            } else if (vec1) {
                const float* b1 = buf + ct;
                int row = 0;
                for (; row + 8 <= n; row += 8) {
                    const int ll = r + row - seg0;
                    float wv[G][8];
#pragma unroll
                    for (int g = 0; g < G; ++g)
#pragma unroll
                        for (int j = 0; j < 8; ++j) wv[g][j] = w_s[g * Lp + ll + j];
#pragma unroll
                    for (int k = 0; k < kAttMaxDPerThread; ++k) {
                        if (k < nk1) {
                            float x[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) x[j] = b1[(size_t)(row + j) * D + NT * k];
#pragma unroll
                            for (int g = 0; g < G; ++g) {
                                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                                for (int j = 0; j < 8; j += 2) {
                                    s0 = fmaf(wv[g][j], x[j], s0);
                                    s1 = fmaf(wv[g][j + 1], x[j + 1], s1);
                                }
                                zacc[g][k] += s0 + s1;
                            }
                        }
                    }
                }
                for (; row < n; ++row) {
                    const int ll = r + row - seg0;
#pragma unroll
                    for (int k = 0; k < kAttMaxDPerThread; ++k)
                        if (k < nk1) {
                            const float x = b1[(size_t)row * D + NT * k];
#pragma unroll
                            for (int g = 0; g < G; ++g) zacc[g][k] = fmaf(w_s[g * Lp + ll], x, zacc[g][k]);
                        }
                }
            } else {
                for (int row = 0; row < n; ++row) {
                    const int ll = r + row - seg0;
                    float wv[G];
#pragma unroll
                    for (int g = 0; g < G; ++g) wv[g] = w_s[g * Lp + ll];
                    const float* xrow = buf + (size_t)row * D;
#pragma unroll
                    for (int k = 0; k < kAttMaxDPerThread; ++k) {
                        if (k < nper) {
                            const int d = ct + NT * k;
                            const float x = d < D ? xrow[d] : 0.f;
#pragma unroll
                            for (int g = 0; g < G; ++g) zacc[g][k] = fmaf(wv[g], x, zacc[g][k]);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
            if (p.dbg) { if (zacc[0][0] == 12345.678f) ph_d = 1; ph_d += clock64() - tp0; }
        }
        // feature index of accumulator k of this thread
        auto feat = [&](int k) { return vec2 ? 2 * ct + 2 * NT * (k >> 1) + (k & 1) : ct + NT * k; };
        const int nacc = vec2 ? 2 * nk2 : nper;

        if (ct == 0 && seg0 == r_begin) trace_stamp(p.dbg, 5);
        // ---- publish the partial, last CTA of the image merges
        const int slot_id = img - r_begin / L;                // ordinal of this segment within the CTA
        float* part = p.part + ((size_t)c * p.segmax + slot_id) * G * (D + 2);
#pragma unroll
        for (int g = 0; g < G; ++g) {
#pragma unroll
            for (int k = 0; k < kAttMaxDPerThread; ++k) {
                const int d = feat(k);
                if (k < nacc && d < D) part[(size_t)g * (D + 2) + d] = zacc[g][k];
            }
            if (ct == 0) { part[(size_t)g * (D + 2) + D] = misc[g]; part[(size_t)g * (D + 2) + D + 1] = misc[G + g]; }
        }
        // contributors of this image: CTAs c_lo..c_hi whose row ranges overlap [img*L, (img+1)*L)
        int c_lo = (int)(((long long)img * L * P) / NR);
        while (c_lo + 1 < P && att_rbegin(NR, P, c_lo + 1) <= img * L) ++c_lo;
        while (c_lo > 0 && att_rbegin(NR, P, c_lo) > img * L) --c_lo;
        int c_hi = (int)((((long long)(img + 1) * L - 1) * P) / NR);
        while (c_hi + 1 < P && att_rbegin(NR, P, c_hi + 1) <= (img + 1) * L - 1) ++c_hi;
        while (c_hi > 0 && att_rbegin(NR, P, c_hi) > (img + 1) * L - 1) --c_hi;
        named_bar_sync(1, NT);                                // every thread's partial stores are ordered before ...
        unsigned* flag = reinterpret_cast<unsigned*>(misc + 2 * G);
        if (ct == 0) {
            __threadfence();                                  // ... this (cumulative) release
            *flag = atomicAdd(p.rowcnt + img, 1u) == (unsigned)(c_hi - c_lo) ? 1u : 0u;
        }
        named_bar_sync(1, NT);
        if (ct == 0 && seg0 == r_begin) trace_stamp(p.dbg, 6);
        if (ct == 0 && seg1 == r_end) tl_main_done(p.tl);
        if (*flag) {
            __threadfence();
            if (ct == 0) p.rowcnt[img] = 0u;                  // ready for the next launch
            // every thread redundantly reads the (max, sum) pair of each contributor (a few L2 loads, all in
            // flight together with its own slice of the partial contexts and of the logits): one round trip
            const int nc = c_hi - c_lo + 1;
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float* er = p.e + ((size_t)img * G + g) * L;
                float ev[2];
                ev[0] = ct < L ? __ldcg(er + ct) : 0.f;
                ev[1] = ct + NT < L ? __ldcg(er + ct + NT) : 0.f;
                float M = -INFINITY;
                for (int j0 = 0; j0 < nc; j0 += 8) {
                    float mm[8];
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
                        const int j = j0 + jj;
                        mm[jj] = -INFINITY;
                        if (j < nc) {
                            const int cc = c_lo + j;
                            const int sid = img - att_rbegin(NR, P, cc) / L;
                            mm[jj] = __ldcg(p.part + (((size_t)cc * p.segmax + sid) * G + g) * (D + 2) + D);
                        }
                    }
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) M = fmaxf(M, mm[jj]);
                }
                float S = 0.f;
                float zz[kAttMaxDPerThread];
#pragma unroll
                for (int k = 0; k < kAttMaxDPerThread; ++k) zz[k] = 0.f;
                for (int j0 = 0; j0 < nc; j0 += 4) {           // partials of up to 4 contributors in flight
                    float v[4][kAttMaxDPerThread], ms[4], ss[4];
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int j = j0 + jj;
                        ms[jj] = -INFINITY;
                        ss[jj] = 0.f;
                        if (j < nc) {
                            const int cc = c_lo + j;
                            const int sid = img - att_rbegin(NR, P, cc) / L;
                            const float* pp = p.part + (((size_t)cc * p.segmax + sid) * G + g) * (D + 2);
                            ms[jj] = __ldcg(pp + D);
                            ss[jj] = __ldcg(pp + D + 1);
#pragma unroll
                            for (int k = 0; k < kAttMaxDPerThread; ++k) {
                                const int d = feat(k);
                                v[jj][k] = (k < nacc && d < D) ? __ldcg(pp + d) : 0.f;
                            }
                        }
                    }
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        if (j0 + jj < nc) {
                            const float sc = expf(ms[jj] - M);
                            S = fmaf(ss[jj], sc, S);
#pragma unroll
                            for (int k = 0; k < kAttMaxDPerThread; ++k) zz[k] = fmaf(v[jj][k], sc, zz[k]);
                        }
                    }
                }
                const float inv = 1.0f / S;
#pragma unroll
                for (int k = 0; k < kAttMaxDPerThread; ++k) {
                    const int d = feat(k);
                    if (k < nacc && d < D) {
                        const float zv = zz[k] * inv;
                        p.z[((size_t)img * G + g) * D + d] = zv;
                        if (p.pa_z) pa_store(p.pa_z, p.pa_mode, p.pa_row_tile, D >> 6, img * G + g, d, zv);
                    }
                }
                if (ct < L) p.alpha[((size_t)img * G + g) * L + ct] = expf(ev[0] - M) * inv;
                if (ct + NT < L) p.alpha[((size_t)img * G + g) * L + ct + NT] = expf(ev[1] - M) * inv;
                for (int l = ct + 2 * NT; l < L; l += NT) p.alpha[((size_t)img * G + g) * L + l] = expf(__ldcg(er + l) - M) * inv;
            }
            named_bar_sync(1, NT);                            // st_sc (= w_s) is rewritten by the next segment
        }
        seg0 = seg1;
    }
    if (ct == 0) { trace_stamp(p.dbg, 7); tl_end(p.tl); }
    if (ct == 0 && p.dbg) {
        p.dbg[(size_t)blockIdx.x * 16 + 8] = (unsigned long long)wait1;
        p.dbg[(size_t)blockIdx.x * 16 + 9] = (unsigned long long)wait2;
        p.dbg[(size_t)blockIdx.x * 16 + 10] = (unsigned long long)ph_a;
        p.dbg[(size_t)blockIdx.x * 16 + 11] = (unsigned long long)ph_b;
        p.dbg[(size_t)blockIdx.x * 16 + 12] = (unsigned long long)ph_c;
        p.dbg[(size_t)blockIdx.x * 16 + 13] = (unsigned long long)ph_d;
    }
}

// =====================================================================================================
// Warp-per-chunk variant for rows of exactly 512 floats (RL == D == 512: the reference's dim_attend_layer and
// dim_ctx).  Same algorithm and outputs as att_fused_kernel, but cut so that the shared-memory port and the
// synchronisation cost stop limiting a single SM well below its share of the HBM stream:
//   * a TMA chunk is 8 rows (16 KB) and belongs to ONE consumer warp (chunk i -> warp i % 8): a warp
//     synchronises twice per 16 KB (one wait, one arrive) instead of eight warps doing so per 32 KB, and up to
//     8 chunks are being consumed concurrently;
//   * pass 1: lane j holds elements {4j..4j+3} + 128k of w2 and q; the 8 row sums of a chunk are reduced with
//     a 9-shuffle transposing butterfly (instead of 5 shuffles per row);
//   * pass 2: lane j accumulates the same 16 of the 512 context features for its own rows; the softmax weights
//     exp(e - m) of the 8 rows are computed by 8 lanes and broadcast; the 8 warps' partial contexts and weight
//     sums meet once per image segment in shared memory (fixed order: bit-reproducible);
//   * a CTA that owns a whole image (grid == NI) normalises in place: no publish / counter / merge.
__device__ __forceinline__ float warp_reduce8(const float (&a)[8], int lane) {
    // returns, in every lane, the all-lane sum of a[lane >> 2]
    const bool u4 = (lane & 16) != 0, u3 = (lane & 8) != 0, u2 = (lane & 4) != 0;
    float b[4], c2[2];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float mine = u4 ? a[i + 4] : a[i], theirs = u4 ? a[i] : a[i + 4];
        b[i] = mine + __shfl_xor_sync(0xffffffffu, theirs, 16);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float mine = u3 ? b[i + 2] : b[i], theirs = u3 ? b[i] : b[i + 2];
        c2[i] = mine + __shfl_xor_sync(0xffffffffu, theirs, 8);
    }
    const float mine = u2 ? c2[1] : c2[0], theirs = u2 ? c2[0] : c2[1];
    float d = mine + __shfl_xor_sync(0xffffffffu, theirs, 4);
    d += __shfl_xor_sync(0xffffffffu, d, 2);
    d += __shfl_xor_sync(0xffffffffu, d, 1);
    return d;
}

// Wait until use `round` of ring slot `s` has landed.  Successive occupants of a slot belong to DIFFERENT warps
// here, and an mbarrier wait only distinguishes the current phase from the one before it: a warp that ran ahead
// (bulk copies may complete out of order) could otherwise mistake "the previous occupant has not even landed"
// for "my chunk is here".  Waiting first for the previous occupant's release (which the producer needs as well
// before it issues this chunk) pins the phase the second wait refers to.  That first wait cannot be fooled in
// turn: this warp has consumed chunk id-8, whose producer lane had issued chunk id-nslots before it (same lane,
// in order, because nslots is even and > 8), which required the release of chunk id-2*nslots.
__device__ __forceinline__ void att_wpc_wait(uint64_t* full, uint64_t* empty, int s, int round) {
    if (round > 0) mbar_wait(&empty[s], (uint32_t)(round - 1) & 1u);
    mbar_wait(&full[s], (uint32_t)round & 1u);
}

template <int G>
__global__ void __launch_bounds__(10 * 32, 1) att_wpc_kernel(const __grid_constant__ AttParams p) {
    constexpr int NW = 8, NT = NW * 32, RW = 512, CR = 8, RW4 = RW / 4;
    extern __shared__ __align__(1024) uint8_t smem[];
    // layout: [slots][full, empty barriers][w_s G*Lp][misc 64][zred NW*G*512]
    uint8_t* slots = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.nslots * p.slot_bytes);
    uint64_t* empty = full + p.nslots;
    const int Lp = (p.L + 3) & ~3;
    float* w_s = reinterpret_cast<float*>(empty + p.nslots);   // logits of the current segment
    float* misc = w_s + (size_t)G * Lp;                         // [NW][G] weight sums, flag at [48]
    float* zred = misc + 64;                                    // [NW][G][512] partial contexts

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int P = gridDim.x, c = blockIdx.x;
    const int L = p.L;
    const long long NR = (long long)p.NI * L;
    const int r_begin = att_rbegin(NR, P, c), r_end = att_rbegin(NR, P, c + 1);

    if (threadIdx.x == 0) {
        trace_stamp(p.dbg, 0);
        tl_begin(p.tl);
        for (int s = 0; s < p.nslots; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= NW) {
        // ============================ producers ============================
        // Two producer warps (one lane each) take the even / odd chunks, so that issuing a chunk (wait for the
        // slot, arm the barrier, bulk copy) is not a single serial chain.  T1 and ctx do not change while a
        // caption is decoded: the ring is filled before the predecessor kernel has finished (programmatic
        // dependent launch); only the consumers wait for it.
        if (lane == 0) {
            const int pw = warp - NW;                           // 0 or 1
            const uint64_t pol_t = l2_policy(p.l2_t), pol_c = l2_policy(p.l2_ctx);
            int idx = 0;                                        // chunk counter (all chunks)
            int s = 0;                                          // its ring slot and the use count of that slot
            uint32_t round = 0;
            for (int seg0 = r_begin; seg0 < r_end;) {
                const int img = seg0 / L;
                const int seg1 = min(r_end, (img + 1) * L);
                for (int pass = 0; pass < 2; ++pass) {
                    const float* src = pass == 0 ? p.T : p.ctx;
                    const int pol_k = pass == 0 ? p.l2_t : p.l2_ctx;
                    const uint64_t pol = pass == 0 ? pol_t : pol_c;
                    for (int r = seg0; r < seg1; r += CR, ++idx) {
                        if ((idx & 1) == pw) {
                            const int n = min(CR, seg1 - r);
                            mbar_wait(&empty[s], (round & 1u) ^ 1u);
                            const uint32_t bytes = (uint32_t)n * RW * 4u;
                            mbar_arrive_expect_tx(&full[s], bytes);
                            tma_bulk_g2s_hint(slots + (size_t)s * p.slot_bytes, src + (size_t)r * RW, bytes, &full[s], pol_k, pol);
                        }
                        if (++s == p.nslots) { s = 0; ++round; }
                    }
                }
                seg0 = seg1;
            }
            // (only this lane: a blocking wait issued by the idle lanes would stall the whole warp, loop included)
            if (p.pdl) { pdl_wait(); pdl_launch_dependents(); }
        }
        return;
    }

    // ============================== consumers ==============================
    const int ct = threadIdx.x;  // 0..255
    float4 wreg[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) wreg[k] = __ldg(reinterpret_cast<const float4*>(p.vec) + lane + 32 * k);
    // q / the fed words come from earlier kernels of the step; with `nowait` the immediate predecessor produced
    // none of them (and everything older is complete, see pdl_wait), so this kernel runs beside it
    if (p.pdl) { if (!p.nowait) pdl_wait(); pdl_launch_dependents(); }
    if (p.qflag) {   // q comes from a phase of the predecessor launch, which is still running: wait for that phase only
        if (lane == 0) { wait_counter(p.qflag, p.qtarget, "attention: state branch of the running dense launch"); __threadfence(); }
        __syncwarp();
    }
    if (threadIdx.x == 0) tl_go(p.tl);
    if (p.emb_pa) att_pack_embedding(p, c * NT + ct, P * NT, G);
    if (ct == 0) trace_stamp(p.dbg, 1);

    // this warp's next chunk is number `mine` (chunks idx, idx+1, ... go to warps idx % 8, ...); its ring slot and
    // the use count of that slot advance by 8 chunks at a time without divisions
    int idx = 0;
    int ms = warp % p.nslots;
    uint32_t mround = (uint32_t)(warp / p.nslots);
    bool first_seg = true;
    for (int seg0 = r_begin; seg0 < r_end;) {
        const int img = seg0 / L;
        const int seg1 = min(r_end, (img + 1) * L);
        const int nseg = seg1 - seg0;
        const int nch = (nseg + CR - 1) / CR;
        float4 qreg[G][4];
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                qreg[g][k] = p.q ? __ldcg(reinterpret_cast<const float4*>(p.q + ((size_t)img * G + g) * RW) + lane + 32 * k)
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
        if (!first_seg) named_bar_sync(1, NT);      // previous segment's w_s / zred fully consumed

        // ---- pass 1: logits of this warp's chunks
        for (int ci = ((warp - idx) % NW + NW) % NW; ci < nch; ci += NW) {
            const int s = ms;
            att_wpc_wait(full, empty, s, (int)mround);
            ms += NW;
            while (ms >= p.nslots) { ms -= p.nslots; ++mround; }
            if (ct == 0 && first_seg && ci < NW) trace_stamp(p.dbg, 2);
            const float4* buf = reinterpret_cast<const float4*>(slots + (size_t)s * p.slot_bytes);
            const int n = min(CR, nseg - ci * CR);
            float acc[G][CR];
#pragma unroll
            for (int i = 0; i < CR; ++i) {
#pragma unroll
                for (int g = 0; g < G; ++g) acc[g][i] = 0.f;
                if (i < n) {
                    float4 t[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) t[k] = buf[i * RW4 + lane + 32 * k];
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        float a0 = 0.f, a1 = 0.f;
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const float4 w = wreg[k], qq = qreg[g][k];
                            a0 = fmaf(w.x, t[k].x + qq.x, a0);
                            a1 = fmaf(w.y, t[k].y + qq.y, a1);
                            a0 = fmaf(w.z, t[k].z + qq.z, a0);
                            a1 = fmaf(w.w, t[k].w + qq.w, a1);
                        }
                        acc[g][i] = a0 + a1;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);     // the chunk is in registers: hand the slot back early
#pragma unroll
            for (int g = 0; g < G; ++g) {
                float v = warp_reduce8(acc[g], lane);
                const int i = lane >> 2;
                if ((lane & 3) == 0 && i < n) {
                    const int ll = ci * CR + i;              // location index within the segment
                    const int l = seg0 + ll - img * L;       // location index within the image
                    const size_t o = ((size_t)img * G + g) * L + l;
                    if (p.eadd) v += p.eadd[o];
                    p.e[o] = v;
                    w_s[g * Lp + ll] = v;
                }
            }
        }
        idx += nch;
        named_bar_sync(1, NT);
        if (ct == 0 && first_seg) trace_stamp(p.dbg, 3);

        // ---- segment-local maximum (every warp computes the same value)
        float m[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            float mm = -INFINITY;
            for (int l = lane; l < nseg; l += 32) mm = fmaxf(mm, w_s[g * Lp + l]);
            m[g] = warp_max(mm);
        }

        // ---- pass 2: un-normalised partial context of this warp's chunks; lane owns features 4*(lane+32k)..+3
        float zacc[G][16];
        float wsum[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            wsum[g] = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) zacc[g][k] = 0.f;
        }
        for (int ci = ((warp - idx) % NW + NW) % NW; ci < nch; ci += NW) {
            const int s = ms;
            const int n = min(CR, nseg - ci * CR);
            float wl[G];
#pragma unroll
            for (int g = 0; g < G; ++g) {      // weights of the chunk's rows: lanes 0..7 (before the wait: off its path)
                wl[g] = lane < n ? expf(w_s[g * Lp + ci * CR + lane] - m[g]) : 0.f;
                wsum[g] += wl[g];
            }
            att_wpc_wait(full, empty, s, (int)mround);
            ms += NW;
            while (ms >= p.nslots) { ms -= p.nslots; ++mround; }
            if (ct == 0 && first_seg && ci < NW) trace_stamp(p.dbg, 4);
            const float4* buf = reinterpret_cast<const float4*>(slots + (size_t)s * p.slot_bytes);
#pragma unroll
            for (int i = 0; i < CR; ++i) {
                float wv[G];
#pragma unroll
                for (int g = 0; g < G; ++g) wv[g] = __shfl_sync(0xffffffffu, wl[g], i);
                if (i < n) {
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const float4 x = buf[i * RW4 + lane + 32 * k];
#pragma unroll
                        for (int g = 0; g < G; ++g) {
                            zacc[g][4 * k + 0] = fmaf(wv[g], x.x, zacc[g][4 * k + 0]);
                            zacc[g][4 * k + 1] = fmaf(wv[g], x.y, zacc[g][4 * k + 1]);
                            zacc[g][4 * k + 2] = fmaf(wv[g], x.z, zacc[g][4 * k + 2]);
                            zacc[g][4 * k + 3] = fmaf(wv[g], x.w, zacc[g][4 * k + 3]);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        idx += nch;
        // ---- the 8 warps' partials meet in shared memory
#pragma unroll
        for (int g = 0; g < G; ++g) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
                *reinterpret_cast<float4*>(zred + ((size_t)(warp * G + g) * RW) + 4 * (lane + 32 * k)) =
                    make_float4(zacc[g][4 * k], zacc[g][4 * k + 1], zacc[g][4 * k + 2], zacc[g][4 * k + 3]);
            const float ws = warp_sum(wsum[g]);
            if (lane == 0) misc[warp * G + g] = ws;
        }
        named_bar_sync(1, NT);
        if (ct == 0 && first_seg) trace_stamp(p.dbg, 5);
        float zsum[G][2], ssum[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            ssum[g] = 0.f;
            zsum[g][0] = zsum[g][1] = 0.f;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                ssum[g] += misc[w * G + g];
                zsum[g][0] += zred[(size_t)(w * G + g) * RW + ct];
                zsum[g][1] += zred[(size_t)(w * G + g) * RW + ct + NT];
            }
        }

        // contributors of this image: CTAs c_lo..c_hi whose row ranges overlap [img*L, (img+1)*L)
        int c_lo = (int)(((long long)img * L * P) / NR);
        while (c_lo + 1 < P && att_rbegin(NR, P, c_lo + 1) <= img * L) ++c_lo;
        while (c_lo > 0 && att_rbegin(NR, P, c_lo) > img * L) --c_lo;
        int c_hi = (int)((((long long)(img + 1) * L - 1) * P) / NR);
        while (c_hi + 1 < P && att_rbegin(NR, P, c_hi + 1) <= (img + 1) * L - 1) ++c_hi;
        while (c_hi > 0 && att_rbegin(NR, P, c_hi) > (img + 1) * L - 1) --c_hi;
        const int nc = c_hi - c_lo + 1;
        if (ct == 0 && seg1 == r_end) tl_main_done(p.tl);
        if (nc == 1) {
            // ---- this CTA saw the whole image: normalise in place
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float inv = 1.0f / ssum[g];
#pragma unroll
                for (int kk = 0; kk < 2; ++kk) {
                    const int d = ct + NT * kk;
                    const float zv = zsum[g][kk] * inv;
                    p.z[((size_t)img * G + g) * RW + d] = zv;
                    if (p.pa_z) pa_store(p.pa_z, p.pa_mode, p.pa_row_tile, RW >> 6, img * G + g, d, zv);
                }
                for (int l = ct; l < L; l += NT) p.alpha[((size_t)img * G + g) * L + l] = expf(w_s[g * Lp + l] - m[g]) * inv;
            }
        } else {
            // ---- publish the partial, the last CTA of the image merges
            const int slot_id = img - r_begin / L;                // ordinal of this segment within the CTA
            float* part = p.part + ((size_t)c * p.segmax + slot_id) * G * (RW + 2);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                part[(size_t)g * (RW + 2) + ct] = zsum[g][0];
                part[(size_t)g * (RW + 2) + ct + NT] = zsum[g][1];
                if (ct == 0) { part[(size_t)g * (RW + 2) + RW] = m[g]; part[(size_t)g * (RW + 2) + RW + 1] = ssum[g]; }
            }
            named_bar_sync(1, NT);                                // every thread's partial stores are ordered before ...
            unsigned* flag = reinterpret_cast<unsigned*>(misc + 48);
            if (ct == 0) {
                __threadfence();                                  // ... this (cumulative) release
                *flag = atomicAdd(p.rowcnt + img, 1u) == (unsigned)(nc - 1) ? 1u : 0u;
            }
            named_bar_sync(1, NT);
            if (ct == 0 && first_seg) trace_stamp(p.dbg, 6);
            if (*flag) {
                __threadfence();
                if (ct == 0) p.rowcnt[img] = 0u;                  // ready for the next launch
#pragma unroll 1
                for (int g = 0; g < G; ++g) {
                    const float* er = p.e + ((size_t)img * G + g) * L;
                    // (max, sum) and this thread's two features of every contributor: all loads of a batch of 4
                    // contributors in flight together
                    float M = -INFINITY;
                    for (int j = 0; j < nc; ++j) {
                        const int cc = c_lo + j;
                        const int sid = img - att_rbegin(NR, P, cc) / L;
                        M = fmaxf(M, __ldcg(p.part + (((size_t)cc * p.segmax + sid) * G + g) * (RW + 2) + RW));
                    }
                    float S = 0.f, z0 = 0.f, z1 = 0.f;
                    for (int j0 = 0; j0 < nc; j0 += 4) {
                        float v0[4], v1[4], ms[4], ss[4];
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj) {
                            const int cc = c_lo + min(j0 + jj, nc - 1);
                            const int sid = img - att_rbegin(NR, P, cc) / L;
                            const float* pp = p.part + (((size_t)cc * p.segmax + sid) * G + g) * (RW + 2);
                            ms[jj] = __ldcg(pp + RW);
                            ss[jj] = __ldcg(pp + RW + 1);
                            v0[jj] = __ldcg(pp + ct);
                            v1[jj] = __ldcg(pp + ct + NT);
                        }
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj) {
                            if (j0 + jj < nc) {
                                const float sc = expf(ms[jj] - M);
                                S = fmaf(ss[jj], sc, S);
                                z0 = fmaf(v0[jj], sc, z0);
                                z1 = fmaf(v1[jj], sc, z1);
                            }
                        }
                    }
                    const float inv = 1.0f / S;
                    p.z[((size_t)img * G + g) * RW + ct] = z0 * inv;
                    p.z[((size_t)img * G + g) * RW + ct + NT] = z1 * inv;
                    if (p.pa_z) {
                        pa_store(p.pa_z, p.pa_mode, p.pa_row_tile, RW >> 6, img * G + g, ct, z0 * inv);
                        pa_store(p.pa_z, p.pa_mode, p.pa_row_tile, RW >> 6, img * G + g, ct + NT, z1 * inv);
                    }
                    for (int l = ct; l < L; l += NT) p.alpha[((size_t)img * G + g) * L + l] = expf(__ldcg(er + l) - M) * inv;
                }
            }
        }
        first_seg = false;
        seg0 = seg1;
    }
    if (ct == 0) { trace_stamp(p.dbg, 7); tl_end(p.tl); }
    if (p.pdl && p.nowait) pdl_wait();   // do not complete before the predecessor: later kernels rely on the chain
}

size_t att_smem_bytes(const AttParams& p) {
    const int Lp = (p.L + 3) & ~3;
    if (p.wpc)
        return (size_t)p.nslots * p.slot_bytes + 2 * (size_t)p.nslots * 8 + 4 * ((size_t)p.G * Lp + 64 + (size_t)8 * p.G * 512);
    return (size_t)p.nslots * p.slot_bytes + 2 * (size_t)p.nslots * 8 +
           4 * ((size_t)p.RL + (size_t)p.G * p.RL + (size_t)p.G * Lp + 64);
}

// Fill in chunking / ring parameters from the device limits.  Returns false if the shape is unsupported.
bool att_plan(AttParams& p, int smem_optin, int num_sms) {
    // occ CTAs per SM: each CTA gets 1/occ of the shared memory (a shorter ring) and the SM holds occ x 8
    // consumer warps, which hides the shared-memory / shuffle latencies of the two passes
    const int occ = (p.occ == 2 && p.G == 1) ? 2 : 1;
    p.occ = occ;
    smem_optin = occ == 2 ? (smem_optin - 2048) / 2 : smem_optin;
    num_sms *= occ;
    if (p.G < 1 || p.G > 4 || p.L < 1 || (p.D % 4) || (p.RL % 4) || p.D > kAttMaxDPerThread * 8 * 32) return false;
    if (p.warps != 16 || p.G != 1 || p.occ == 2) p.warps = 8;
    p.wpc = (p.wpc && p.RL == 512 && p.D == 512 && occ == 1) ? 1 : 0;   // warp-per-chunk kernel (att_wpc_kernel)
    if (p.wpc) p.warps = 8;
    const int target = p.wpc ? 16 * 1024 : 32 * 1024;                       // bytes per ring slot (16 rows of 512 floats: 2 rows per warp)
    int rch = target / (p.RL * 4), cch = target / (p.D * 4);
    if (rch < 1) rch = 1;
    if (cch < 1) cch = 1;
    int slot = rch * p.RL * 4;
    if (cch * p.D * 4 > slot) slot = cch * p.D * 4;
    slot = (slot + 127) & ~127;
    p.rch = rch;
    p.cch = cch;
    p.slot_bytes = slot;
    AttParams t = p;
    t.nslots = 0;
    const size_t fixed = att_smem_bytes(t) + 64;
    if ((size_t)smem_optin < fixed + 2 * (size_t)slot) return false;
    int n = (int)(((size_t)smem_optin - fixed) / ((size_t)slot + 16));
    if (n > (p.wpc ? 24 : 16)) n = p.wpc ? 24 : 16;
    // warp-per-chunk kernel: an even ring, so that the successive occupants of a slot come from the same one of
    // its two producer lanes (each issues its chunks in order), which is what att_wpc_wait's argument needs
    if (p.wpc) n &= ~1;
    p.nslots = n;
    const long long NR = (long long)p.NI * p.L;
    p.grid = (int)(NR < num_sms ? NR : num_sms);
    if (p.NI <= num_sms) {
        // k CTAs per image: every CTA owns one segment of exactly one image (one softmax-statistics pass,
        // one publish) and every image has exactly k contributors; costs at most (1 - NI*k/#SMs) of the SMs
        int k = num_sms / p.NI;
        if (k > p.L) k = p.L;
        if (k >= 1 && (double)(p.NI * k) >= 0.8 * p.grid) p.grid = p.NI * k;
    }
    const int share = (int)((NR + p.grid - 1) / p.grid);
    p.segmax = share / p.L + 2;
    return n >= 2;
}

size_t att_part_floats(const AttParams& p) { return (size_t)p.grid * p.segmax * p.G * (p.D + 2); }

template <int G, int RV, int OCC, int NW>
static cudaError_t att_launch_gro(const AttParams& p, cudaStream_t st) {
    const size_t smem = att_smem_bytes(p);
    cudaError_t e = cudaFuncSetAttribute(att_fused_kernel<G, RV, OCC, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.grid);
    cfg.blockDim = dim3((NW + 1) * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = p.pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, att_fused_kernel<G, RV, OCC, NW>, p);
}
template <int G, int RV>
static cudaError_t att_launch_gr(const AttParams& p, cudaStream_t st) {
    if (G == 1 && p.occ == 2) return att_launch_gro<G, RV, (G == 1 ? 2 : 1), 8>(p, st);
    if (G == 1 && p.warps == 16) return att_launch_gro<G, RV, 1, (G == 1 ? 16 : 8)>(p, st);
    return att_launch_gro<G, RV, 1, 8>(p, st);
}

template <int G>
static cudaError_t att_launch_g(const AttParams& p, cudaStream_t st) {
    // register-resident w2/q when a row is exactly 512 floats (dim_attend_layer = 512, the reference default)
    if (p.RL == 512) return att_launch_gr<G, 4>(p, st);
    return att_launch_gr<G, 0>(p, st);
}

template <int G>
static cudaError_t att_launch_wpc(const AttParams& p, cudaStream_t st) {
    const size_t smem = att_smem_bytes(p);
    cudaError_t e = cudaFuncSetAttribute(att_wpc_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(p.grid);
    cfg.blockDim = dim3(10 * 32);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = p.pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, att_wpc_kernel<G>, p);
}

cudaError_t att_launch(const AttParams& p, cudaStream_t st) {
    if (p.wpc) {
        switch (p.G) {
            case 1: return att_launch_wpc<1>(p, st);
            case 2: return att_launch_wpc<2>(p, st);
            case 3: return att_launch_wpc<3>(p, st);
            case 4: return att_launch_wpc<4>(p, st);
        }
        return cudaErrorInvalidValue;
    }
    switch (p.G) {
        case 1: return att_launch_g<1>(p, st);
        case 2: return att_launch_g<2>(p, st);
        case 3: return att_launch_g<3>(p, st);
        case 4: return att_launch_g<4>(p, st);
    }
    return cudaErrorInvalidValue;
}

// mean over the L locations (model.py:240): out[i, d] = (1/L) sum_l ctx[i, l, d]
// One block per (image, 128-feature slab): 8 row groups x 32 float4 columns, rows summed in location order per
// group and the 8 groups added in fixed order (bit-reproducible); loads of 4 rows are in flight per thread.
// PACK: the same pass also writes every row in the packed-activation layout the context projection (attend/fc_1a)
// fetches by TMA (SURVEY section 8 row f3: one pass over the conv features for the mean AND the projection operand;
// the summation order — and with it the mean, bit for bit — is that of the plain kernel).
template <bool PACK>
__global__ void __launch_bounds__(256) ctx_mean_kernel(const float* __restrict__ ctx, float* __restrict__ out, int L, int D,
                                                       uint8_t* __restrict__ pa, int row_tile, int mode) {
    constexpr int RG = 8, C4 = 32;
    __shared__ float4 red[RG][C4];
    const int i = blockIdx.y;
    const int c4 = threadIdx.x % C4, rg = threadIdx.x / C4;
    const int d = blockIdx.x * (4 * C4) + 4 * c4;
    const int kblocks = D >> 6;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (d < D) {
        const float* p = ctx + (size_t)i * L * D + d;
        int l = rg;
        for (; l + 3 * RG < L; l += 4 * RG) {
            const float4 a = *reinterpret_cast<const float4*>(p + (size_t)l * D);
            const float4 b = *reinterpret_cast<const float4*>(p + (size_t)(l + RG) * D);
            const float4 c = *reinterpret_cast<const float4*>(p + (size_t)(l + 2 * RG) * D);
            const float4 e = *reinterpret_cast<const float4*>(p + (size_t)(l + 3 * RG) * D);
            s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
            s.x += b.x; s.y += b.y; s.z += b.z; s.w += b.w;
            s.x += c.x; s.y += c.y; s.z += c.z; s.w += c.w;
            s.x += e.x; s.y += e.y; s.z += e.z; s.w += e.w;
            if (PACK) {
                pa_store4(pa, mode, row_tile, kblocks, i * L + l, d, &a.x);
                pa_store4(pa, mode, row_tile, kblocks, i * L + l + RG, d, &b.x);
                pa_store4(pa, mode, row_tile, kblocks, i * L + l + 2 * RG, d, &c.x);
                pa_store4(pa, mode, row_tile, kblocks, i * L + l + 3 * RG, d, &e.x);
            }
        }
        for (; l < L; l += RG) {
            const float4 a = *reinterpret_cast<const float4*>(p + (size_t)l * D);
            s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
            if (PACK) pa_store4(pa, mode, row_tile, kblocks, i * L + l, d, &a.x);
        }
    }
    red[rg][c4] = s;
    __syncthreads();
    if (rg == 0 && d < D) {
        float4 t = red[0][c4];
#pragma unroll
        for (int r = 1; r < RG; ++r) { t.x += red[r][c4].x; t.y += red[r][c4].y; t.z += red[r][c4].z; t.w += red[r][c4].w; }
        const float inv = 1.0f / (float)L;
        *reinterpret_cast<float4*>(out + (size_t)i * D + d) = make_float4(t.x * inv, t.y * inv, t.z * inv, t.w * inv);
    }
}

cudaError_t ctx_mean_launch(const float* ctx, float* out, int NI, int L, int D, cudaStream_t st) {
    dim3 grid((D + 127) / 128, NI);
    ctx_mean_kernel<false><<<grid, 256, 0, st>>>(ctx, out, L, D, nullptr, 0, 0);
    return cudaGetLastError();
}

// mean + packed rows (row tile `row_tile`, D % 64 == 0) in one pass; rows beyond NI * L of the last row tile are not
// written (they only feed output rows the projection never stores)
cudaError_t ctx_mean_pack_launch(const float* ctx, float* out, uint8_t* pa, int row_tile, int layout_mode, int NI, int L, int D,
                                 cudaStream_t st) {
    dim3 grid((D + 127) / 128, NI);
    ctx_mean_kernel<true><<<grid, 256, 0, st>>>(ctx, out, L, D, pa, row_tile, layout_mode);
    return cudaGetLastError();
}

}  // namespace sat
