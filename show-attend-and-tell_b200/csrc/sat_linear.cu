// sat_linear.cu — small-batch dense layers on Hopper tensor cores (wgmma).
//
// Computes, for up to 4 grouped problems per launch,
//     out[b, n] = epilogue( sum_k X[b, k] * W[k, n] + bias[n] )
// which is tf.layers.dense (utils/nn.py:85-105) and the LSTMCell matmul
// (model.py:276-279) of the reference.  The batch is small (4..384) and the
// weights are large, so every problem is bound by streaming W once from HBM.
//
// Formulation ("swap-AB"): the weight matrix is the MMA M operand — a CTA owns
// 128 output features x a K-range — and the batch rows are the MMA N operand
// (16..256).  fp32 parity (1e-3 vs the fp32 reference) is kept with a
// split-precision product: W and X are each held as bf16 hi + bf16 lo
// (w = hi + lo to 16 mantissa bits) and three MMAs are issued per K-step,
//     acc += Whi*Xhi + Wlo*Xhi + Whi*Xlo        (fp32 accumulation in registers).
// W is repacked once at sat_set_weight() into the exact shared-memory image of
// the wgmma K-major operand (hi and lo halves adjacent: 4 bytes per weight, the
// same HBM traffic as the fp32 original), so a pipeline stage is filled by ONE
// 32 KB cp.async.bulk (TMA) per CTA.  X (tiny) arrives the same way when its
// producer kernel wrote it as a "packed activation" (x_mode 2, the steady state
// of the decode loop); otherwise all CTAs convert it once in a cooperative
// pre-pass (x_mode 1) or producer warps convert it per stage (x_mode 0).  The
// concats of model.py:277,283-286 are never materialised: the K range of a
// problem is a list of segments.
// Split-K: the S CTAs of a tile are one thread-block cluster; partial tiles meet
// in distributed shared memory and are summed in fixed rank order
// (bit-reproducible), then the fused epilogue runs (bias / tanh / LSTM gates /
// greedy argmax of the vocabulary layer / packed copy for the next layer).
//
// Warp roles (320 threads): warps 0..7 = two warpgroups that issue the wgmma
// (warpgroup g: outputs [64g, 64g + 64) of the tile, accumulator in registers),
// convert X (modes 0/1) and run the epilogue; warp 8 = TMA producer (one lane),
// warp 9 = activation TMA stream (x_mode 2).
//
// Launch chaining: every launch carries the programmatic-dependent-launch attribute.  The TMA lane fills its
// first stages with weights before griddepcontrol.wait; launch_dependents is called only after the wait (so a
// kernel never starts before the predecessor of its predecessor has completed).  While the first stages are in
// flight, the consumer warps run the (short) epilogue once without side effects to pull its code into the
// instruction caches: epilogues execute once per launch from cold caches, and that costs microseconds.
// The vocabulary layer's fused arg-max ends in a grid-wide rendezvous of its one-wave launch; CTA i then merges
// row i's candidates and packs the embedding row of the chosen word for the next LSTM / decode layers.
// The training step (sat_train.cu) uses the same kernel through sat_dense_packed(): packed operands of either
// role, an accumulate epilogue, weights that may come from the preceding kernel (w_dynamic).
#include "sat_common.cuh"
#include "sat_linear.cuh"
#include "sat_linear_dev.cuh"

namespace sat {

// (split_bf16x8, lstm_gates: sat_linear_dev.cuh)
// fp32 source of the 8 consecutive K elements starting at k0 of activation row b (zeros outside).
__device__ __forceinline__ void load_x8(const LinProblem& P, int b, int k0, float4& a, float4& c) {
    a = make_float4(0.f, 0.f, 0.f, 0.f);
    c = a;
    if (b >= P.rows || k0 >= P.K) return;
    int start = 0;
#pragma unroll
    for (int s = 0; s < kMaxSeg; ++s) {
        if (s < P.nseg) {
            const LinSeg& sg = P.seg[s];
            if (k0 >= start && k0 < start + sg.width) {
                const int row = sg.gather ? sg.gather[b] : b / sg.row_div;
                const float4* p = reinterpret_cast<const float4*>(sg.ptr + (size_t)row * sg.ld + (k0 - start));
                a = p[0];
                c = p[1];
            }
            start += sg.width;
        }
    }
}

struct EpiCtx {
    const LinProblem* P;
    int n_tile, row0, rows_here;
};

// generic epilogues on one value
__device__ __forceinline__ float epi_scalar(const LinProblem& P, float acc, int n) {
    if (P.epi == kEpiNone) return acc;
    acc += P.bias[n];
    return P.epi == kEpiBiasTanh ? act_tanh(acc) : acc;
}

// ------------------------------------------------------------- wgmma kernel
struct XChunk {
    float4 a[2], c[2];
};

// NT = (row tile of the launch) / 16: the accumulator fragments per warpgroup
// WP: the fused arg-max also produces the probability of the word fed to the next step (LinProblem::am_probs); a
// separate instance, so that launches without it run the code they ran before
// SMP: sampling — the arg-max ranks logit / temperature + Gumbel noise (LinProblem::smp); instances of their own,
// with WP (the sampled word's probability) or without it (no softmax partials: nothing but the draw is added)
template <int NT, bool WP, bool SMP = false>
__global__ void __launch_bounds__(kLinThreads, 1) lin_mma_kernel(const __grid_constant__ LinLaunch L) {
    constexpr bool SWP = SMP && WP;   // sampling with word probabilities: the raw logits ride beside the keys
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // control block: barriers etc. live in the first 1024 bytes
    uint64_t* full_w = reinterpret_cast<uint64_t*>(smem_raw);  // [stages]
    uint64_t* full_x = full_w + 8;
    uint64_t* empty = full_x + 8;
    uint8_t* stage_base = smem_raw + 1024;
    const bool xpa = L.x_mode == 2;   // every X segment was packed by its producer kernel
    const bool xpre = L.x_mode == 1;  // activations packed by a cooperative pre-pass of this launch
    const bool xtma = xpa || xpre;    // X stages are fetched by TMA

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // ---- which problem / tile / split am I?
    int pi = 0;
#pragma unroll
    for (int i = 1; i < kMaxProb; ++i)
        if (i < L.nprob && (int)blockIdx.x >= L.p[i].cta_begin) pi = i;
    const LinProblem& P = L.p[pi];
    const int local = blockIdx.x - P.cta_begin;
    const int split = local % P.splits;
    const int t = local / P.splits;
    const int n_tile = t % P.n_tiles;
    const int rt = t / P.n_tiles;
    const int row0 = rt * P.row_tile;
    const int N = P.row_tile;
    const int kb0 = (int)(((long long)P.k_blocks * split) / P.splits);
    const int kb1 = (int)(((long long)P.k_blocks * (split + 1)) / P.splits);
    const int nkb = kb1 - kb0;
    const int S = L.stages;
    const int mode = L.layout_mode;
    const uint32_t x_half_bytes = (uint32_t)N * kBK * 2;
    const uint32_t stage_bytes = kWStageBytes + 2 * x_half_bytes;
    constexpr int kTmaWarp = kLinProducers / 32;   // warp 8
    constexpr int kXWarp = kTmaWarp + 1;           // warp 9

    // ---- one-time setup
    if (threadIdx.x == 0) {
        trace_stamp(L.dbg, 0);
        tl_begin(L.tl);
        for (int s = 0; s < S; ++s) {
            mbar_init(&full_w[s], 1);
            mbar_init(&full_x[s], 1);
            mbar_init(&empty[s], kLinProducers / 32);   // one arrival per consumer warp once its MMAs are complete
        }
        fence_mbar_init();
    }
    // grid-barrier generation must be sampled before this CTA can possibly arrive on it
    unsigned gen0 = 0;
    if (xpre && threadIdx.x == kTmaWarp * 32) gen0 = ld_acquire_gpu(P.xbar + 1);
    __syncthreads();
    const uint32_t x_stage_bytes = 2 * x_half_bytes;
    float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);   // epilogue warps: bias of this thread's 4 outputs
    // Programmatic dependent launch: everything above touched no global memory.  The weights are immutable
    // while a step runs, so the TMA lane may fetch them before the predecessor has finished; every other
    // global access (activations, outputs) waits for the predecessor.
    // launch_dependents is issued only AFTER the wait, which gives every kernel of the chain the invariant
    // "when I start, everything before my immediate predecessor is complete and visible".
    // Every warp but the TMA warp waits here (the TMA lane waits later): a blocking wait issued by the idle lanes of
    // the TMA warp would stall the TMA lane's weight prefetch with them.
    if (L.pdl && warp != kTmaWarp) { pdl_wait(); pdl_launch_dependents(); }

    // ---- TMA production when every operand arrives packed (x_mode 2: the steady state of loops and of the training
    // step's products).  Two warps: warp 8 streams the weight halves of the stages (immutable: it starts before the
    // dependency wait), warp 9 streams the activation halves — the two wait -> arm -> issue chains overlap, and this production paces the tile.  Each is a WHOLE warp running the loop
    // converged with one elected lane issuing (see elect_one in sat_common.cuh): issued from `if (lane == 0)` code each
    // bulk copy paid register->uniform moves and an indexed walk over the launch descriptor.  Running cursors: no divisions.
    auto stream_half = [&](const bool wside) {
        const uint64_t wpol = l2_policy(P.l2_w);
        const int l2w = wside ? P.l2_w : 0;
        const uint32_t stage0 = smem_u32(stage_base) + (wside ? 0u : (uint32_t)kWStageBytes);
        const uint32_t bar0 = smem_u32(wside ? full_w : full_x);
        const uint32_t bytes = wside ? (uint32_t)kWStageBytes : x_stage_bytes;
        const uint8_t* ptr;
        int sg = 0, seg_left = nkb + 1;        // (weights: one contiguous run)
        if (wside) {
            ptr = P.wpack + ((size_t)n_tile * P.k_blocks + kb0) * kWStageBytes;
        } else {
            int kb = kb0;                       // the K block lives in the packed activation of the segment that covers it
            while (sg + 1 < P.nseg && kb >= (P.seg[sg].width >> 6)) { kb -= P.seg[sg].width >> 6; ++sg; }
            ptr = P.seg[sg].pa + ((size_t)rt * (P.seg[sg].width >> 6) + kb) * x_stage_bytes;
            seg_left = (P.seg[sg].width >> 6) - kb;
        }
        int st = 0;
        uint32_t par = 1u;                      // parity of empty[st] that means "free" (fresh barrier: the first pass is free)
        if (wside && L.pdl && L.w_dynamic) pdl_wait();   // the weight operand was written by the preceding kernel
        for (int it = 0; it < nkb; ++it) {
            if (it >= S) mbar_wait_mma(&empty[st], par);
            if (elect_one()) {
                const uint32_t bar = bar0 + 8u * (uint32_t)st;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
                const uint32_t dst = stage0 + (uint32_t)st * stage_bytes;
                if (l2w == 0)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                                 "l"(ptr), "r"(bytes), "r"(bar) : "memory");
                else
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
                                 "l"(ptr), "r"(bytes), "r"(bar), "l"(wpol) : "memory");
                // (option) the rest of this CTA's weight stream: into L2 while the predecessor drains
                if (wside && L.pdl && L.l2_prefetch && it + 1 == (nkb < S ? nkb : S))
                    for (int j = it + 1; j < nkb; ++j) prefetch_l2_bulk(ptr + (size_t)(j - it) * kWStageBytes, kWStageBytes);
            }
            ptr += bytes;
            if (++st == S) { st = 0; if (it >= S) par ^= 1u; else par = 0u; }
            if (--seg_left == 0 && !wside && sg + 1 < P.nseg) {
                ++sg;
                ptr = P.seg[sg].pa + (size_t)rt * (P.seg[sg].width >> 6) * x_stage_bytes;
                seg_left = P.seg[sg].width >> 6;
            }
        }
    };
    if (warp == kTmaWarp && xpa) {
        stream_half(true);
    } else if (warp == kXWarp) {
        if (xpa) {   // (this warp waited for the predecessor above)
            if (lane == 0) tl_go(L.tl);
            stream_half(false);
        }
    } else if (warp == kTmaWarp) {
        // ===================== TMA producer: one 32 KB bulk copy per stage =====================
        if (lane == 0) {
            const uint8_t* src = P.wpack + ((size_t)n_tile * P.k_blocks + kb0) * kWStageBytes;
            const uint8_t* xsrc = P.xpack + ((size_t)rt * P.k_blocks + kb0) * x_stage_bytes;
            const uint64_t wpol = l2_policy(P.l2_w);
            auto load_w = [&](int it) {
                const int s = it % S;
                mbar_arrive_expect_tx(&full_w[s], kWStageBytes);
                tma_bulk_g2s_hint(stage_base + (size_t)s * stage_bytes, src + (size_t)it * kWStageBytes, kWStageBytes,
                                  &full_w[s], P.l2_w, wpol);
            };
            auto load_x = [&](int it) {
                const int s = it % S;
                const uint8_t* xs = xsrc + (size_t)it * x_stage_bytes;
                if (xpa) {  // K block kb0+it lives in the packed activation of the segment that covers it
                    int kb = kb0 + it, sg = 0;
                    while (sg + 1 < P.nseg && kb >= (P.seg[sg].width >> 6)) { kb -= P.seg[sg].width >> 6; ++sg; }
                    xs = P.seg[sg].pa + ((size_t)rt * (P.seg[sg].width >> 6) + kb) * x_stage_bytes;
                }
                mbar_arrive_expect_tx(&full_x[s], x_stage_bytes);
                tma_bulk_g2s(stage_base + (size_t)s * stage_bytes + kWStageBytes, xs, x_stage_bytes, &full_x[s]);
            };
            const int pre = nkb < S ? nkb : S;
            if (!L.pdl) tl_go(L.tl);
            if (L.pdl) {
                if (L.w_dynamic) pdl_wait();          // (a second wait further down returns at once)
                for (int it = 0; it < pre; ++it) load_w(it);
                // the rest of this CTA's weight stream: into L2 while the predecessor drains
                if (L.l2_prefetch)
                    for (int it = pre; it < nkb; ++it) prefetch_l2_bulk(src + (size_t)it * kWStageBytes, kWStageBytes);
                pdl_wait();
                pdl_launch_dependents();
                tl_go(L.tl);
                if (xpa) for (int it = 0; it < pre; ++it) load_x(it);
            }
            if (xpa) {
                if (!L.pdl) for (int it = 0; it < pre; ++it) { load_w(it); load_x(it); }
            } else if (xpre) {
                // weights do not depend on the activation pre-pass: fill the pipeline with W first, then
                // wait for the grid-wide pack to complete and fetch the X halves of the same stages
                if (!L.pdl) for (int it = 0; it < pre; ++it) load_w(it);
                const long long t0 = clock64();
                while (ld_acquire_gpu(P.xbar + 1) == gen0) {
                    if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) __trap();   // activation pack barrier
                }
                fence_proxy_async_global();
                trace_stamp(L.dbg, 3);
                for (int it = 0; it < pre; ++it) load_x(it);
            }
            for (int it = (xtma || L.pdl) ? pre : 0; it < nkb; ++it) {
                const int s = it % S;
                const uint32_t ph = (uint32_t)(it / S) & 1u;
                mbar_wait_mma(&empty[s], ph ^ 1u);
                load_w(it);
                if (xtma) load_x(it);
            }
        }
    } else if (warp < kTmaWarp) {
        // ===================== consumer warpgroups (warps 0..7): X producers, MMA, epilogue =====================
        // The fp32 sources of X are L2 resident; their latency is hidden by keeping the loads of the
        // NEXT chunk in flight while the current one is converted and stored.
        const int pt = threadIdx.x;  // 0..255
        if (pt == 0) trace_stamp(L.dbg, 1);
        if (xpre) {
            // ---- cooperative pre-pass: this problem's CTAs convert X (fp32 -> bf16 hi/lo MMA operand tiles) ONCE
            // into global scratch; consecutive threads take consecutive 8-element groups of a row (coalesced).
            const int kgroups = P.k_blocks * 8;
            const int utot = P.n_row_tiles * N * kgroups;
            for (int u = local * kLinProducers + pt; u < utot; u += P.cta_count * kLinProducers) {
                const int rr = u / kgroups, kgk = u - rr * kgroups;
                const int rt2 = rr / N, r = rr - rt2 * N;
                float4 a, c;
                load_x8(P, rt2 * N + r, kgk * 8, a, c);
                uint4 hi, lo;
                split_bf16x8(a, c, hi, lo);
                uint8_t* dst = P.xpack + ((size_t)rt2 * P.k_blocks + (kgk >> 3)) * x_stage_bytes +
                               mma_tile_off(mode, r, kgk & 7);
                *reinterpret_cast<uint4*>(dst) = hi;
                *reinterpret_cast<uint4*>(dst + x_half_bytes) = lo;
            }
            __threadfence();
            fence_proxy_async_global();
            named_bar_sync(1, kLinProducers);
            if (pt == 0) {  // grid barrier arrive: the last CTA opens the next generation
                trace_stamp(L.dbg, 2);
                const unsigned old = atomicAdd(P.xbar, 1u);
                if (old == (unsigned)(P.cta_count - 1)) {
                    P.xbar[0] = 0u;
                    __threadfence();
                    atomicAdd(P.xbar + 1, 1u);
                }
            }
        }
        const int units = xtma ? 0 : N * 8;  // 16-byte groups per K block (in-kernel producer mode)
        const int JC = (units + 2 * kLinProducers - 1) / (2 * kLinProducers);  // chunks (2 units/thread) per block
        const int total = xtma ? 0 : nkb * JC;
        auto load_chunk = [&](int g, XChunk& ch) {
            const int it = g / JC, jc = g - it * JC;
            const int kbase = (kb0 + it) * kBK;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int u = pt + kLinProducers * (jc * 2 + e);
                if (u < units) {
                    const int kg = u / N, r = u - kg * N;
                    load_x8(P, row0 + r, kbase + kg * 8, ch.a[e], ch.c[e]);
                }
            }
        };
        // ---- epilogue.  Code that runs once per launch is fetched cold (the instruction caches do not survive
        // the other kernels of a step), and a cold straight-line epilogue costs several microseconds on the
        // critical path.  In the TMA-fed modes these warps would wait for the first stages anyway, so they first
        // run the epilogue once "dry" (same instructions, loads from harmless addresses, no stores, no
        // synchronisation with other CTAs) purely to pull its code into the instruction caches.
        // (the bias does not depend on the accumulator: fetch it while the main loop runs)
        if (P.epi != kEpiNone && P.bias) bias4 = *reinterpret_cast<const float4*>(P.bias + n_tile * kTileN + 4 * (pt & 31));
        const int u = pt & 31;
        // problem fields used in the loops, hoisted out of (indexed) constant memory
        const int splits = P.splits, epi = P.epi, n_out = P.n_out, ldo = P.ldo, Hh = P.H;
        float* const out = P.out;
        uint8_t* const out_pa = P.out_pa;
        const float* const c_in = P.c_in;
        const int rows_here = min(N, P.rows - row0);
        float* tile_s = reinterpret_cast<float*>(stage_base);
        const uint32_t tile_addr = smem_u32(tile_s);
        const int lo = (int)(((long long)rows_here * split) / splits) * 32;
        const int hi = (int)(((long long)rows_here * (split + 1)) / splits) * 32;
        const bool do_am = P.am_key != nullptr && splits == 1;
        const int ng = n_tile * kTileN + 4 * u;          // first of this thread's 4 outputs (all rows)
        const int unit = n_tile * 32 + u;                // LSTM: the unit whose 4 gates this thread holds
        const bool vec_out = ng + 3 < n_out && (ldo & 3) == 0;
        // the row loop is skipped when the arg-max is all that is wanted from this layer
        const bool row_loop = epi == kEpiLstm || out != nullptr || out_pa != nullptr;
        unsigned long long* const am_key = do_am ? P.am_key + (size_t)(rt * P.n_tiles + n_tile) * N : nullptr;
        // arg-max layers fold the bias into the tile as it leaves the accumulator: the arg-max scan then reads
        // finished values; the row loop must not add it again
        const float* const bias_fold = (do_am && P.bias) ? P.bias + n_tile * kTileN : nullptr;
        // LSTM: c_prev of the (at most two) rows this thread finishes, fetched while the main loop runs
        float cpre[2] = {0.f, 0.f};
        if (epi == kEpiLstm && unit < Hh) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int idx = lo + pt + j * kLinProducers;
                if (idx < hi) cpre[j] = c_in[(size_t)(row0 + (idx >> 5)) * Hh + unit];
            }
        }
        // generation of the "words picked" signal, sampled before any CTA of this launch can have raised it
        const unsigned am_gen0 = (do_am && pt == 0) ? ld_acquire_gpu(P.am_ctr + 1) : 0u;
#pragma unroll 1
        // (the warm-up pass only pays for short epilogues: a long row loop warms itself)
        for (int pass = (xtma && L.warm_epilogue && (!row_loop || hi - lo <= 8 * kLinProducers)) ? 0 : 1; pass < 2; ++pass) {
            const bool dry = pass == 0;
            if (!dry) {
                // ---- main loop: per K block, both warpgroups issue their 64 x N x 64 share of the three products
                AccTile<NT> acc;
                const uint32_t stage0 = smem_u32(stage_base);
                if (xtma) {
                    int s = 0;
                    uint32_t ph = 0u;
#pragma unroll 1
                    for (int it = 0; it < nkb; ++it) {
                        mbar_wait_mma(&full_w[s], ph);
                        if (it == 0 && pt == 0) trace_stamp(L.dbg, 4);
                        mbar_wait_mma(&full_x[s], ph);
                        if (it == 0 && pt == 0) trace_stamp(L.dbg, 5);
                        mma_kblock(acc, stage0 + (uint32_t)s * stage_bytes, x_half_bytes, mode, it == 0);
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty[s]);   // frees the stage: this warp's MMAs have read it
                        if (++s == S) { s = 0; ph ^= 1u; }
                    }
                } else {
                    // X converted by these warps, one K block at a time: its stage is free (this thread's MMAs on
                    // it completed S blocks ago; with one stage, the barrier below waits for the other warpgroup)
                    XChunk cur, nxt;
                    load_chunk(0, cur);
#pragma unroll 1
                    for (int g = 0; g < total; ++g) {
                        const int it = g / JC, jc = g - it * JC;
                        const int s = it % S;
                        if (g + 1 < total) load_chunk(g + 1, nxt);
                        if (jc == 0 && S == 1 && it > 0) named_bar_sync(1, kLinProducers);
                        uint8_t* xh = stage_base + (size_t)s * stage_bytes + kWStageBytes;
                        uint8_t* xl = xh + x_half_bytes;
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int uu = pt + kLinProducers * (jc * 2 + e);
                            if (uu < units) {
                                const int kg = uu / N, r = uu - kg * N;
                                uint4 xhi, xlo;
                                split_bf16x8(cur.a[e], cur.c[e], xhi, xlo);
                                const uint32_t off = mma_tile_off(mode, r, kg);
                                *reinterpret_cast<uint4*>(xh + off) = xhi;
                                *reinterpret_cast<uint4*>(xl + off) = xlo;
                            }
                        }
                        if (jc == JC - 1) {
                            fence_proxy_async_smem();                 // X stores -> visible to the wgmma reads
                            named_bar_sync(1, kLinProducers);         // every consumer warp has stored its part
                            mbar_wait_mma(&full_w[s], (uint32_t)(it / S) & 1u);
                            if (it == 0 && pt == 0) trace_stamp(L.dbg, 4);
                            mma_kblock(acc, stage0 + (uint32_t)s * stage_bytes, x_half_bytes, mode, it == 0);
                            __syncwarp();
                            if (lane == 0) mbar_arrive(&empty[s]);
                        }
                        cur = nxt;
                    }
                }
                if (pt == 0) trace_stamp(L.dbg, 6);
                if (L.tl && pt == 0) tl_main_done(L.tl);
                // ---- part 1: accumulator tile -> shared memory.  tile_s[col][n] (fp32, n fastest) lives in the idle
                // pipeline stages: every TMA write has landed, and every MMA has read its operands once both
                // warpgroups are past this barrier.
                named_bar_sync(1, kLinProducers);
                if (pt == 0) trace_stamp(L.dbg, 7);
                acc_for_each(acc, N, [&](int m, int n, float v) {
                    tile_s[n * kTileN + m] = bias_fold ? v + bias_fold[m] : v;
                });
                // ---- split-K partials meet through distributed shared memory.  The `splits` CTAs of a tile form
                // one thread-block cluster; after the cluster barrier CTA `split` sums rows [lo, hi) of all
                // partial tiles in fixed rank order (bit-reproducible), applies the fused epilogue and writes
                // coalesced rows.  splits == 1 is the same code reading only its own tile.
                if (splits > 1) {
                    __syncwarp();
                    cluster_sync_all();
                } else {
                    named_bar_sync(1, kLinProducers);   // the tile is complete: only the epilogue warps read it
                }
                if (pt == 0) trace_stamp(L.dbg, 8);
            }
            // ---- part 2: one warp = one activation row per iteration (lane u owns outputs 4u..4u+3).  Kept
            // ROLLED and small on purpose: this code runs a handful of times per launch, so its cost is the
            // number of distinct instructions fetched, not arithmetic.
            // (dry pass: every shared-memory read goes to a 512-byte scratch line of the control block instead of the
            // pipeline stages, which the TMA is still filling: same instructions, no race with the async writes)
            const float* const row_base = dry ? reinterpret_cast<const float*>(smem_raw + 512) : tile_s;
            const int row_mul = dry ? 0 : kTileN;
            const uint32_t row_addr = dry ? smem_u32(smem_raw + 512) : tile_addr;
            uint32_t peer[8];
#pragma unroll
            for (int r = 0; r < 8; ++r)   // (dry: the own scratch line stands in for every peer)
                peer[r] = (splits > 1 && r < splits) ? dsmem_map(row_addr, (uint32_t)(dry ? split : r)) : row_addr;
            if (pt == 0 && !dry) trace_stamp(L.dbg, 15);
            const bool long_rows = row_loop && splits == 1 && epi != kEpiLstm && !out_pa && vec_out && !dry &&
                                   hi - lo > 4 * kLinProducers;
            if (long_rows) {
                // many rows per warp and nothing but bias / tanh / a coalesced store to do (context projection,
                // wide batches): four rows per iteration keep four shared-memory loads, activation chains and
                // stores in flight instead of one
#pragma unroll 1
                for (int idx = lo + pt; idx < hi; idx += 4 * kLinProducers) {
                    float4 g4[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int id = idx + j * kLinProducers;
                        if (id < hi) g4[j] = *reinterpret_cast<const float4*>(tile_s + (id >> 5) * kTileN + 4 * u);
                    }
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int id = idx + j * kLinProducers;
                        if (id < hi) {
                            float4 g = g4[j];
                            if (!do_am) { g.x += bias4.x; g.y += bias4.y; g.z += bias4.z; g.w += bias4.w; }
                            if (epi == kEpiBiasTanh) { g.x = act_tanh(g.x); g.y = act_tanh(g.y); g.z = act_tanh(g.z); g.w = act_tanh(g.w); }
                            if (out) {
                                float4* o = reinterpret_cast<float4*>(out + (size_t)(row0 + (id >> 5)) * ldo + ng);
                                if (P.accumulate) { const float4 a = *o; g.x += a.x; g.y += a.y; g.z += a.z; g.w += a.w; }
                                *o = g;
                            }
                        }
                    }
                }
            } else if (row_loop) {
                // the partial tiles of the NEXT row are requested before the current row is finished: the DSMEM /
                // shared-memory round trips of a thread's (typically two) rows overlap
                float4 cur[8], nxt[8];
                auto fetch = [&](float4 (&dst)[8], int idx) {
                    const int bb = idx >> 5;
                    if (splits == 1) {
                        dst[0] = *reinterpret_cast<const float4*>(row_base + bb * row_mul + 4 * u);
                    } else {
                        const uint32_t off = (uint32_t)(bb * row_mul + 4 * u) * 4u;
#pragma unroll
                        for (int r = 0; r < 8; ++r)
                            if (r < splits) dst[r] = ld_dsmem_f4(peer[r] + off);
                    }
                };
                if (splits > 1) {
                    if (lo + pt < hi) fetch(cur, lo + pt);
                    if (lo + pt + kLinProducers < hi) fetch(nxt, lo + pt + kLinProducers);
                }
#pragma unroll 1
                for (int idx = lo + pt; idx < hi; idx += kLinProducers) {
                    const int bb = idx >> 5;
                    float cprev = idx == lo + pt ? cpre[0] : cpre[1];
                    if (epi == kEpiLstm && unit < Hh && idx >= lo + pt + 2 * kLinProducers)
                        cprev = c_in[(size_t)(row0 + bb) * Hh + unit];
                    float4 g;
                    if (splits == 1) {
                        g = *reinterpret_cast<const float4*>(row_base + bb * row_mul + 4 * u);
                    } else {
                        g = cur[0];
#pragma unroll
                        for (int r = 1; r < 8; ++r)
                            if (r < splits) { g.x += cur[r].x; g.y += cur[r].y; g.z += cur[r].z; g.w += cur[r].w; }
#pragma unroll
                        for (int r = 0; r < 8; ++r) cur[r] = nxt[r];
                        if (idx + 2 * kLinProducers < hi) fetch(nxt, idx + 2 * kLinProducers);
                    }
                    if (!do_am) { g.x += bias4.x; g.y += bias4.y; g.z += bias4.z; g.w += bias4.w; }
                    if (pt == 0 && !dry && L.dbg && g.x != 12345.678f) trace_stamp(L.dbg, 2);   // partial sums arrived
                    if (epi == kEpiLstm) {
                        if (unit < Hh) lstm_gates(P, g, cprev, row0 + bb, unit, mode, dry);
                        if (pt == 0 && !dry) trace_stamp(L.dbg, 3);
                        continue;
                    }
                    if (epi == kEpiBiasTanh) { g.x = act_tanh(g.x); g.y = act_tanh(g.y); g.z = act_tanh(g.z); g.w = act_tanh(g.w); }
                    if (dry) continue;
                    if (pt == 0 && L.dbg && g.x != 12345.678f) trace_stamp(L.dbg, 3);   // activation done
                    if (out) {
                        float* o = out + (size_t)(row0 + bb) * ldo + ng;
                        if (vec_out) {
                            if (P.accumulate) { const float4 a = *reinterpret_cast<const float4*>(o); g.x += a.x; g.y += a.y; g.z += a.z; g.w += a.w; }
                            *reinterpret_cast<float4*>(o) = g;
                        } else {
                            const bool acc = P.accumulate != 0;   // (never read `o` otherwise: it may hold anything)
                            if (ng + 0 < n_out) o[0] = acc ? g.x + o[0] : g.x;
                            if (ng + 1 < n_out) o[1] = acc ? g.y + o[1] : g.y;
                            if (ng + 2 < n_out) o[2] = acc ? g.z + o[2] : g.z;
                            if (ng + 3 < n_out) o[3] = acc ? g.w + o[3] : g.w;
                        }
                    }
                    if (out_pa) {
                        const float y[4] = {g.x, g.y, g.z, g.w};
                        if (ng + 3 < n_out) {
                            pa_store4(out_pa, mode, N, n_out >> 6, row0 + bb, ng, y);
                        } else {
#pragma unroll 1
                            for (int e = 0; e < 4; ++e)
                                if (ng + e < n_out) pa_store(out_pa, mode, N, n_out >> 6, row0 + bb, ng + e, y[e]);
                        }
                    }
                }
            }
            if (do_am) {
                // greedy prediction (model.py:289): 4 threads per row, each scans 32 of the tile's 128 outputs
                // (accumulator + bias, folded in part 1: the value the row loop stores) in a skewed,
                // bank-conflict-free order;
                // first maximum wins (tf.argmax), so ties go to the smaller index
                const int part = pt & 3;
#pragma unroll 1
                for (int r0 = 0; r0 < rows_here; r0 += kLinProducers / 4) {
                    const int r = r0 + (pt >> 2);
                    const bool live = r < rows_here;
                    const float4* row_t = reinterpret_cast<const float4*>(row_base + (live ? r : 0) * row_mul) + part * 8;
                    // every element becomes an ordered 64-bit key (value bits, then inverted index) and the scan is a
                    // running 64-bit max: two independent chains of 2-instruction steps instead of one chain of
                    // compare / compare / select per element
                    unsigned long long k0 = 0ull, k1 = 0ull;
                    float mr = -INFINITY;   // (SWP) raw maximum: the keys rank the perturbed values
                    if constexpr (SMP) {
                        // the draw of (seed, row, step, word): key once per row, one hash + two logarithms per logit
                        const SampleKey sk = sample_key(P.smp->seed, row0 + r, P.am_step);
                        const float itau = P.smp->inv_tau;
                        auto draw = [&](float v, int i) -> unsigned long long {
                            return i < n_out ? argmax_key(fmaf(v, itau, sample_gumbel(sample_bits(sk, i))), i) : 0ull;
                        };
                        // (the warm-up pass runs before the main loop of its warps: one unrolled iteration warms the
                        // code, all eight would hold the MMAs back by the cost of the draw)
                        const int jn = dry ? 2 : 8;
#pragma unroll 2
                        for (int j = 0; j < jn; ++j) {
                            const int jj = (j + pt) & 7;
                            const float4 a4 = row_t[jj];
                            const int i0 = n_tile * kTileN + part * 32 + jj * 4;
                            k0 = max(k0, max(draw(a4.x, i0 + 0), draw(a4.y, i0 + 1)));
                            k1 = max(k1, max(draw(a4.z, i0 + 2), draw(a4.w, i0 + 3)));
                            if constexpr (WP) {
                                mr = fmaxf(mr, fmaxf(i0 + 0 < n_out ? a4.x : -INFINITY, i0 + 1 < n_out ? a4.y : -INFINITY));
                                mr = fmaxf(mr, fmaxf(i0 + 2 < n_out ? a4.z : -INFINITY, i0 + 3 < n_out ? a4.w : -INFINITY));
                            }
                        }
                    } else {
#pragma unroll 2
                    for (int j = 0; j < 8; ++j) {
                        const int jj = (j + pt) & 7;
                        const float4 a4 = row_t[jj];
                        const int i0 = n_tile * kTileN + part * 32 + jj * 4;
                        const unsigned long long e0 = i0 + 0 < n_out ? argmax_key(a4.x, i0 + 0) : 0ull;
                        const unsigned long long e1 = i0 + 1 < n_out ? argmax_key(a4.y, i0 + 1) : 0ull;
                        const unsigned long long e2 = i0 + 2 < n_out ? argmax_key(a4.z, i0 + 2) : 0ull;
                        const unsigned long long e3 = i0 + 3 < n_out ? argmax_key(a4.w, i0 + 3) : 0ull;
                        k0 = max(k0, max(e0, e1));
                        k1 = max(k1, max(e2, e3));
                    }
                    }
                    unsigned long long key = max(k0, k1);
                    key = max(key, __shfl_xor_sync(0xffffffffu, key, 1));
                    key = max(key, __shfl_xor_sync(0xffffffffu, key, 2));
                    if (live && part == 0 && !dry) am_key[r] = key;
                    if constexpr (WP) {
                        // softmax partial of the row over this tile, relative to the tile maximum (the key's value;
                        // sampling: the raw maximum)
                        float mt;
                        if constexpr (SMP) {
                            mt = fmaxf(mr, __shfl_xor_sync(0xffffffffu, mr, 1));
                            mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, 2));
                        } else {
                            mt = argmax_key_value(key);
                        }
                        float s = 0.f;
#pragma unroll 2
                        for (int j = 0; j < 8; ++j) {
                            const int jj = (j + pt) & 7;
                            const float4 a4 = row_t[jj];
                            const int i0 = n_tile * kTileN + part * 32 + jj * 4;
                            if (i0 + 0 < n_out) s += expf(a4.x - mt);
                            if (i0 + 1 < n_out) s += expf(a4.y - mt);
                            if (i0 + 2 < n_out) s += expf(a4.z - mt);
                            if (i0 + 3 < n_out) s += expf(a4.w - mt);
                        }
                        s += __shfl_xor_sync(0xffffffffu, s, 1);
                        s += __shfl_xor_sync(0xffffffffu, s, 2);
                        if (live && part == 0) {
                            float* const am_sum = P.am_sum + (size_t)(rt * P.n_tiles + n_tile) * N;
                            if (!dry) am_sum[r] = s;
                            if constexpr (SMP) {   // the tile's sampled candidate keeps its raw logit beside the key
                                const int c = (argmax_key_index(key) - n_tile * kTileN) & (kTileN - 1);
                                const float lw = row_base[r * row_mul + c];
                                if (!dry) P.am_smp[(size_t)(rt * P.n_tiles + n_tile) * N + r] = make_float2(mt, lw);
                            } else if (P.am_forced) {   // teacher forcing: the tile that owns the forced word keeps its logit
                                const int w = P.am_forced[(size_t)(row0 + r) * P.am_forced_ld + P.am_step];
                                const int c = w - n_tile * kTileN;
                                if (c >= 0 && c < kTileN && w < n_out) {
                                    const float lw = row_base[r * row_mul + c];
                                    if (!dry) P.am_wlogit[row0 + r] = lw;
                                }
                            }
                        }
                    }
                }
            }
            if (splits > 1 && !dry) cluster_arrive_relaxed();   // this CTA no longer reads its peers' tiles
            if (do_am) {
                // Tile candidates are in global memory.  All CTAs of the layer (one wave: co-resident, so waiting
                // cannot deadlock) meet at a grid barrier; then CTA i finishes row i, i + #CTAs, ...: it merges the
                // row's per-tile candidates (one L2 round trip), records the word and - in the decode loop - hands
                // the embedding row of the chosen word (model.py:272-274), packed, to the next LSTM / decode layers.
                // Every step of this tail is a round trip on the critical path of the decode step, which is why it
                // is spread over the CTAs instead of being a serial pass of the last one.
                unsigned long long* red_s = reinterpret_cast<unsigned long long*>(smem_raw + 256);   // [8] + word (clear of the dry pass's scratch line)
                if (!dry) {
                    if (pt == 0) trace_stamp(L.dbg, 11);
                    __threadfence();
                    named_bar_sync(1, kLinProducers);
                    if (pt == 0) {
                        if (atomicAdd(P.am_ctr, 1u) == (unsigned)(P.cta_count - 1)) {
                            *P.am_ctr = 0u;
                            __threadfence();
                            atomicAdd(P.am_ctr + 1, 1u);          // opens the generation: every candidate is visible
                        } else if (local < P.rows) {             // (CTAs with no row to finish leave at once)
                            const long long t0 = clock64();
                            while (ld_acquire_gpu(P.am_ctr + 1) == am_gen0) {
                                if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) __trap();   // arg-max rendezvous
                            }
                        }
                        trace_stamp(L.dbg, 12);
                    }
                    named_bar_sync(1, kLinProducers);
                }
                const int n_tiles = P.n_tiles;
                const int E = P.am_E;
                const size_t halfb = (size_t)N * kBK * 2;
#pragma unroll 1
                for (int r = local; r < P.rows; r += P.cta_count) {
                    const int rt2 = r / N, cc = r - rt2 * N;
                    const unsigned long long* pk = P.am_key + (size_t)rt2 * n_tiles * N + cc;
                    unsigned long long best = 0ull;
                    float lm = -INFINITY, ls = 0.f;   // (WP) merged softmax partials of this thread's tiles
                    float braw = 0.f;                 // (SWP) raw logit of the best candidate
                    for (int tl = pt; tl < n_tiles; tl += kLinProducers) {
                        const unsigned long long k = __ldcg(pk + (size_t)tl * N);
                        if constexpr (SWP) {
                            const float2 ms = __ldcg(P.am_smp + (pk - P.am_key) + (size_t)tl * N);
                            if (k > best) braw = ms.y;
                            best = max(best, k);
                            lse_merge(lm, ls, ms.x, __ldcg(P.am_sum + (pk - P.am_key) + (size_t)tl * N));
                        } else {
                        best = max(best, k);
                        if constexpr (WP) lse_merge(lm, ls, argmax_key_value(k), __ldcg(P.am_sum + (pk - P.am_key) + (size_t)tl * N));
                        }
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        if constexpr (SWP) {
                            const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
                            const float orw = __shfl_xor_sync(0xffffffffu, braw, o);
                            if (ob > best) { best = ob; braw = orw; }
                        } else {
                        best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
                        }
                        if constexpr (WP) lse_merge(lm, ls, __shfl_xor_sync(0xffffffffu, lm, o), __shfl_xor_sync(0xffffffffu, ls, o));
                    }
                    float2* const red_ms = reinterpret_cast<float2*>(smem_raw + 384);   // [8] (between red_s and the scratch line)
                    float* const red_raw = reinterpret_cast<float*>(smem_raw + 448);    // [8] (SWP)
                    if ((pt & 31) == 0) {
                        red_s[pt >> 5] = best;
                        if constexpr (WP) red_ms[pt >> 5] = make_float2(lm, ls);
                        if constexpr (SWP) red_raw[pt >> 5] = braw;
                    }
                    named_bar_sync(1, kLinProducers);
                    if (pt == 0) {
#pragma unroll
                        for (int w = 1; w < kLinProducers / 32; ++w) {
                            if constexpr (SWP) {
                                if (red_s[w] > best) braw = red_raw[w];
                            }
                            best = max(best, red_s[w]);
                            if constexpr (WP) lse_merge(lm, ls, red_ms[w].x, red_ms[w].y);
                        }
                        const int bi2 = argmax_key_index(best);
                        const int nw = P.am_forced ? P.am_forced[(size_t)r * P.am_forced_ld + P.am_step] : bi2;
                        if constexpr (SWP) {
                            // softmax(logits)[w] at temperature 1 of the sampled word w: lm is the raw row maximum
                            if (!dry) P.am_probs[(size_t)r * P.am_probs_ld + P.am_step] = expf(braw - lm) / ls;
                        } else if constexpr (WP) {
                            // softmax(logits)[nw] = exp(l_nw - M) / S; M is the row maximum (lm == its value); a forced
                            // word outside [0, V) has probability 0 and is never used as an index
                            float pw = 0.f;
                            if (!P.am_forced) pw = 1.0f / ls;
                            else if (nw >= 0 && nw < P.n_out) pw = expf(__ldcg(P.am_wlogit + r) - lm) / ls;
                            if (!dry) P.am_probs[(size_t)r * P.am_probs_ld + P.am_step] = pw;
                        }
                        if (!dry) {
                            if (P.am_tokens) P.am_tokens[(size_t)r * P.am_tokens_ld + P.am_step] = bi2;
                            if (P.am_next_word) P.am_next_word[r] = nw;
                        }
                        *reinterpret_cast<int*>(red_s + 8) = dry ? 0 : nw;
                    }
                    named_bar_sync(1, kLinProducers);
                    if (P.am_emb_pa) {
                        const int w = *reinterpret_cast<const int*>(red_s + 8);
                        const int rr = cc;
#pragma unroll 1
                        for (int gi = pt; gi < (E >> 3); gi += kLinProducers) {
                            const float4* src = reinterpret_cast<const float4*>(P.am_emb + (size_t)w * E + gi * 8);
                            const float4 a4 = __ldg(src), c4 = __ldg(src + 1);
                            uint4 hi4, lo4;
                            split_bf16x8(a4, c4, hi4, lo4);
                            uint8_t* dst = P.am_emb_pa + ((size_t)rt2 * (E >> 6) + (gi >> 3)) * 2 * halfb +
                                           mma_tile_off(mode, rr, gi & 7);
                            if (!dry) {
                                *reinterpret_cast<uint4*>(dst) = hi4;
                                *reinterpret_cast<uint4*>(dst + halfb) = lo4;
                            }
                        }
                    }
                }
                if (pt == 0 && !dry) trace_stamp(L.dbg, 13);
            }
        }
    }
    if (warp >= kTmaWarp && P.splits > 1) {   // the TMA warps join the cluster rendezvous of the epilogue
        __syncwarp();
        cluster_sync_all();
        cluster_arrive_relaxed();
    }
    if (threadIdx.x == 0) trace_stamp(L.dbg, 9);
    if (P.splits > 1) cluster_wait();   // peers may still be reading this CTA's tile

    __syncthreads();
    if (threadIdx.x == 0) { trace_stamp(L.dbg, 10); tl_end(L.tl); }
}

// -------------------------------------------------- SIMT bring-up kernel
// Same math on CUDA cores from the same packed weights (w = hi + lo).  Used by
// the tests to cross-check the wgmma path and its packing; selected with
// sat_set_option("gemm", 0).  Grid: one CTA per (n_tile, 16-row group).
__global__ void __launch_bounds__(128) lin_simt_kernel(const __grid_constant__ LinLaunch L) {
    __shared__ float xs[16][kBK + 1];
    int pi = 0;
#pragma unroll
    for (int i = 1; i < kMaxProb; ++i)
        if (i < L.nprob && (int)blockIdx.x >= L.p[i].cta_begin) pi = i;
    const LinProblem& P = L.p[pi];
    const int local = blockIdx.x - P.cta_begin;
    const int n_tile = local % P.n_tiles;
    const int rg = local / P.n_tiles;
    const int row0 = rg * 16;
    const int r = threadIdx.x;  // output feature within tile
    const int mode = L.layout_mode;
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    for (int kb = 0; kb < P.k_blocks; ++kb) {
        __syncthreads();
        {   // 16 rows x 8 k-groups = 128 groups, one per thread
            const int b = threadIdx.x >> 3, kg = threadIdx.x & 7;
            float4 a, c;
            load_x8(P, row0 + b, kb * kBK + kg * 8, a, c);
            float* d = &xs[b][kg * 8];
            d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = c.x; d[5] = c.y; d[6] = c.z; d[7] = c.w;
        }
        __syncthreads();
        const uint8_t* tile = P.wpack + ((size_t)n_tile * P.k_blocks + kb) * kWStageBytes;
        for (int kg = 0; kg < 8; ++kg) {
            const uint32_t off = mma_tile_off(mode, r, kg);
            const uint4 hi = *reinterpret_cast<const uint4*>(tile + off);
            const uint4 lo = *reinterpret_cast<const uint4*>(tile + kWHalfBytes + off);
            const uint32_t hh[4] = {hi.x, hi.y, hi.z, hi.w}, ll[4] = {lo.x, lo.y, lo.z, lo.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const uint32_t hv = (e & 1) ? (hh[e >> 1] >> 16) : (hh[e >> 1] & 0xffffu);
                const uint32_t lv = (e & 1) ? (ll[e >> 1] >> 16) : (ll[e >> 1] & 0xffffu);
                const float w = __uint_as_float(hv << 16) + __uint_as_float(lv << 16);
#pragma unroll
                for (int j = 0; j < 16; ++j) acc[j] = fmaf(xs[j][kg * 8 + e], w, acc[j]);
            }
        }
    }
    const int n = n_tile * kTileN + r;
    if (P.epi == kEpiLstm) {
        const int lane = threadIdx.x & 31, base = lane & ~3;
        for (int j = 0; j < 16; ++j) {
            const float v = acc[j] + P.bias[n];
            float4 g;
            g.x = __shfl_sync(0xffffffffu, v, base + 0);
            g.y = __shfl_sync(0xffffffffu, v, base + 1);
            g.z = __shfl_sync(0xffffffffu, v, base + 2);
            g.w = __shfl_sync(0xffffffffu, v, base + 3);
            const int unit = n >> 2;
            if ((lane & 3) == 0 && row0 + j < P.rows && unit < P.H)
                lstm_gates(P, g, P.c_in[(size_t)(row0 + j) * P.H + unit], row0 + j, unit, mode, false);
        }
    } else if (n < P.n_out) {
        for (int j = 0; j < 16; ++j)
            if (row0 + j < P.rows) {
                const float y = epi_scalar(P, acc[j], n);
                if (P.out) P.out[(size_t)(row0 + j) * P.ldo + n] = y;
                if (P.out_pa) pa_store(P.out_pa, mode, P.row_tile, P.n_out >> 6, row0 + j, n, y);
            }
    }
}

// ---------------------------------------------------- one-time weight repack
// TF kernel [K, n_out] fp32 row-major (tf.layers.dense, utils/nn.py:96-105) ->
// packed bf16 hi/lo MMA operand tiles.  perm_H > 0 selects the LSTM gate interleave:
// packed output p = unit*4 + gate  <->  TF column gate*H + unit (split order i,j,f,o).
__global__ void repack_weight_kernel(const float* __restrict__ w, int K, int n_out, int perm_H, uint8_t* wpack,
                                     int k_blocks, int n_tiles, int mode, DropSpec drop, int pdl) {
    if (pdl) { pdl_wait(); pdl_launch_dependents(); }   // launched with programmatic serialization (training path)
    const unsigned long long seed = drop.seedp ? *drop.seedp : 0ull;
    const DropGen gen = drop_gen(seed, drop.stream, drop.keep);
    const size_t total = (size_t)n_tiles * k_blocks * kTileN * 8;  // 16-byte groups
    for (size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        const int r = (int)(g % kTileN);
        size_t t = g / kTileN;
        const int kg = (int)(t % 8);
        t /= 8;
        const int kb = (int)(t % k_blocks);
        const int nt = (int)(t / k_blocks);
        const int p = nt * kTileN + r;
        int col = -1;
        if (p < n_out) col = perm_H > 0 ? (p & 3) * perm_H + (p >> 2) : p;
        float x[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int k = kb * kBK + kg * 8 + e;
            x[e] = (col >= 0 && k < K) ? w[(size_t)k * n_out + col] : 0.f;
            if (seed && col >= 0 && k < K) x[e] *= gen.scale((unsigned long long)k * n_out + col);
        }
        uint4 hi, lo;
        split_bf16x8(make_float4(x[0], x[1], x[2], x[3]), make_float4(x[4], x[5], x[6], x[7]), hi, lo);
        uint8_t* tile = wpack + ((size_t)nt * k_blocks + kb) * kWStageBytes;
        const uint32_t off = mma_tile_off(mode, r, kg);
        *reinterpret_cast<uint4*>(tile + off) = hi;
        *reinterpret_cast<uint4*>(tile + kWHalfBytes + off) = lo;
    }
}

__global__ void repack_bias_kernel(const float* __restrict__ b, int n_out, int perm_H, float* out, int npad) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npad; p += gridDim.x * blockDim.x) {
        float v = 0.f;
        if (p < n_out && b) v = b[perm_H > 0 ? (p & 3) * perm_H + (p >> 2) : p];
        out[p] = v;
    }
}

// fp32 rows (optionally gathered: embedding lookup) -> packed activation; up to 2 jobs per launch
struct PackJobs {
    PackJob j[2];
    int n, mode;
    DropSpec drop;
    int pdl;
};
__global__ void pack_rows_kernel(const PackJobs J) {
    if (J.pdl) { pdl_wait(); pdl_launch_dependents(); }   // launched with programmatic serialization (training path)
    const unsigned long long seed = J.drop.seedp ? *J.drop.seedp : 0ull;
    const DropGen gen = drop_gen(seed, J.drop.stream, J.drop.keep);
    for (int q = 0; q < J.n; ++q) {
        const PackJob& jb = J.j[q];
        const int groups = jb.width >> 3;
        const int nrt = (jb.rows + jb.row_tile - 1) / jb.row_tile;
        const int total = nrt * jb.row_tile * groups;   // padded rows are zero filled
        const size_t half = (size_t)jb.row_tile * kBK * 2;
        for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < total; u += gridDim.x * blockDim.x) {
            const int b = u / groups, g = u - b * groups;
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f), c = a;
            if (b < jb.rows) {
                const int row = jb.gather ? jb.gather[b] : b;
                const float4* src = reinterpret_cast<const float4*>(jb.src + (size_t)row * jb.ld + g * 8);
                a = src[0];
                c = src[1];
                if (seed) {
                    const unsigned long long i0 = (unsigned long long)row * jb.width + g * 8;
                    a.x *= gen.scale(i0);
                    a.y *= gen.scale(i0 + 1);
                    a.z *= gen.scale(i0 + 2);
                    a.w *= gen.scale(i0 + 3);
                    c.x *= gen.scale(i0 + 4);
                    c.y *= gen.scale(i0 + 5);
                    c.z *= gen.scale(i0 + 6);
                    c.w *= gen.scale(i0 + 7);
                }
            }
            uint4 hi, lo;
            split_bf16x8(a, c, hi, lo);
            const int rt = b / jb.row_tile, r = b - rt * jb.row_tile;
            const int kbs = jb.k_blocks > 0 ? jb.k_blocks : (jb.width >> 6);
            uint8_t* dst = jb.pa + ((size_t)rt * kbs + (g >> 3)) * 2 * half + mma_tile_off(J.mode, r, g & 7);
            *reinterpret_cast<uint4*>(dst) = hi;
            *reinterpret_cast<uint4*>(dst + half) = lo;
        }
    }
}

// launch with the programmatic-serialization attribute: the kernel waits for its predecessor itself (first statement)
template <typename... KA, typename... A>
static cudaError_t launch_serialized(void (*kernel)(KA...), int grid, int block, cudaStream_t st, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KA>(args)...);
}

cudaError_t pack_rows_launch(const PackJob* jobs, int njobs, int layout_mode, cudaStream_t st, const DropSpec* drop, int pdl) {
    PackJobs J;
    J.pdl = pdl;
    J.n = njobs;
    J.mode = layout_mode;
    J.drop = drop ? *drop : DropSpec{nullptr, 0ull, 1.0f};
    int total = 0;
    for (int i = 0; i < njobs; ++i) {
        J.j[i] = jobs[i];
        const int nrt = (jobs[i].rows + jobs[i].row_tile - 1) / jobs[i].row_tile;
        total = max(total, nrt * jobs[i].row_tile * (jobs[i].width >> 3));
    }
    int grid = (total + 255) / 256;
    if (grid > device_sm_count() * 8) grid = device_sm_count() * 8;   // every thread converts a few 32-byte groups: short dependent chains
    if (grid < 1) grid = 1;
    if (pdl) return launch_serialized(pack_rows_kernel, grid, 256, st, J);
    pack_rows_kernel<<<grid, 256, 0, st>>>(J);
    return cudaGetLastError();
}

// ------------------------------------------------------------ host side
int device_sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0 && cudaDeviceGetAttribute(&cached[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
        cudaGetLastError();
        return 132;
    }
    return cached[dev];
}

static int g_smem_optin = 0;

// [plain, word probabilities, sampling with word probabilities, sampling][row tile / 16 - 1]
static void (*const g_lin_kernels[4][kMaxRowTile / 16])(LinLaunch) = {
    {lin_mma_kernel<1, false>, lin_mma_kernel<2, false>, lin_mma_kernel<3, false>, lin_mma_kernel<4, false>,
     lin_mma_kernel<5, false>, lin_mma_kernel<6, false>, lin_mma_kernel<7, false>, lin_mma_kernel<8, false>},
    {lin_mma_kernel<1, true>, lin_mma_kernel<2, true>, lin_mma_kernel<3, true>, lin_mma_kernel<4, true>,
     lin_mma_kernel<5, true>, lin_mma_kernel<6, true>, lin_mma_kernel<7, true>, lin_mma_kernel<8, true>},
    {lin_mma_kernel<1, true, true>, lin_mma_kernel<2, true, true>, lin_mma_kernel<3, true, true>,
     lin_mma_kernel<4, true, true>, lin_mma_kernel<5, true, true>, lin_mma_kernel<6, true, true>,
     lin_mma_kernel<7, true, true>, lin_mma_kernel<8, true, true>},
    {lin_mma_kernel<1, false, true>, lin_mma_kernel<2, false, true>, lin_mma_kernel<3, false, true>,
     lin_mma_kernel<4, false, true>, lin_mma_kernel<5, false, true>, lin_mma_kernel<6, false, true>,
     lin_mma_kernel<7, false, true>, lin_mma_kernel<8, false, true>}};

cudaError_t lin_init_attrs() {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    e = cudaDeviceGetAttribute(&g_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) return e;
    for (auto& inst : g_lin_kernels)
        for (auto k : inst) {
            e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, g_smem_optin);
            if (e != cudaSuccess) return e;
        }
    return cudaSuccess;
}

size_t lin_smem_bytes(int row_tile, int stages) {
    return 1024 + (size_t)stages * (kWStageBytes + 2 * (size_t)row_tile * kBK * 2);
}

int lin_pick_stages(int row_tile) {
    const size_t budget = (size_t)(g_smem_optin > 0 ? g_smem_optin : 232448) - 1024;
    const size_t per = kWStageBytes + 2 * (size_t)row_tile * kBK * 2;
    int s = (int)(budget / per);
    if (s > 8) s = 8;
    return s;
}

cudaError_t lin_launch(const LinLaunch& L, cudaStream_t st, bool use_simt) {
    int total = 0;
    if (use_simt) {
        LinLaunch M = L;
        for (int i = 0; i < M.nprob; ++i) {
            M.p[i].cta_begin = total;
            M.p[i].cta_count = M.p[i].n_tiles * ((M.p[i].rows + 15) / 16);
            total += M.p[i].cta_count;
        }
        lin_simt_kernel<<<total, 128, 0, st>>>(M);
        return cudaGetLastError();
    }
    int max_rt = 16, wp = 0;
    for (int i = 0; i < L.nprob; ++i) {
        total += L.p[i].cta_count;
        if (L.p[i].am_probs) {
            if (!L.p[i].am_key || !L.p[i].am_sum || L.p[i].splits != 1 || (L.p[i].am_forced && !L.p[i].am_wlogit))
                return cudaErrorInvalidValue;
            wp = 1;
        }
        if (L.p[i].smp) {
            if (!L.p[i].am_key || L.p[i].splits != 1 || L.p[i].am_forced || (L.p[i].am_probs && !L.p[i].am_smp))
                return cudaErrorInvalidValue;
            wp = L.p[i].am_probs ? 2 : 3;
        }
        if (L.p[i].row_tile > max_rt) max_rt = L.p[i].row_tile;
        // (one MMA width per launch: grouped problems share the row tile, so no MMA reads past its operand)
        if (L.p[i].row_tile % 16 || L.p[i].row_tile > kMaxRowTile || L.p[i].row_tile != L.p[0].row_tile)
            return cudaErrorInvalidValue;
    }
    const size_t smem = lin_smem_bytes(max_rt, L.stages);
    // every problem of a launch uses the same split factor: the `splits` CTAs of a tile are one cluster
    const int splits = L.p[0].splits;
    for (int i = 1; i < L.nprob; ++i)
        if (L.p[i].splits != splits) return cudaErrorInvalidValue;
    if (splits > 1 && L.x_mode == 1) return cudaErrorInvalidValue;   // grid barrier + clusters are not combined
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(total);
    cfg.blockDim = dim3(kLinThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[3];
    int na = 0;
    if (splits > 1) {
        at[na].id = cudaLaunchAttributeClusterDimension;
        at[na].val.clusterDim.x = (unsigned)splits;
        at[na].val.clusterDim.y = 1;
        at[na].val.clusterDim.z = 1;
        ++na;
    } else if (L.x_mode == 1) {   // the activation pre-pass ends in a grid barrier: CTAs must be co-resident
        at[na].id = cudaLaunchAttributeCooperative;
        at[na].val.cooperative = 1;
        ++na;
    }
    if (L.pdl) {
        at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = at;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, g_lin_kernels[wp][max_rt / 16 - 1], L);
}

cudaError_t lin_repack_weight(const float* w_tf, int K, int n_out, int perm_H, uint8_t* wpack, int layout_mode,
                              cudaStream_t st, const DropSpec* drop, int pdl) {
    const int k_blocks = (K + kBK - 1) / kBK, n_tiles = (n_out + kTileN - 1) / kTileN;
    const DropSpec ds = drop ? *drop : DropSpec{nullptr, 0ull, 1.0f};
    if (pdl) return launch_serialized(repack_weight_kernel, 1184, 256, st, w_tf, K, n_out, perm_H, wpack, k_blocks, n_tiles, layout_mode, ds, 1);
    repack_weight_kernel<<<1184, 256, 0, st>>>(w_tf, K, n_out, perm_H, wpack, k_blocks, n_tiles, layout_mode, ds, 0);
    return cudaGetLastError();
}

cudaError_t lin_repack_bias(const float* b_tf, int n_out, int perm_H, float* bias_packed, cudaStream_t st) {
    const int npad = ((n_out + kTileN - 1) / kTileN) * kTileN;
    repack_bias_kernel<<<(npad + 255) / 256, 256, 0, st>>>(b_tf, n_out, perm_H, bias_packed, npad);
    return cudaGetLastError();
}

}  // namespace sat
