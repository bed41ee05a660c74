// sat_chain.cu — the dense layers of one greedy decode step as ONE persistent launch.
//
//   phase 0  LSTM cell                       G = [z, emb(word), h] K + b -> (c, h)            model.py:276-279
//   phase 1  decode fc_1  ||  attend fc_1b   t = tanh([h, z, emb] Wd1 + b) ; q' = tanh(h W1b + b)   :448-453, :421-424
//   phase 2  decode fc_2 + arg-max           logits = t Wd2 + b ; word = argmax ; emb(word)    :455-458, :289, :272-274
//
// Why one launch.  Each layer needs the complete output of the layer before it, and every layer alone is one CTA per SM
// (its pipeline stages fill the shared memory), so with one launch per layer a successor CTA becomes resident only when
// the predecessor CTA on its SM has EXITED — after its tail — and then starts its weight stream cold: with the weights
// largely L2 resident, cold starts, tails and dependency releases rather than bandwidth bound such a step.  Here
// every CTA is resident for the whole step; its TMA lane keeps streaming the (immutable) weights of its NEXT tile into
// the stages the tensor core has released, i.e. under the epilogue and the rendezvous of the current phase, and the
// phases meet at grid-wide arrival counters (one L2 round trip) instead of at kernel boundaries.
//
// Same arithmetic as lin_mma_kernel (sat_linear.cu): swap-AB wgmma tiles (128 outputs x row_tile batch rows), packed
// bf16 hi/lo operands fetched by 1-D bulk TMA, three MMAs per K step, fp32 accumulation in registers, split-K partials
// summed in fixed split order — the two kernels produce bit-identical results.  Differences: split-K partials meet in an L2
// resident scratch buffer behind a per-tile arrival counter (no thread-block clusters: the grid need not be cut into
// clusters and phases may use different split factors); the accumulator tile is parked in a shared-memory region of its
// own (the stages belong to the next tile's weights by then); the arg-max of the vocabulary phase is one atomicMax per
// (row, tile) on the ordered 64-bit key, all CTAs but the last to arrive exit at once, and the last arriver records
// the words and packs their embedding rows for the next step.
//
// Warp roles (320 threads): warps 0-7 = two warpgroups that issue the wgmma (accumulator in registers) and run the
// epilogues, warp 8 = weight TMA warp (runs ahead across phases), warp 9 = activation TMA warp (a phase's activations
// only after the counter of the phase before says they are complete).
#include "sat_common.cuh"
#include "sat_linear.cuh"
#include "sat_linear_dev.cuh"

namespace sat {

constexpr int kChainThreads = kLinThreads;
constexpr int kChainWWarp = kLinProducers / 32;   // warp 8
constexpr int kChainXWarp = kChainWWarp + 1;      // warp 9
constexpr int kChainNT = 4;                       // accumulator fragments: row tile 64, the only one the loop uses

struct ChainJob {
    const LinProblem* P;
    int n_tile, split, kb0, nkb, tile_id, cta0;   // cta0: CTA that holds split 0 of this tile
};

__device__ __forceinline__ void chain_job(const LinChain& C, int ph, ChainJob& J) {
    J.P = &C.ph[0].p[0];
    J.n_tile = J.split = J.kb0 = J.nkb = J.tile_id = J.cta0 = 0;
    if (ph >= C.nphase) return;
    const ChainPhase& F = C.ph[ph];
    if ((int)blockIdx.x >= F.ctas) return;
    const int pi = (F.nprob > 1 && (int)blockIdx.x >= F.p[1].cta_begin) ? 1 : 0;
    const LinProblem& P = F.p[pi];
    const int local = (int)blockIdx.x - P.cta_begin;
    J.P = &P;
    J.split = local % P.splits;
    J.n_tile = local / P.splits;
    J.kb0 = (P.k_blocks * J.split) / P.splits;               // (same rounding as lin_mma_kernel's 64-bit form)
    J.nkb = (P.k_blocks * (J.split + 1)) / P.splits - J.kb0;
    J.tile_id = (pi ? F.p[0].n_tiles : 0) + J.n_tile;
    J.cta0 = (int)blockIdx.x - J.split;
}

__global__ void __launch_bounds__(kChainThreads, 1) lin_chain_kernel(const __grid_constant__ LinChain C) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint64_t* full_w = reinterpret_cast<uint64_t*>(smem_raw);  // [stages]
    uint64_t* full_x = full_w + 8;
    uint64_t* empty = full_x + 8;
    uint64_t* gather_bar = empty + 8;                            // embedding rows of the last arriver's tail
    uint64_t* peer_ready = gather_bar + 1;                       // [kChainMaxPhase] every split of my tile has parked its partial
    uint64_t* peer_done = peer_ready + kChainMaxPhase;           // [kChainMaxPhase] every split of my tile has read mine
    unsigned* flag_s = reinterpret_cast<unsigned*>(smem_raw + 256);
    int* word_s = reinterpret_cast<int*>(smem_raw + 512);      // [<= 64] words picked by the last arriver
    uint8_t* stage_base = smem_raw + 1024;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = C.stages, N = C.row_tile, mode = C.layout_mode;
    const uint32_t x_half_bytes = (uint32_t)N * kBK * 2;
    const uint32_t x_stage_bytes = 2 * x_half_bytes;
    const uint32_t stage_bytes = kWStageBytes + x_stage_bytes;
    float* tile_s = reinterpret_cast<float*>(stage_base + (size_t)S * stage_bytes);   // [N][128] fp32, own region

    ChainJob job[kChainMaxPhase];
#pragma unroll
    for (int ph = 0; ph < kChainMaxPhase; ++ph) chain_job(C, ph, job[ph]);
    unsigned long long* const dbg0 = C.dbg_mode == 0 ? C.dbg : nullptr;   // phase milestones
    unsigned long long* const dbg1 = (C.dbg_mode == 1 || C.dbg_mode == 2) ? C.dbg : nullptr;   // per-K-block stamps of phase 0
    unsigned long long* const dbg3 = C.dbg_mode == 3 ? C.dbg : nullptr;   // fine stamps of K blocks 0..3 of phase 0
    unsigned long long* const dbg4 = C.dbg_mode == 4 ? C.dbg : nullptr;   // epilogue internals: phase 0 (6..12), last arriver's tail (0..5)

    if (threadIdx.x == 0) {
        trace_stamp(dbg0, 0);
        tl_begin(C.tl);
        for (int s = 0; s < S; ++s) {
            mbar_init(&full_w[s], 1);
            mbar_init(&full_x[s], 1);
            mbar_init(&empty[s], kLinProducers / 32);   // one arrival per consumer warp once its MMAs are complete
        }
        mbar_init(gather_bar, 1);
#pragma unroll
        for (int ph = 0; ph < kChainMaxPhase; ++ph) {            // (used once each: one tile per phase and launch)
            const int sp = job[ph].nkb ? job[ph].P->splits : 1;
            mbar_init(&peer_ready[ph], (uint32_t)sp);
            mbar_init(&peer_done[ph], (uint32_t)sp);
        }
        fence_mbar_init();
    }
    __syncthreads();
    // (cluster mode: a peer may arrive on this CTA's peer_ready / peer_done barriers as soon as it runs: they must be
    // initialised cluster-wide first.  All threads, once, before anything waits for the predecessor launch.)
    if (C.cluster > 1) cluster_sync_all();

    if (warp == kChainWWarp || warp == kChainXWarp) {
        // ===================== TMA warps: warp 8 streams the weights, warp 9 the activations =====================
        // The K blocks of this CTA's tiles form one sequence over the phases.  A block's weight half is issued as soon
        // as its stage is free (weights are immutable: no dependency, so this warp runs ahead into the next phase's
        // tile under the epilogue and the rendezvous of the current one); its activation half is issued by the other
        // warp when the stage is free AND the phase before the block's own is complete grid-wide.  These loops pace the
        // whole tile, so: two warps (the wait -> arm -> issue chains of the two halves overlap), each converged with one
        // elected lane issuing (see elect_one), every decision a warp vote, everything needed a running cursor in
        // registers — no divisions, no indexed reads of the launch descriptor.
        const bool wside = warp == kChainWWarp;
        const uint64_t wpol = l2_policy(C.l2_w);
        const int l2w = wside ? C.l2_w : 0;
        const uint32_t stage0 = smem_u32(stage_base) + (wside ? 0u : (uint32_t)kWStageBytes);
        const uint32_t bar0 = smem_u32(wside ? full_w : full_x);
        const uint32_t bytes = wside ? (uint32_t)kWStageBytes : x_stage_bytes;
        int ph = -1, left = 0, st = 0, g = 0, sg = 0, seg_left = 0;
        uint32_t par = 1u;                     // parity of empty[st] that means "free" (fresh barrier: the first pass is free)
        const uint8_t* ptr = nullptr;
        const LinProblem* Pp = nullptr;
        auto next_phase = [&]() {
            while (++ph < kChainMaxPhase) {
                const int n = ph == 0 ? job[0].nkb : ph == 1 ? job[1].nkb : job[2].nkb;
                if (n == 0) continue;
                Pp = ph == 0 ? job[0].P : ph == 1 ? job[1].P : job[2].P;
                const int nt = ph == 0 ? job[0].n_tile : ph == 1 ? job[1].n_tile : job[2].n_tile;
                int kb = ph == 0 ? job[0].kb0 : ph == 1 ? job[1].kb0 : job[2].kb0;
                left = n;
                if (wside) {
                    ptr = Pp->wpack + ((size_t)nt * Pp->k_blocks + kb) * kWStageBytes;
                    seg_left = n + 1;          // (never reaches 0: the weights of a tile are contiguous)
                } else {
                    sg = 0;                    // the K block lives in the packed activation of the segment that covers it
                    while (sg + 1 < Pp->nseg && kb >= (Pp->seg[sg].width >> 6)) { kb -= Pp->seg[sg].width >> 6; ++sg; }
                    ptr = Pp->seg[sg].pa + (size_t)kb * x_stage_bytes;
                    seg_left = (Pp->seg[sg].width >> 6) - kb;
                }
                return;
            }
        };
        auto issue = [&]() {
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
                if (dbg1 && wside && ph == 0 && g < 8) trace_stamp(dbg1, 8 + g);
                if (dbg3 && !wside && ph == 0 && g < 4) trace_stamp(dbg3, g);
            }
            ptr += bytes;
            ++g;
            if (++st == S) { st = 0; par ^= 1u; }
            if (--left == 0) { next_phase(); return; }
            if (--seg_left == 0) {                 // the tile's K range continues in the next operand segment
                ++sg;
                ptr = Pp->seg[sg].pa;
                seg_left = Pp->seg[sg].width >> 6;
            }
        };
        next_phase();
        int ready_ph = kChainMaxPhase;             // (weights: every phase is "ready")
        if (!wside) {
            // activations (and everything else global) wait for the predecessor launch; launch_dependents only after the
            // wait, which keeps "a launch never starts before the predecessor of its predecessor has completed"
            if (C.pdl) { pdl_wait(); pdl_launch_dependents(); }
            if (lane == 0) {
                trace_stamp(dbg0, 1);
                tl_go(C.tl);
                if (C.tl) tl_begin(C.tl + 4);
            }
            ready_ph = 0;                          // activations of phases <= ready_ph may be fetched
        }
        // (no busy polling: these warps share their schedulers with the consumer warps, and a spinning warp takes issue
        // slots from them — the stage wait suspends in hardware (mbarrier.try_wait), the phase wait sleeps between polls)
        while (ph < kChainMaxPhase) {
            if (ph > ready_ph) {
                long long t0 = 0;
                int spins = 0;
                while (!__all_sync(0xffffffffu, (int)(ld_acquire_gpu(C.ctr + ph - 1) - C.target[ph - 1]) >= 0)) {
                    __nanosleep(128);
                    if ((++spins & 1023) == 0) {
                        if (spins == 1024) t0 = clock64();
                        else if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) {
                            __trap();   // the phase before never completed
                        }
                    }
                }
                fence_proxy_async_global();        // other SMs' (generic-proxy) stores -> visible to the TMA reads below
                ready_ph = ph;
                if (C.tl && lane == 0) tl_begin(C.tl + 4 * (1 + ph));   // (timeline) first CTA that saw the phase open
            }
            mbar_wait_mma(&empty[st], par);
            issue();
        }
    } else if (warp < kChainWWarp) {
        // ===================== consumer warpgroups (warps 0..7): MMA, epilogues =====================
        const int pt = threadIdx.x;   // 0..255
        const int u = pt & 31;
        if (C.pdl) { pdl_wait(); pdl_launch_dependents(); }
        int s = 0;                         // pipeline stage of the next K block (one sequence over the phases)
        uint32_t par = 0u;
        int wait_done_ph = -1;             // cluster mode: phase whose peer_done barrier guards tile_s
#pragma unroll 1
        for (int ph = 0; ph < C.nphase; ++ph) {
            // (selected by VALUE: a reference into job[] with a run-time index would put the array in local memory)
            const int j_nkb = ph == 0 ? job[0].nkb : ph == 1 ? job[1].nkb : job[2].nkb;
            if (j_nkb == 0) continue;
            const LinProblem* const Pp = ph == 0 ? job[0].P : ph == 1 ? job[1].P : job[2].P;
            const LinProblem& P = *Pp;
            const int split = ph == 0 ? job[0].split : ph == 1 ? job[1].split : job[2].split;
            const int n_tile = ph == 0 ? job[0].n_tile : ph == 1 ? job[1].n_tile : job[2].n_tile;
            const int j_tile_id = ph == 0 ? job[0].tile_id : ph == 1 ? job[1].tile_id : job[2].tile_id;
            const int j_cta0 = ph == 0 ? job[0].cta0 : ph == 1 ? job[1].cta0 : job[2].cta0;
            const int splits = P.splits, epi = P.epi, n_out = P.n_out, ldo = P.ldo, Hh = P.H;
            float* const out = P.out;
            uint8_t* const out_pa = P.out_pa;
            const float* const c_in = P.c_in;
            const int rows_here = min(N, P.rows);
            const int lo = (int)(((long long)rows_here * split) / splits) * 32;
            const int hi = (int)(((long long)rows_here * (split + 1)) / splits) * 32;
            const bool do_am = P.am_key != nullptr;           // (host: splits == 1 for the arg-max phase)
            const bool csplit = splits > 1 && C.cluster > 1;  // partial tiles meet in distributed shared memory
            const bool gsplit = splits > 1 && C.cluster <= 1; // ... or in the L2 scratch buffer
            const int ng = n_tile * kTileN + 4 * u;           // first of this thread's 4 outputs (all rows)
            const int unit = n_tile * 32 + u;                 // LSTM: the unit whose 4 gates this thread holds
            const bool vec_out = ng + 3 < n_out && (ldo & 3) == 0;
            const bool row_loop = epi == kEpiLstm || out != nullptr || out_pa != nullptr;
            float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (epi != kEpiNone && P.bias) bias4 = *reinterpret_cast<const float4*>(P.bias + n_tile * kTileN + 4 * u);
            const float* const bias_fold = (do_am && P.bias) ? P.bias + n_tile * kTileN : nullptr;
            float cpre[2] = {0.f, 0.f};
            if (epi == kEpiLstm && unit < Hh) {
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int idx = lo + pt + j * kLinProducers;
                    if (idx < hi) cpre[j] = c_in[(size_t)(idx >> 5) * Hh + unit];
                }
            }
            // ---- main loop: per K block, both warpgroups issue their 64 x N x 64 share of the three products
            AccTile<kChainNT> acc;
#pragma unroll 1
            for (int it = 0; it < j_nkb; ++it) {
                mbar_wait_mma(&full_w[s], par);
                if (dbg3 && ph == 0 && it < 4 && pt == 0) trace_stamp(dbg3, 12 + it);
                mbar_wait_mma(&full_x[s], par);
                if (pt == 0) {
                    if (dbg3 && ph == 0 && it < 4) trace_stamp(dbg3, 4 + it);
                    if (dbg0 && it == 0) trace_stamp(dbg0, ph == 0 ? 2 : ph == 1 ? 9 : 11);      // first operands of the phase landed
                    if (dbg1 && ph == 0 && it < 8) trace_stamp(dbg1, it);
                }
                mma_kblock(acc, smem_u32(stage_base) + (uint32_t)s * stage_bytes, x_half_bytes, mode, it == 0);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);   // frees the stage: this warp's MMAs have read it
                if (++s == S) { s = 0; par ^= 1u; }
            }
            // ---- part 1: accumulator -> shared memory (and, split-K, the rows other CTAs reduce -> L2 scratch)
            {
                if (C.tl && pt == 0) { tl_main_done(C.tl); tl_go(C.tl + 4 * (1 + ph)); tl_main_done(C.tl + 4 * (1 + ph)); }
                if (dbg0 && pt == 0) trace_stamp(dbg0, ph == 0 ? 4 : ph == 1 ? 10 : 12);
                if (dbg4 && pt == 0 && ph == 0) trace_stamp(dbg4, 6);
                float* const my_part = C.scratch + (size_t)blockIdx.x * N * kTileN;
                // (cluster mode: the peers of my PREVIOUS split tile must have finished reading tile_s before it is rewritten)
                if (wait_done_ph >= 0) { mbar_wait_cluster(&peer_done[wait_done_ph], 0u); wait_done_ph = -1; }
                acc_for_each(acc, N, [&](int m, int row, float v) {
                    tile_s[row * kTileN + m] = bias_fold ? v + bias_fold[m] : v;
                    if (gsplit && row < rows_here && (row * 32 < lo || row * 32 >= hi)) __stcg(my_part + row * kTileN + m, v);
                });
                if (dbg4 && pt == 0 && ph == 0) trace_stamp(dbg4, 7);
            }
            const uint32_t tile_addr = smem_u32(tile_s);
            uint32_t peer[8];
            if (csplit) {
                // the `splits` CTAs of the tile are consecutive ranks of one cluster: tell every one of them (and myself)
                // that my partial tile is parked, wait until all of theirs are (mbarrier, cluster scope: no
                // barrier.cluster, so the TMA / MMA warps are not involved), then CTA `split` sums rows [lo, hi) of
                // the partial tiles read through distributed shared memory, in fixed split order
                const uint32_t rank0 = cluster_ctarank() - (uint32_t)split;
#pragma unroll
                for (int r = 0; r < 8; ++r) peer[r] = r < splits ? dsmem_map(tile_addr, rank0 + (uint32_t)r) : tile_addr;
                named_bar_sync(1, kLinProducers);
                if (dbg4 && pt == 0 && ph == 0) trace_stamp(dbg4, 8);
                if (pt < splits) mbar_arrive_remote(&peer_ready[ph], rank0 + (uint32_t)pt);
                mbar_wait_cluster(&peer_ready[ph], 0u);
                if (pt == 0 && ph == 0) { trace_stamp(dbg0, 6); trace_stamp(dbg4, 9); }
            } else if (gsplit) {
                // the `splits` CTAs of the tile meet at its arrival counter; afterwards CTA `split` sums rows [lo, hi)
                __threadfence();
                named_bar_sync(1, kLinProducers);
                if (dbg4 && pt == 0 && ph == 0) trace_stamp(dbg4, 8);
                if (pt == 0) {
                    unsigned* tc = C.tile_ctr + ph * kChainMaxTiles + j_tile_id;
                    atomicAdd(tc, 1u);
                    wait_counter_mma(tc, C.tile_target[ph]);   // split-K rendezvous
                    __threadfence();
                    if (ph == 0) trace_stamp(dbg0, 6);
                    if (ph == 0) trace_stamp(dbg4, 9);
                }
                named_bar_sync(1, kLinProducers);
            } else {
                named_bar_sync(1, kLinProducers);
            }
            // ---- part 2: one warp = one activation row per iteration (lane u owns outputs 4u..4u+3)
            if (row_loop) {
                // split-K: the other splits' partial rows come from L2 (one round trip).  A thread has at most two rows at
                // the batch sizes this launch serves; the loads of BOTH are issued before the first is consumed.
                auto remote = [&](int r, int bb) {
                    if (csplit) return ld_dsmem_f4(peer[r] + (uint32_t)(bb * kTileN + 4 * u) * 4u);
                    return __ldcg(reinterpret_cast<const float4*>(C.scratch + (size_t)(j_cta0 + r) * N * kTileN + bb * kTileN + 4 * u));
                };
                // (eight registers-quads in all: splits <= 4 -> pfa = first row, pfb = second row; splits == 8 -> one row,
                // pfa = splits 0..3, pfb = splits 4..7)
                float4 pfa[4], pfb[4];
                const int idx0 = lo + pt, idx1 = idx0 + kLinProducers;
                const bool wide = splits > 4;
                const bool pre1 = splits > 1 && !wide && idx1 < hi;
                if (splits > 1 && idx0 < hi) {
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        if (r < splits && r != split) pfa[r] = remote(r, idx0 >> 5);
                        if (wide && r + 4 < splits && r + 4 != split) pfb[r] = remote(r + 4, idx0 >> 5);
                    }
                }
                if (pre1) {
#pragma unroll
                    for (int r = 0; r < 4; ++r)
                        if (r < splits && r != split) pfb[r] = remote(r, idx1 >> 5);
                }
#pragma unroll 1
                for (int idx = idx0; idx < hi; idx += kLinProducers) {
                    const int bb = idx >> 5;
                    float4 g;
                    if (splits == 1) {
                        g = *reinterpret_cast<const float4*>(tile_s + bb * kTileN + 4 * u);
                    } else {
                        const float4 own = *reinterpret_cast<const float4*>(tile_s + bb * kTileN + 4 * u);
                        float4 part[8];
#pragma unroll
                        for (int r = 0; r < 8; ++r)
                            if (r < splits)
                                part[r] = r == split ? own
                                          : idx == idx0 ? (r < 4 ? pfa[r & 3] : pfb[r & 3])
                                          : (idx == idx1 && pre1) ? pfb[r & 3]
                                                                  : remote(r, bb);
                        g = part[0];   // fixed split order: bit-identical to the cluster reduction of lin_mma_kernel
#pragma unroll
                        for (int r = 1; r < 8; ++r)
                            if (r < splits) { g.x += part[r].x; g.y += part[r].y; g.z += part[r].z; g.w += part[r].w; }
                    }
                    if (!do_am) { g.x += bias4.x; g.y += bias4.y; g.z += bias4.z; g.w += bias4.w; }
                    if (dbg4 && pt == 0 && ph == 0 && idx == idx0 && g.x != 12345.678f) trace_stamp(dbg4, 10);   // first row's partials arrived
                    if (epi == kEpiLstm) {
                        float cprev = idx == lo + pt ? cpre[0] : cpre[1];
                        if (unit < Hh && idx >= lo + pt + 2 * kLinProducers) cprev = c_in[(size_t)bb * Hh + unit];
                        if (unit < Hh) lstm_gates(P, g, cprev, bb, unit, mode, false);
                        continue;
                    }
                    if (epi == kEpiBiasTanh) { g.x = act_tanh(g.x); g.y = act_tanh(g.y); g.z = act_tanh(g.z); g.w = act_tanh(g.w); }
                    if (out) {
                        float* o = out + (size_t)bb * ldo + ng;
                        if (vec_out) {
                            *reinterpret_cast<float4*>(o) = g;
                        } else {
                            if (ng + 0 < n_out) o[0] = g.x;
                            if (ng + 1 < n_out) o[1] = g.y;
                            if (ng + 2 < n_out) o[2] = g.z;
                            if (ng + 3 < n_out) o[3] = g.w;
                        }
                    }
                    if (out_pa) {
                        const float y[4] = {g.x, g.y, g.z, g.w};
                        if (ng + 3 < n_out) {
                            pa_store4(out_pa, mode, N, n_out >> 6, bb, ng, y);
                        } else {
#pragma unroll 1
                            for (int e = 0; e < 4; ++e)
                                if (ng + e < n_out) pa_store(out_pa, mode, N, n_out >> 6, bb, ng + e, y[e]);
                        }
                    }
                }
            }
            if (do_am) {
                // greedy prediction (model.py:289): 4 threads per row scan the tile's 128 finished values (bias folded in
                // part 1) as ordered 64-bit keys (value, then inverted index: max = first maximum, like tf.argmax) and
                // the tile's best goes into the row's global key with one atomicMax (order independent: deterministic)
                const int part = pt & 3;
#pragma unroll 1
                for (int r0 = 0; r0 < rows_here; r0 += kLinProducers / 4) {
                    const int r = r0 + (pt >> 2);
                    const bool live = r < rows_here;
                    const float4* row_t = reinterpret_cast<const float4*>(tile_s + (live ? r : 0) * kTileN) + part * 8;
                    unsigned long long k0 = 0ull, k1 = 0ull;
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
                    unsigned long long key = max(k0, k1);
                    key = max(key, __shfl_xor_sync(0xffffffffu, key, 1));
                    key = max(key, __shfl_xor_sync(0xffffffffu, key, 2));
                    if (live && part == 0) atomicMax(P.am_key + r, key);
                }
            }
            if (csplit) {
                // my reads of the peers' tiles are complete (the loads above returned their data): every peer may reuse
                // its tile buffer or exit; mine is guarded by my own peer_done barrier until all of them said the same
                named_bar_sync(1, kLinProducers);
                const uint32_t rank0 = cluster_ctarank() - (uint32_t)split;
                if (pt < splits) mbar_arrive_remote(&peer_done[ph], rank0 + (uint32_t)pt);
                wait_done_ph = ph;
            }
            if (dbg0 && pt == 0 && ph == 0) trace_stamp(dbg0, 7);
            if (dbg4 && pt == 0 && ph == 0) trace_stamp(dbg4, 11);
            // ---- this CTA's part of the phase is complete and visible (also to the TMA reads of the CTAs that fetch
            // the packed outputs): arrive at the phase counter
            __threadfence();
            fence_proxy_async_global();
            named_bar_sync(1, kLinProducers);
            if (pt == 0) {
                if (C.tl) tl_end(C.tl + 4 * (1 + ph));
                const unsigned old = atomicAdd(C.ctr + ph, 1u);
                flag_s[0] = (do_am && old + 1u == C.target[ph]) ? 1u : 0u;
                if (dbg0) trace_stamp(dbg0, ph == 0 ? 8 : ph == 1 ? 15 : 13);
                if (dbg4 && ph == 0) trace_stamp(dbg4, 12);
                if (dbg4 && flag_s[0]) trace_stamp(dbg4, 0);
            }
            if (do_am) {
                named_bar_sync(1, kLinProducers);
                if (flag_s[0]) {
                    // last CTA of the vocabulary phase: every row's key is final.  Record the words (and the word fed
                    // to the next step: the prediction, or the forced word of teacher forcing, model.py:310) and hand
                    // the embedding rows of the fed words (model.py:272-274), packed, to the next step's layers.
                    __threadfence();
                    const int rows = P.rows;
                    for (int r = pt; r < rows; r += kLinProducers) {
                        const unsigned long long best = atomicExch(P.am_key + r, 0ull);   // (and ready for the next launch)
                        const int bi = argmax_key_index(best);
                        const int nw = P.am_forced ? P.am_forced[(size_t)r * P.am_forced_ld + P.am_step] : bi;
                        if (P.am_tokens) P.am_tokens[(size_t)r * P.am_tokens_ld + P.am_step] = bi;
                        if (P.am_next_word) P.am_next_word[r] = nw;
                        word_s[r] = nw;
                    }
                    named_bar_sync(1, kLinProducers);
                    if (dbg0 && pt == 0) trace_stamp(dbg0, 14);
                    if (dbg4 && pt == 0) trace_stamp(dbg4, 1);
                    if (P.am_emb_pa) {
                        // 64 rows x 2 KB from a 20 MB table: mostly HBM misses, and one SM sustains too few outstanding
                        // loads to fetch 128 KB with ld.global in less than ~7 us (measured).  The pipeline stages are
                        // idle by now (this is the launch's last tile), so the rows are fetched by bulk TMA into them
                        // (each warp issues its rows), then converted from shared memory.
                        const int E = P.am_E, G8 = E >> 3, total = rows * G8;
                        const size_t halfb = (size_t)N * kBK * 2;
                        const uint32_t row_bytes = (uint32_t)E * 4u;
                        // (row pitch = row + 16 bytes: the conversion below reads 8 rows at the same column at once)
                        const uint32_t row_pitch = row_bytes + 16u;
                        const bool fits = (size_t)rows * row_pitch <= (size_t)S * stage_bytes && (row_bytes & 15u) == 0;
                        const uint8_t* const rows_s = stage_base;
                        if (fits) {
                            if (pt == 0) mbar_arrive_expect_tx(gather_bar, (uint32_t)rows * row_bytes);
                            named_bar_sync(1, kLinProducers);                 // (armed before any copy can complete)
                            const int w8 = pt >> 5;
                            for (int r = w8; r < rows; r += kLinProducers / 32)
                                if (elect_one())
                                    tma_bulk_g2s(stage_base + (size_t)r * row_pitch, P.am_emb + (size_t)word_s[r] * E, row_bytes, gather_bar);
                            if (dbg4 && pt == 0) trace_stamp(dbg4, 2);
                            mbar_wait_mma(gather_bar, 0);
                            if (dbg4 && pt == 0) trace_stamp(dbg4, 3);
                        }
                        // conversion fp32 -> packed bf16 hi / lo.  Task t = one 16-byte group of the destination; the low
                        // task bits run over (row & 7, k-group & 3) so that a warp's stores fill whole 128-byte lines of
                        // the operand image (row-major task order made every 16-byte store its own sector: ~4 us)
                        const int KB8 = E >> 6;                                     // K blocks of the operand
                        const int nrb = (rows + 7) >> 3;                            // 8-row blocks
                        (void)total;
                        // thread-constant low bits (the stride of 256 tasks keeps them), the rest advances by 4 per step:
                        // no division in the loop
                        const int r7 = pt & 7, kg = ((pt >> 3) & 3) | (((pt >> 5) & 1) << 2);
                        int kb = (pt >> 6) % KB8, rblk = (pt >> 6) / KB8;
                        constexpr int GB = 4;
#pragma unroll 1
                        while (rblk < nrb) {
                            float4 a4[GB], c4[GB];
                            int kbs[GB], rs[GB];
#pragma unroll
                            for (int j = 0; j < GB; ++j) {
                                kbs[j] = kb;
                                rs[j] = rblk < nrb ? rblk * 8 + r7 : rows;          // (rows: nothing to do)
                                if (rs[j] < rows) {
                                    const int g8 = kb * 8 + kg;
                                    const float4* src = fits ? reinterpret_cast<const float4*>(rows_s + (size_t)rs[j] * row_pitch + (size_t)g8 * 32)
                                                             : reinterpret_cast<const float4*>(P.am_emb + (size_t)word_s[rs[j]] * E + g8 * 8);
                                    a4[j] = src[0];
                                    c4[j] = src[1];
                                }
                                kb += 4;
                                while (kb >= KB8) { kb -= KB8; ++rblk; }
                            }
#pragma unroll
                            for (int j = 0; j < GB; ++j) {
                                if (rs[j] < rows) {
                                    uint4 hi4, lo4;
                                    split_bf16x8(a4[j], c4[j], hi4, lo4);
                                    uint8_t* dst = P.am_emb_pa + (size_t)kbs[j] * 2 * halfb + mma_tile_off(mode, rs[j], kg);
                                    *reinterpret_cast<uint4*>(dst) = hi4;
                                    *reinterpret_cast<uint4*>(dst + halfb) = lo4;
                                }
                            }
                        }
                    }
                }
            }
            if (dbg4 && pt == 0 && do_am && flag_s[0]) trace_stamp(dbg4, 4);
        }
        // (cluster mode: a CTA's shared memory must outlive the peers' reads of it)
        if (wait_done_ph >= 0) mbar_wait_cluster(&peer_done[wait_done_ph], 0u);
    }
    __syncthreads();
    if (threadIdx.x == 0) { trace_stamp(dbg0, 5); trace_stamp(dbg4, 5); tl_end(C.tl); }
}

// ------------------------------------------------------------ host side
static int g_chain_optin = 0;

size_t lin_chain_smem_bytes(int row_tile, int stages) {
    return 1024 + (size_t)stages * (kWStageBytes + 2 * (size_t)row_tile * kBK * 2) + (size_t)row_tile * kTileN * 4;
}

int lin_chain_pick_stages(int row_tile) {
    if (g_chain_optin == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 0;
        if (cudaDeviceGetAttribute(&g_chain_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return 0;
        if (cudaFuncSetAttribute(lin_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, g_chain_optin) != cudaSuccess) return 0;
    }
    const long long budget = (long long)g_chain_optin - 1024 - (long long)row_tile * kTileN * 4;
    const long long per = kWStageBytes + 2 * (long long)row_tile * kBK * 2;
    long long s = budget / per;
    if (s > 8) s = 8;
    return s < 0 ? 0 : (int)s;
}

// clusters of `cluster` CTAs of this kernel that can be resident at once (0 on error): a chained launch waits on
// grid-wide counters, so ALL its clusters must be
int lin_chain_max_clusters(int row_tile, int stages, int cluster) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cluster * 64);
    cfg.blockDim = dim3(kChainThreads);
    cfg.dynamicSmemBytes = lin_chain_smem_bytes(row_tile, stages);
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)cluster;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, lin_chain_kernel, &cfg) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

cudaError_t lin_chain_launch(const LinChain& C, int grid, cudaStream_t st) {
    if (C.stages < 2 || C.row_tile != 16 * kChainNT) return cudaErrorInvalidValue;   // (the MMA width is the row tile)
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kChainThreads);
    cfg.dynamicSmemBytes = lin_chain_smem_bytes(C.row_tile, C.stages);
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (C.cluster > 1) {
        if (grid % C.cluster) return cudaErrorInvalidValue;
        at[na].id = cudaLaunchAttributeClusterDimension;
        at[na].val.clusterDim.x = (unsigned)C.cluster;
        at[na].val.clusterDim.y = 1;
        at[na].val.clusterDim.z = 1;
        ++na;
    }
    if (C.pdl) {
        at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = at;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, lin_chain_kernel, C);
}

}  // namespace sat
