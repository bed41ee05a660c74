// sat_common.cuh — sm_90a PTX wrappers shared by the sat_b200 kernels:
// mbarrier, TMA (cp.async.bulk / cp.async.bulk.tensor), wgmma (warpgroup MMA
// from shared-memory descriptors), proxy fences.  Hand-written inline PTX; no
// CUTLASS/CuTe dependency.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#ifndef SAT_SPIN_LIMIT_CYCLES
// A barrier wait that lasts longer than this many SM cycles (~4 s) is a bug:
// trap instead of hanging the GPU.
#define SAT_SPIN_LIMIT_CYCLES (8000000000ll)
#endif

namespace sat {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a system-dependent time; a polling loop that also
// watches something else wants test_wait)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) {
            printf("sat_b200: mbarrier wait timed out (block %d thread %d)\n", (int)blockIdx.x, (int)threadIdx.x);
            __trap();
        }
    }
}
// Kernels that issue wgmma (sat_linear.cu, sat_chain.cu) use the _mma forms of the waits: no printf, because a call
// (vprintf) anywhere in such a kernel makes ptxas serialise its MMAs (C7510).  A hang there ends in a bare trap.
__device__ __forceinline__ void mbar_wait_mma(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) __trap();
}

// ----------------------------------------------------------------------- TMA
// 1-D bulk copy global -> shared, completion on an mbarrier (UBLKCP).
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// Bring a span of global memory into L2 without a destination (no shared memory, no barrier): used by kernels that
// were launched early (programmatic dependent launch) to pull their weight stream towards the SMs while the
// predecessor is still in its tail and the HBM channels are idle.
__device__ __forceinline__ void prefetch_l2_bulk(const void* src_gmem, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src_gmem), "r"(bytes) : "memory");
}
// L2 eviction-priority policies for TMA loads: 0 = none, 1 = evict_first (streamed once per step),
// 2 = evict_last (data re-read while it is still in L2), 3 = evict_normal.  The 50 MB L2 of an H100 cannot keep
// the weights of a decode step across steps (see plan() in sat_api.cu for the policy of the dense weight streams).
__device__ __forceinline__ uint64_t l2_policy(int kind) {
    uint64_t pol = 0;
    if (kind == 1) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    else if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    else if (kind == 3) asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tma_bulk_g2s_hint(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar,
                                                  int kind, uint64_t pol) {
    if (kind == 0) {
        tma_bulk_g2s(dst_smem, src_gmem, bytes, bar);
        return;
    }
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}
__device__ __forceinline__ void tma_tensor2d_g2s_hint(void* dst_smem, const void* tmap, int c0, int c1, uint64_t* bar,
                                                      int kind, uint64_t pol);

// 2-D tiled tensor copy global -> shared through a CUtensorMap (UTMALDG).
__device__ __forceinline__ void tma_tensor2d_g2s(void* dst_smem, const void* tmap, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::
            "r"(smem_u32(dst_smem)),
        "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_tensor2d_g2s_hint(void* dst_smem, const void* tmap, int c0, int c1, uint64_t* bar,
                                                      int kind, uint64_t pol) {
    if (kind == 0) {
        tma_tensor2d_g2s(dst_smem, tmap, c0, c1, bar);
        return;
    }
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint "
        "[%0], [%1, {%2, %3}], [%4], %5;" ::"r"(smem_u32(dst_smem)),
        "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "l"(pol)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// generic-proxy global writes (possibly by other SMs, already acquired) -> visible to TMA reads
__device__ __forceinline__ void fence_proxy_async_global() {
    asm volatile("fence.proxy.async.global;" ::: "memory");
}

// One lane of a CONVERGED warp (elect.sync).  The async-unit instructions (cp.async.bulk) take their
// operands from the uniform register file: issued from `if (lane == 0)` code their addresses live in per-thread registers
// and every instruction costs a handful of register->uniform moves plus an elect/branch loop; issued as `if (elect_one()) ...` from a loop the whole warp runs, the operands are
// computed in uniform registers to begin with.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// --------------------------------------------------------------------- wgmma
// Warpgroup MMA: the four warps of an aligned warpgroup issue together, the accumulator lives in their registers.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// d[64 x N] (+)= A[64 x 16] * B[N x 16]^T for N = 16, 32, ..., 128: bf16 inputs from shared-memory descriptors, both
// K-major, fp32 accumulate; scale_d == 0: d = A * B (the previous contents are ignored), else d += A * B.
// Fragment of thread t of the warpgroup (w = t / 32, l = t % 32): d[4i + 2h + e] is row w*16 + l/4 + 8h, column
// 8i + 2(l%4) + e.
template <int N>
struct Wgmma;

template <>
struct Wgmma<16> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<48> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<80> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<96> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<112> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55}, %56, %57, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};

template <>
struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(desc_a), "l"(desc_b), "r"(scale_d)
            : "memory");
    }
};
// pins the n accumulator registers at this point of the instruction stream (no access is moved across it)
__device__ __forceinline__ void wgmma_fence_operand(float* d, int n) {
#pragma unroll
    for (int i = 0; i < n; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of wgmma (sm_90 format).
//   bits [0,14)  start address >> 4      bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4 bits [62,64) layout: 0 = no swizzle (interleave), 1 = 128B swizzle
__device__ __forceinline__ uint64_t gmma_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t layout) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)(layout & 3) << 62;
    return d;
}

// ------------------------------------------------ programmatic dependent launch
// A kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start while its predecessor in
// the stream is still draining; it must not touch memory the predecessor (or anything before it) writes, nor
// write anything they read, before pdl_wait() returns (= all prerequisite grids complete and flushed).
// Every kernel here calls pdl_launch_dependents() only after its own pdl_wait(): a kernel therefore never starts
// before the predecessor of its predecessor has completed, and may read that older data without waiting.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ------------------------------------------------ thread-block clusters / distributed shared memory
__device__ __forceinline__ void cluster_sync_all() {   // every thread of every CTA of the cluster
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// split form for a barrier that only orders "I am done reading your shared memory" (no data is published)
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t dsmem_map(uint32_t local_smem_addr, uint32_t cta_rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
    return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t cluster_addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "r"(cluster_addr)
                 : "memory");
    return v;
}

// mbarrier signalling between the CTAs of a cluster (no barrier.cluster: only the threads that need it take part)
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// arrive on an mbarrier in the shared memory of CTA `cta_rank` of this cluster; release at cluster scope: the writes of
// this thread (and, through a preceding bar.sync, of its CTA) are visible to whoever acquires the barrier's phase
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* local_bar, uint32_t cta_rank) {
    const uint32_t raddr = dsmem_map(smem_u32(local_bar), cta_rank);
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(raddr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    uint32_t ok = 0;
    long long t0 = 0;
    int spins = 0;
    while (true) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(a), "r"(parity)
            : "memory");
        if (ok) return;
        if ((++spins & 255) == 0) {
            if (spins == 256) t0 = clock64();
            else if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) __trap();   // cluster mbarrier wait (wgmma kernels only)
        }
    }
}

// in-kernel timeline stamps (debug option "trace"): ns since an arbitrary origin, one row of 16 per CTA
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void trace_stamp(unsigned long long* dbg, int slot) {
    if (dbg) dbg[(size_t)blockIdx.x * 16 + slot] = globaltimer_ns();
}

// loop timeline (debug option "trace" = 3): per launch four cells: min CTA start, max CTA end, min "go" (first
// CTA past its dependency wait), max "main loop done" (accumulator complete / streaming complete)
__device__ __forceinline__ void tl_begin(unsigned long long* tl) {
    if (tl) atomicMin(tl, globaltimer_ns());
}
__device__ __forceinline__ void tl_end(unsigned long long* tl) {
    if (tl) atomicMax(tl + 1, globaltimer_ns());
}
__device__ __forceinline__ void tl_go(unsigned long long* tl) {
    if (tl) atomicMin(tl + 2, globaltimer_ns());
}
__device__ __forceinline__ void tl_main_done(unsigned long long* tl) {
    if (tl) atomicMax(tl + 3, globaltimer_ns());
}

// --------------------------------------------------------------- misc math
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
// Activations of the fused dense epilogues.  Those epilogues run once per launch from a cold instruction cache,
// so they are built from the short ex2/rcp forms: a handful of instructions each, absolute error ~2e-7 (the
// parity budget of the decode path is 1e-3 relative).
__device__ __forceinline__ float act_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float act_tanh(float x) {
    const float e = __expf(-2.0f * fabsf(x));                 // in (0, 1]: no overflow, no cancellation blow-up
    return copysignf(__fdividef(1.0f - e, 1.0f + e), x);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// spin until a monotonic arrival counter has reached `target` (wrap-safe); traps instead of hanging the GPU
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p);
__device__ __forceinline__ void wait_counter(const unsigned* ctr, unsigned target, const char* what) {
    if ((int)(ld_acquire_gpu(ctr) - target) >= 0) return;
    const long long t0 = clock64();
    while ((int)(ld_acquire_gpu(ctr) - target) < 0) {
        if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) {
            printf("sat_b200: %s timed out (block %d)\n", what, (int)blockIdx.x);
            __trap();
        }
    }
}
__device__ __forceinline__ void wait_counter_mma(const unsigned* ctr, unsigned target) {   // (see mbar_wait_mma)
    const long long t0 = clock64();
    while ((int)(ld_acquire_gpu(ctr) - target) < 0)
        if (clock64() - t0 > SAT_SPIN_LIMIT_CYCLES) __trap();
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

}  // namespace sat
