// tools/stream_bench.cu — per-SM ingest rate of 1-D bulk TMA (cp.async.bulk global -> shared) on H100.
// Each CTA streams `per_cta` bytes through a ring of `nslots` x `chunk` bytes with no compute (one lane issues, the same
// lane waits and releases), from (a) an L2-resident region (every CTA re-reads a small window) or (b) HBM (disjoint
// regions, buffer >> L2).  Answers: what is the most one SM can pull, and how does it scale with the number of SMs
// pulling at once?  (The decode step's dense CTAs and attention CTAs all sit at ~55 GB/s per SM.)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/stream_bench tools/stream_bench.cu && tools/stream_bench
// `tools/stream_bench --residency` measures instead how much evict_last data survives streaming (see residency()).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma(void* dst, const void* src, uint32_t bytes, uint64_t* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(b)) : "memory");
}

__global__ void stream_kernel(const uint8_t* src, size_t region, size_t stride, int chunk, int nslots, int nchunks, unsigned long long* t) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
    uint8_t* ring = smem + 1024;
    if (threadIdx.x == 0) {
        for (int s = 0; s < nslots; ++s) mbar_init(&bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint8_t* base = src + (size_t)blockIdx.x * stride;
        unsigned long long t0;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        int issued = 0;
        for (; issued < nslots && issued < nchunks; ++issued) {
            mbar_expect(&bar[issued], chunk);
            tma(ring + (size_t)issued * chunk, base + ((size_t)issued * chunk) % region, chunk, &bar[issued]);
        }
        for (int i = 0; i < nchunks; ++i) {
            const int s = i % nslots;
            mbar_wait(&bar[s], (i / nslots) & 1);
            if (issued < nchunks) {      // the slot is free at once (no consumer): refill it
                mbar_expect(&bar[s], chunk);
                tma(ring + (size_t)s * chunk, base + ((size_t)issued * chunk) % region, chunk, &bar[s]);
                ++issued;
            }
        }
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        t[2 * blockIdx.x] = t0;
        t[2 * blockIdx.x + 1] = t1;
    }
}

__global__ void stream_group_kernel(const uint8_t* src, size_t region, int share, int chunk, int nslots, int nchunks, unsigned long long* t) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
    uint8_t* ring = smem + 1024;
    if (threadIdx.x == 0) {
        for (int s = 0; s < nslots; ++s) mbar_init(&bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint8_t* base = src + (size_t)(blockIdx.x / share) * region;
        const int per = (int)(region / chunk);
        unsigned long long t0;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        int issued = 0, off = 0;
        for (; issued < nslots && issued < nchunks; ++issued) {
            mbar_expect(&bar[issued], chunk);
            tma(ring + (size_t)issued * chunk, base + (size_t)off * chunk, chunk, &bar[issued]);
            if (++off == per) off = 0;
        }
        for (int i = 0; i < nchunks; ++i) {
            const int s = i % nslots;
            mbar_wait(&bar[s], (i / nslots) & 1);
            if (issued < nchunks) {
                mbar_expect(&bar[s], chunk);
                tma(ring + (size_t)s * chunk, base + (size_t)off * chunk, chunk, &bar[s]);
                if (++off == per) off = 0;
                ++issued;
            }
        }
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        t[2 * blockIdx.x] = t0;
        t[2 * blockIdx.x + 1] = t1;
    }
}

// Residency mode: CTA i bulk-reads slice i of [src, src + bytes) through a ring, every copy carrying the L2 policy
// `kind` (1 = evict_first, 2 = evict_last).  Stamps {start, end} per CTA with %globaltimer.
__global__ void pass_kernel(const uint8_t* src, size_t bytes, int kind, int chunk, int nslots, unsigned long long* t) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
    uint8_t* ring = smem + 1024;
    if (threadIdx.x != 0) return;
    uint64_t pol;
    if (kind == 2) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    else asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    for (int s = 0; s < nslots; ++s) mbar_init(&bar[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const size_t total = bytes / chunk;
    const size_t c0 = total * blockIdx.x / gridDim.x, c1 = total * (blockIdx.x + 1) / gridDim.x;
    const int n = (int)(c1 - c0);
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    auto issue = [&](int i) {
        const int s = i % nslots;
        mbar_expect(&bar[s], chunk);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
                         "r"(smem_u32(ring + (size_t)s * chunk)), "l"(src + (c0 + i) * chunk), "r"(chunk), "r"(smem_u32(&bar[s])), "l"(pol)
                     : "memory");
    };
    int issued = 0;
    for (; issued < nslots && issued < n; ++issued) issue(issued);
    for (int i = 0; i < n; ++i) {
        mbar_wait(&bar[i % nslots], (i / nslots) & 1);
        if (issued < n) issue(issued++);
    }
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    t[2 * blockIdx.x] = t0;
    t[2 * blockIdx.x + 1] = t1;
}

// How much evict_last data survives a decode step's streaming?  Every SM reads a resident region of R MB with
// evict_last, then S MB of distinct data with evict_first, and again; the time of the R pass after the streaming pass
// is printed next to the same pass read right after a cold pass and to a pass over an evicted region (all HBM).  The
// largest R whose pass after streaming still runs at L2 rate (on an H100: ~6 TB/s, against ~2.2 TB/s from HBM) is the
// residency budget of the L2.
static int residency(int grid, unsigned long long* t) {
    const int chunk = 16 * 1024, nslots = 8;
    const size_t smem = 1024 + (size_t)nslots * chunk;
    const size_t S = (size_t)128 << 20, flush = (size_t)512 << 20;
    uint8_t *res, *str, *fl;
    if (cudaMalloc(&res, (size_t)64 << 20) != cudaSuccess || cudaMalloc(&str, S) != cudaSuccess ||
        cudaMalloc(&fl, flush) != cudaSuccess) { printf("error: cudaMalloc\n"); return 1; }
    cudaMemset(res, 1, (size_t)64 << 20);
    cudaMemset(str, 2, S);
    cudaFuncSetAttribute(pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    std::vector<unsigned long long> h(2 * grid);
    auto span_us = [&]() {
        cudaMemcpy(h.data(), t, sizeof(unsigned long long) * 2 * grid, cudaMemcpyDeviceToHost);
        unsigned long long a = ~0ull, b = 0;
        for (int i = 0; i < grid; ++i) { a = std::min(a, h[2 * i]); b = std::max(b, h[2 * i + 1]); }
        return (b - a) / 1e3;
    };
    auto pass = [&](const uint8_t* p, size_t bytes, int kind) {
        pass_kernel<<<grid, 32, smem>>>(p, bytes, kind, chunk, nslots, t);
        return cudaDeviceSynchronize() == cudaSuccess;
    };
    printf("residency: grid %d, resident pass evict_last, streaming pass of %zu MB evict_first (median of 9)\n", grid, S >> 20);
    printf("R_MB,us_after_stream,us_back_to_back,us_cold,GBps_after_stream,GBps_back_to_back,GBps_cold\n");
    for (int rmb = 8; rmb <= 48; rmb += 4) {
        const size_t R = (size_t)rmb << 20;
        std::vector<double> after, b2b, cold;
        for (int rep = 0; rep < 9; ++rep) {
            cudaMemset(fl, rep, flush);                       // evict everything
            if (!pass(res, R, 2)) { printf("error: pass\n"); return 1; }
            cold.push_back(span_us());
            if (!pass(res, R, 2)) return 1;
            b2b.push_back(span_us());
            for (int it = 0; it < 3; ++it) {                  // steady state: resident pass, streaming pass, ...
                if (!pass(str, S, 1) || !pass(res, R, 2)) return 1;
            }
            after.push_back(span_us());
        }
        auto med = [](std::vector<double> v) { std::sort(v.begin(), v.end()); return v[v.size() / 2]; };
        const double a = med(after), b = med(b2b), c = med(cold);
        printf("%d,%.2f,%.2f,%.2f,%.0f,%.0f,%.0f\n", rmb, a, b, c, R / a / 1e3, R / b / 1e3, R / c / 1e3);
    }
    cudaFree(res); cudaFree(str); cudaFree(fl);
    return 0;
}

int main(int argc, char** argv) {
    const size_t buf_bytes = (size_t)2 << 30;
    if (argc > 1 && !strcmp(argv[1], "--residency")) {
        int dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceProp prop;
        cudaGetDeviceProperties(&prop, dev);
        printf("device %s, %d SMs, L2 %d MB\n", prop.name, sms, prop.l2CacheSize >> 20);
        unsigned long long* t;
        cudaMalloc(&t, 2 * sizeof(unsigned long long) * sms);
        return residency(sms, t);
    }
    uint8_t* buf;
    cudaMalloc(&buf, buf_bytes);
    cudaMemset(buf, 1, buf_bytes);
    unsigned long long* t;
    cudaMalloc(&t, 2 * 132 * 8);
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    unsigned long long h[2 * 132];
    printf("source,grid,chunk_KB,ring_KB,per_cta_MB,GBps_per_SM_mean,GBps_per_SM_min,aggregate_TBps\n");
    // (c) the dense layers' activation operand: the SAME L2-resident blocks fetched by many CTAs at once
    for (int share : {4, 32, 128})
        for (int grid : {128})
            for (int chunk : {16 * 1024, 32 * 1024}) {
                const int ring = 64 * 1024, nslots = ring / chunk;
                const size_t per_cta = (size_t)4 << 20;
                const int nchunks = (int)(per_cta / chunk);
                const size_t region = (size_t)128 << 10;          // a 128 KB window per group of `share` CTAs
                for (int rep = 0; rep < 3; ++rep) {
                    stream_kernel<<<grid, 32, 1024 + (size_t)nslots * chunk>>>(buf, region, 0, chunk, nslots, nchunks, t);   // stride 0 ...
                    cudaDeviceSynchronize();
                }
                // groups: CTA i reads window (i / share)
                stream_group_kernel<<<grid, 32, 1024 + (size_t)nslots * chunk>>>(buf, region, share, chunk, nslots, nchunks, t);
                cudaDeviceSynchronize();
                stream_group_kernel<<<grid, 32, 1024 + (size_t)nslots * chunk>>>(buf, region, share, chunk, nslots, nchunks, t);
                cudaError_t e = cudaDeviceSynchronize();
                if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
                cudaMemcpy(h, t, sizeof(unsigned long long) * 2 * grid, cudaMemcpyDeviceToHost);
                double mean = 0, mn = 1e30;
                unsigned long long a = ~0ull, b = 0;
                for (int i = 0; i < grid; ++i) {
                    const double gbps = (double)nchunks * chunk / (double)(h[2 * i + 1] - h[2 * i]);
                    mean += gbps / grid;
                    if (gbps < mn) mn = gbps;
                    if (h[2 * i] < a) a = h[2 * i];
                    if (h[2 * i + 1] > b) b = h[2 * i + 1];
                }
                printf("l2-shared-by-%d,%d,%d,%d,%.0f,%.1f,%.1f,%.2f\n", share, grid, chunk / 1024, ring / 1024, per_cta / 1048576.0, mean, mn,
                       (double)nchunks * chunk * grid / (double)(b - a) / 1e3);
            }
    for (int hbm = 0; hbm < 2; ++hbm)
        for (int grid : {1, 16, 64, 79, 128, 132})
            for (int chunk : {16 * 1024, 32 * 1024, 48 * 1024})
                for (int ring : {96 * 1024, 192 * 1024}) {
                    const int nslots = ring / chunk;
                    if (nslots < 2) continue;
                    const size_t per_cta = hbm ? (size_t)12 << 20 : (size_t)8 << 20;
                    const int nchunks = (int)(per_cta / chunk);
                    // L2: every CTA cycles over its own 256 KB window (132 x 256 KB = 33 MB, resident after the warm-up
                    // run); HBM: disjoint 12 MB regions, and a 2 GB buffer swept between runs
                    const size_t region = hbm ? per_cta : (size_t)256 << 10;
                    const size_t stride = hbm ? per_cta : region;
                    for (int rep = 0; rep < 3; ++rep) {
                        if (hbm) cudaMemset(buf + ((size_t)1 << 30), rep, (size_t)512 << 20);   // flush L2
                        stream_kernel<<<grid, 32, 1024 + (size_t)nslots * chunk>>>(buf, region, stride, chunk, nslots, nchunks, t);
                        cudaError_t e = cudaDeviceSynchronize();
                        if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
                    }
                    cudaMemcpy(h, t, sizeof(unsigned long long) * 2 * grid, cudaMemcpyDeviceToHost);
                    double mean = 0, mn = 1e30;
                    unsigned long long a = ~0ull, b = 0;
                    for (int i = 0; i < grid; ++i) {
                        const double gbps = (double)nchunks * chunk / (double)(h[2 * i + 1] - h[2 * i]);
                        mean += gbps / grid;
                        if (gbps < mn) mn = gbps;
                        if (h[2 * i] < a) a = h[2 * i];
                        if (h[2 * i + 1] > b) b = h[2 * i + 1];
                    }
                    printf("%s,%d,%d,%d,%.0f,%.1f,%.1f,%.2f\n", hbm ? "hbm" : "l2", grid, chunk / 1024, ring / 1024, per_cta / 1048576.0, mean, mn,
                           (double)nchunks * chunk * grid / (double)(b - a) / 1e3);
                }
    return 0;
}
