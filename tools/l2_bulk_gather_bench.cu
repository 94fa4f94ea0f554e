// Micro-benchmark: random ROW gathers from an L2-resident table into SHARED memory, so that the bytes in flight are
// bounded by shared memory instead of registers.  Three ways to fetch one ROWB-byte row per arc:
//   ldg    : each lane ld.global.cg's its 8 bytes into registers (what the den kernels did in round 1);
//   ldgsts : each lane cp.async's its 8 bytes into a per-warp ring in shared memory;
//   bulk   : ONE lane issues cp.async.bulk (TMA 1-D copy, mbarrier complete_tx) for the whole row, up to 32 rows per
//            warp instruction; the warp then reads the ring with LDS.
// Every variant consumes the data the way the recursion does (two FMAs per lane and row).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/l2_bulk_gather_bench tools/l2_bulk_gather_bench.cu
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, unsigned parity) {
    unsigned ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, unsigned bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// R rows per stage, STAGES stages per warp, ROWB bytes per row (lane reads ROWB/32 bytes)
template <int ROWB, int R, int STAGES>
__global__ void bulk_gather(const char *tab, const unsigned *idx, int per_warp, float *out) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    unsigned char *buf = smem + (size_t)warp * STAGES * R * ROWB;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem + (size_t)nw * STAGES * R * ROWB) + warp * STAGES;
    if (lane == 0) {
        for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(bars + s), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    const unsigned *my = idx + ((size_t)blockIdx.x * nw + warp) * per_warp;
    const int n = per_warp / R;
    auto issue = [&](int k) {
        const int s = k % STAGES;
        const uint32_t bar = smem_u32(bars + s);
        if (lane == 0) mbar_expect_tx(bar, R * ROWB);
        __syncwarp();
        for (int r = lane; r < R; r += 32)
            bulk_g2s(smem_u32(buf + (size_t)(s * R + r) * ROWB), tab + (size_t)__ldg(my + k * R + r) * ROWB, ROWB, bar);
    };
    for (int k = 0; k < STAGES && k < n; ++k) issue(k);
    float a0 = 0.f, a1 = 0.f;
    for (int k = 0; k < n; ++k) {
        const int s = k % STAGES;
        mbar_wait(smem_u32(bars + s), (k / STAGES) & 1);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (ROWB == 256) {
                const float2 v = *reinterpret_cast<const float2 *>(buf + (size_t)(s * R + r) * ROWB + lane * 8);
                a0 = fmaf(v.x, 1.0001f, a0); a1 = fmaf(v.y, 1.0001f, a1);
            } else {
                const float v = *reinterpret_cast<const float *>(buf + (size_t)(s * R + r) * ROWB + lane * 4);
                a0 = fmaf(v, 1.0001f, a0);
            }
        }
        __syncwarp();
        if (k + STAGES < n) issue(k + STAGES);
    }
    if (a0 + a1 == 123.456f) out[0] = a0;
}

template <int ROWB, int R, int STAGES>
__global__ void ldgsts_gather(const char *tab, const unsigned *idx, int per_warp, float *out) {
    extern __shared__ __align__(128) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    unsigned char *buf = smem + (size_t)warp * STAGES * R * ROWB;
    const unsigned *my = idx + ((size_t)blockIdx.x * nw + warp) * per_warp;
    const int n = per_warp / R;
    constexpr int LB = ROWB / 32;
    auto issue = [&](int k) {
        const int s = k % STAGES;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const uint32_t dst = smem_u32(buf + (size_t)(s * R + r) * ROWB + lane * LB);
            const char *src = tab + (size_t)__ldg(my + k * R + r) * ROWB + lane * LB;
            asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(dst), "l"(src), "n"(LB) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    for (int k = 0; k < STAGES; ++k) { if (k < n) issue(k); else asm volatile("cp.async.commit_group;" ::: "memory"); }
    float a0 = 0.f, a1 = 0.f;
    for (int k = 0; k < n; ++k) {
        const int s = k % STAGES;
        asm volatile("cp.async.wait_group %0;" ::"n"(STAGES - 1) : "memory");
        __syncwarp();
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (ROWB == 256) {
                const float2 v = *reinterpret_cast<const float2 *>(buf + (size_t)(s * R + r) * ROWB + lane * 8);
                a0 = fmaf(v.x, 1.0001f, a0); a1 = fmaf(v.y, 1.0001f, a1);
            } else {
                const float v = *reinterpret_cast<const float *>(buf + (size_t)(s * R + r) * ROWB + lane * 4);
                a0 = fmaf(v, 1.0001f, a0);
            }
        }
        __syncwarp();
        if (k + STAGES < n) issue(k + STAGES); else asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (a0 + a1 == 123.456f) out[0] = a0;
}

struct Bench {
    int sms, rows;
    char *tab; float *out; unsigned *idx;
    static constexpr int per_warp = 4096;
    void setup(int rows_, int rowb, int max_warps) {
        rows = rows_;
        cudaMalloc(&tab, (size_t)rows * rowb); cudaMemset(tab, 0, (size_t)rows * rowb);
        cudaMalloc(&out, 4);
        std::vector<unsigned> h((size_t)max_warps * per_warp);
        unsigned s = 12345;
        for (auto &x : h) { s = s * 1664525u + 1013904223u; x = (s >> 8) % rows; }
        cudaMalloc(&idx, h.size() * 4); cudaMemcpy(idx, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    }
    void teardown() { cudaFree(tab); cudaFree(out); cudaFree(idx); }
};

template <int ROWB, int R, int STAGES, bool BULK>
void run(Bench &b, int threads) {
    const int nw = threads / 32;
    const size_t smem = (size_t)nw * STAGES * R * ROWB + (size_t)nw * STAGES * 8;
    auto kern = BULK ? bulk_gather<ROWB, R, STAGES> : ldgsts_gather<ROWB, R, STAGES>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
        printf("%s rowB=%d R=%d stages=%d threads=%d: smem %zu too large\n", BULK ? "bulk  " : "ldgsts", ROWB, R, STAGES, threads, smem);
        cudaGetLastError();
        return;
    }
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    kern<<<b.sms, threads, smem>>>(b.tab, b.idx, b.per_warp, b.out);
    cudaEventRecord(e0);
    for (int r = 0; r < 5; ++r) kern<<<b.sms, threads, smem>>>(b.tab, b.idx, b.per_warp, b.out);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
    const double nrows = (double)b.sms * nw * b.per_warp;
    printf("%s rowB=%d R=%d stages=%d threads=%d inflight=%zuKB : %.3f ms  %.1f GB/s  %.2f Grows/s  (%s)\n", BULK ? "bulk  " : "ldgsts",
           ROWB, R, STAGES, threads, (size_t)nw * STAGES * R * ROWB >> 10, ms, nrows * ROWB / ms * 1e-6, nrows / ms * 1e-6,
           cudaGetErrorString(cudaGetLastError()));
    fflush(stdout);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    Bench b; b.sms = p.multiProcessorCount;
    printf("%s SMs=%d\n", p.name, b.sms);
    b.setup(40000, 256, b.sms * 32);
    // TMA 1-D row copies, 256-byte rows
    run<256, 8, 2, true>(b, 512);   run<256, 8, 4, true>(b, 512);   run<256, 16, 2, true>(b, 512);  run<256, 16, 3, true>(b, 512);
    run<256, 32, 2, true>(b, 256);  run<256, 32, 3, true>(b, 256);  run<256, 16, 6, true>(b, 256);
    run<256, 32, 6, true>(b, 128);  run<256, 32, 3, true>(b, 128);
    run<256, 8, 2, true>(b, 1024);  run<256, 8, 3, true>(b, 1024);  run<256, 4, 6, true>(b, 1024);
    // LDGSTS, 8 bytes per lane
    run<256, 8, 2, false>(b, 512);  run<256, 8, 4, false>(b, 512);  run<256, 16, 3, false>(b, 512);
    run<256, 8, 2, false>(b, 1024); run<256, 8, 3, false>(b, 1024); run<256, 4, 6, false>(b, 1024);
    b.teardown();
    b.setup(40000, 128, b.sms * 32);
    run<128, 16, 4, true>(b, 512);  run<128, 32, 3, true>(b, 512);  run<128, 32, 6, true>(b, 256);  run<128, 16, 3, true>(b, 1024);
    run<128, 16, 4, false>(b, 512); run<128, 16, 3, false>(b, 1024);
    b.teardown();
    return 0;
}
