// Micro-benchmark: do L2 eviction-priority hints protect a gathered table from a read-once stream?
// Models one frame of the den backward pass at the headline shape (N = 64: 256-byte rows): every warp gathers rows at
// random from a ~10 MB table written the frame before, writes its share of the next table (ping-pong), and reads its
// share of a ~20 MB read-once stream that no frame reads again (the alpha spill).  One launch per frame, 16 warps per SM.
// Modes: gathers only / + stream, default policy / stream evict_first + L1::no_allocate / tables evict_last / both.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/l2_policy_bench tools/l2_policy_bench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int kRows = 42240;          // table rows (10.8 MB): 20 per warp at 132 SMs x 16 warps
constexpr int kIters = 40, kGath = 6;  // per warp and frame: 240 gathers (~510 k rows per frame), 40 stream rows (21.6 MB)
constexpr int kStreamFrames = 24;     // the stream rotates over 24 frames (~520 MB), so every frame reads it from HBM

__device__ __forceinline__ uint32_t hash(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
__device__ __forceinline__ float2 ld_plain(const float2 *p) { return *p; }
__device__ __forceinline__ float2 ld_hint(const float2 *p, uint64_t pol) {
    float2 r;
    asm volatile("ld.global.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(r.x), "=f"(r.y) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ float2 ld_once(const float2 *p, uint64_t pol) {
    float2 r;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(r.x), "=f"(r.y) : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void st_hint(float2 *p, float2 v, uint64_t pol) {
    asm volatile("st.global.cg.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(pol) : "memory");
}

// STREAM: read the stream; ONCE: stream evict_first + no L1; KEEP: tables stored and gathered evict_last
template <bool STREAM, bool ONCE, bool KEEP>
__global__ void __launch_bounds__(512, 1) frame(const float2 *tab, float2 *next, const float2 *stream, uint32_t seed) {
    uint64_t pol_first, pol_last;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_first));
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_last));
    const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    float2 acc = make_float2(0.f, 0.f);
    for (int i = 0; i < kIters; ++i) {
        float2 v[kGath], s = make_float2(0.f, 0.f);
#pragma unroll
        for (int b = 0; b < kGath; ++b) {
            const float2 *p = tab + (size_t)(hash(seed ^ (warp * 977u + i * 31u + b)) % kRows) * 32 + lane;
            v[b] = KEEP ? ld_hint(p, pol_last) : ld_plain(p);
        }
        if (STREAM) {
            const float2 *p = stream + ((size_t)warp * kIters + i) * 32 + lane;
            s = ONCE ? ld_once(p, pol_first) : ld_plain(p);
        }
#pragma unroll
        for (int b = 0; b < kGath; ++b) { acc.x += v[b].x; acc.y += v[b].y; }
        acc.x += s.x; acc.y += s.y;
        const int row = warp * 20 + i;
        if (i < 20 && row < kRows) {
            float2 *q = next + (size_t)row * 32 + lane;
            if (KEEP) st_hint(q, acc, pol_last); else __stcg(q, acc);
        }
    }
}

template <bool STREAM, bool ONCE, bool KEEP>
void run(const char *name, float2 *tab0, float2 *tab1, const float2 *stream, int sms) {
    const size_t stream_frame = (size_t)sms * 16 * kIters * 32;   // float2 per frame
    const int frames = 96;
    auto launch = [&](int f) {
        frame<STREAM, ONCE, KEEP><<<sms, 512>>>(f & 1 ? tab1 : tab0, f & 1 ? tab0 : tab1,
                                                stream + (size_t)(f % kStreamFrames) * stream_frame, 0x9e3779b9u * (f + 1));
    };
    for (int f = 0; f < 8; ++f) launch(f);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    for (int f = 0; f < frames; ++f) launch(f);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    const double us = ms * 1e3 / frames;
    const double rows = (double)sms * 16 * kIters * kGath;
    printf("%-34s %7.2f us/frame  %6.1f Grows/s gathered  (%s)\n", name, us, rows / us * 1e-3, cudaGetErrorString(cudaGetLastError()));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount;
    printf("%s SMs=%d L2=%d MB; table %.1f MB, stream %.1f MB per frame\n", p.name, sms, p.l2CacheSize >> 20,
           kRows * 256 / 1e6, (double)sms * 16 * kIters * 256 / 1e6);
    float2 *tab0, *tab1, *stream;
    const size_t stream_bytes = (size_t)kStreamFrames * sms * 16 * kIters * 256;
    cudaMalloc(&tab0, (size_t)kRows * 256); cudaMalloc(&tab1, (size_t)kRows * 256); cudaMalloc(&stream, stream_bytes);
    cudaMemset(tab0, 0, (size_t)kRows * 256); cudaMemset(tab1, 0, (size_t)kRows * 256); cudaMemset(stream, 0, stream_bytes);
    for (int rep = 0; rep < 2; ++rep) {
        run<false, false, false>("gathers only", tab0, tab1, stream, sms);
        run<true, false, false>("+ stream, default policy", tab0, tab1, stream, sms);
        run<true, true, false>("+ stream evict_first/no_allocate", tab0, tab1, stream, sms);
        run<true, false, true>("+ stream, tables evict_last", tab0, tab1, stream, sms);
        run<true, true, true>("+ stream evict_first, tables last", tab0, tab1, stream, sms);
        run<false, false, true>("gathers only, tables evict_last", tab0, tab1, stream, sms);
    }
    cudaFree(tab0); cudaFree(tab1); cudaFree(stream);
    return 0;
}
