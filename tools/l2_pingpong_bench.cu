// Micro-benchmark 2: random ROW gathers from a table that every SM REWRITES between passes (the den recursion's
// access pattern: rows produced by other SMs one frame earlier), versus a table written once (read-mostly).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/l2_pingpong_bench tools/l2_pingpong_bench.cu
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>

template <int U> struct V;
template <> struct V<1> { typedef float T; };
template <> struct V<2> { typedef float2 T; };
__device__ inline float sum(float a) { return a; }
__device__ inline float sum(float2 a) { return a.x + a.y; }

template <int U, int B>
__global__ void gather(const float *tab, const unsigned *idx, int per_warp, float *out) {
    typedef typename V<U>::T T;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const unsigned *my = idx + (size_t)warp * per_warp;
    float acc = 0.f;
    for (int i = 0; i < per_warp; i += B) {
        T v[B];
#pragma unroll
        for (int b = 0; b < B; ++b) v[b] = __ldcg(reinterpret_cast<const T *>(tab + (size_t)__ldg(my + i + b) * (32 * U)) + lane);
#pragma unroll
        for (int b = 0; b < B; ++b) acc += sum(v[b]);
    }
    if (acc == 123.456f) out[0] = acc;
}
// every warp rewrites a contiguous slice of rows (like the den kernels' epilogue stores)
template <int U>
__global__ void rewrite(float *tab, int rows, float val) {
    const int warps = gridDim.x * blockDim.x / 32;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int per = (rows + warps - 1) / warps;
    for (int r = warp * per; r < min(rows, (warp + 1) * per); ++r)
        for (int u = 0; u < U; ++u) __stcg(tab + (size_t)r * 32 * U + lane * U + u, val);
}

template <int U, int B>
void run(int rows, int threads, int sms, bool pingpong) {
    const int per_warp = 512;   // ~ one den frame per launch: SMs x 16 warps x 512 row gathers
    const int warps = sms * threads / 32;
    float *tab, *out; unsigned *idx;
    cudaMalloc(&tab, (size_t)rows * 32 * U * 4); cudaMemset(tab, 0, (size_t)rows * 32 * U * 4);
    cudaMalloc(&out, 4);
    std::vector<unsigned> h((size_t)warps * per_warp);
    unsigned s = 12345;
    for (auto &x : h) { s = s * 1664525u + 1013904223u; x = (s >> 8) % rows; }
    cudaMalloc(&idx, h.size() * 4); cudaMemcpy(idx, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float total = 0; const int reps = 20;
    for (int r = 0; r < reps + 2; ++r) {
        if (pingpong || r == 0) rewrite<U><<<sms, threads>>>(tab, rows, (float)r);
        cudaEventRecord(e0);
        gather<U, B><<<sms, threads>>>(tab, idx, per_warp, out);
        cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        if (r >= 2) total += ms;
    }
    float ms = total / reps;
    double bytes = (double)warps * per_warp * 32 * U * 4;
    printf("%-10s rows=%d rowB=%d B=%d threads=%d: %.1f us per pass  %.1f GB/s  (%s)\n", pingpong ? "rewritten" : "read-only", rows,
           32 * U * 4, B, threads, ms * 1e3, bytes / ms * 1e-6, cudaGetErrorString(cudaGetLastError()));
    cudaFree(tab); cudaFree(out); cudaFree(idx);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount;
    printf("%s SMs=%d\n", p.name, sms);
    for (int pp = 0; pp < 2; ++pp) {
        run<2, 16>(40000, 512, sms, pp);
        run<2, 16>(40000, 1024, sms, pp);
        run<1, 16>(40000, 512, sms, pp);
        run<1, 16>(40000, 1024, sms, pp);
        run<1, 16>(20000, 1024, sms, pp);
    }
    return 0;
}
