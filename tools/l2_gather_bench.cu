// Micro-benchmark: L2 -> SM random ROW gather bandwidth on the GPU (the resource that bounds the den kernels).
// A [rows][row_floats] fp32 table that fits L2 is gathered by random row index, one row per warp-load
// (row_floats = 32*U floats, each lane loads a float{U} with ld.global.cg), B loads in flight per warp.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/l2_gather_bench tools/l2_gather_bench.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

template <int U> struct V;
template <> struct V<1> { typedef float T; };
template <> struct V<2> { typedef float2 T; };
template <> struct V<4> { typedef float4 T; };
__device__ inline float sum(float a) { return a; }
__device__ inline float sum(float2 a) { return a.x + a.y; }
__device__ inline float sum(float4 a) { return a.x + a.y + a.z + a.w; }

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

template <int U, int B>
void run(int rows, int threads, int ctas_per_sm, int sms) {
    const int per_warp = 4096;
    const int warps = sms * ctas_per_sm * threads / 32;
    float *tab, *out; unsigned *idx;
    cudaMalloc(&tab, (size_t)rows * 32 * U * 4); cudaMemset(tab, 0, (size_t)rows * 32 * U * 4);
    cudaMalloc(&out, 4);
    std::vector<unsigned> h((size_t)warps * per_warp);
    unsigned s = 12345;
    for (auto &x : h) { s = s * 1664525u + 1013904223u; x = (s >> 8) % rows; }
    cudaMalloc(&idx, h.size() * 4); cudaMemcpy(idx, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    gather<U, B><<<sms * ctas_per_sm, threads>>>(tab, idx, per_warp, out);
    cudaEventRecord(e0);
    for (int r = 0; r < 5; ++r) gather<U, B><<<sms * ctas_per_sm, threads>>>(tab, idx, per_warp, out);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); ms /= 5;
    double bytes = (double)warps * per_warp * 32 * U * 4;
    printf("rows=%d rowB=%d U=%d B=%d threads=%d x%d/SM : %.3f ms  %.1f GB/s  %.2f Grows/s  (%s)\n", rows, 32 * U * 4, U, B, threads,
           ctas_per_sm, ms, bytes / ms * 1e-6, (double)warps * per_warp / ms * 1e-6, cudaGetErrorString(cudaGetLastError()));
    cudaFree(tab); cudaFree(out); cudaFree(idx);
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount;
    printf("%s SMs=%d L2=%d MB\n", p.name, sms, p.l2CacheSize >> 20);
    const int rows = 40000;   // 40k rows: 5 / 10 / 20 MB tables
    run<1, 8>(rows, 512, 1, sms);  run<1, 16>(rows, 512, 1, sms); run<1, 16>(rows, 1024, 1, sms); run<1, 16>(rows, 1024, 2, sms);
    run<2, 8>(rows, 512, 1, sms);  run<2, 16>(rows, 512, 1, sms); run<2, 8>(rows, 1024, 1, sms);  run<2, 16>(rows, 1024, 1, sms); run<2, 16>(rows, 1024, 2, sms);
    run<4, 4>(rows, 512, 1, sms);  run<4, 8>(rows, 512, 1, sms);  run<4, 8>(rows, 1024, 1, sms);  run<4, 8>(rows, 1024, 2, sms);
    run<2, 16>(400000, 1024, 2, sms);   // 100 MB table: twice the 50 MB L2 of an H100
    run<2, 16>(4000000, 1024, 2, sms);  // 1 GB table: HBM random rows
    return 0;
}
