// Probe: can two COOPERATIVE (persistent, grid-synchronising) kernels of one CTA per SM each be co-resident, one CTA of each per
// SM, when launched on two streams?  (Needed for running the forward and the backward recursion concurrently.)
// Each kernel does `iters` rounds of {spin ~2 us, grid barrier}.  Prints the time of A alone, B alone, and A||B.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/coop_overlap_probe tools/coop_overlap_probe.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void __launch_bounds__(256, 2) persist(unsigned *counter, int iters, unsigned long long spin_ns, unsigned *smid_out) {
    extern __shared__ unsigned char smem[];
    unsigned epoch = 0;
    if (threadIdx.x == 0) { unsigned s; asm volatile("mov.u32 %0, %%smid;" : "=r"(s)); smid_out[blockIdx.x] = s; }
    for (int i = 0; i < iters; ++i) {
        if (threadIdx.x == 0) {
            unsigned long long t0, t1;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
            do { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 - t0 < spin_ns);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
            unsigned v, target = (++epoch) * gridDim.x;
            do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory"); } while (v < target);
            asm volatile("fence.acq_rel.gpu;" ::: "memory");
        }
        __syncthreads();
    }
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount, iters = 500;
    unsigned *ca, *cb, *sa, *sb;
    cudaMalloc(&ca, 256); cudaMalloc(&cb, 256); cudaMalloc(&sa, sms * 4); cudaMalloc(&sb, sms * 4);
    cudaStream_t s1, s2; cudaStreamCreate(&s1); cudaStreamCreate(&s2);
    const size_t smem = 100 * 1024;   // ~100 KB each: two fit in 227 KB
    cudaFuncSetAttribute(persist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int per_sm = 0; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, persist, 256, smem);
    printf("%s SMs=%d, occupancy of one kernel: %d CTAs/SM\n", p.name, sms, per_sm);
    unsigned long long spin = 2000;
    auto launch = [&](unsigned *c, unsigned *sm, cudaStream_t s) {
        cudaMemsetAsync(c, 0, 4, s);
        int it = iters; void *args[] = {&c, &it, &spin, &sm};
        cudaError_t e = cudaLaunchCooperativeKernel((const void *)persist, dim3(sms), dim3(256), args, smem, s);
        if (e != cudaSuccess) printf("launch: %s\n", cudaGetErrorString(e));
    };
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms;
    launch(ca, sa, s1); cudaDeviceSynchronize();
    cudaEventRecord(e0, s1); launch(ca, sa, s1); cudaEventRecord(e1, s1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    printf("A alone: %.3f ms (%d rounds of 2 us spin + grid barrier = %.2f us per round)\n", ms, iters, 1e3 * ms / iters);
    cudaDeviceSynchronize();
    cudaEventRecord(e0, 0);
    launch(ca, sa, s1); launch(cb, sb, s2);
    cudaDeviceSynchronize();
    cudaEventRecord(e1, 0); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    printf("A || B on two streams: %.3f ms  (%s)  [%s]\n", ms, ms < 1.5f * 1e-3f * iters * 3.5f ? "concurrent" : "serialised?", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
