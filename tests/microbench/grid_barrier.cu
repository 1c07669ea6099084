// Microbenchmark (not a test): latency of a grid-wide barrier on one 256-thread CTA per SM (132 on an H100 SXM) --
// cooperative_groups grid.sync() against a ticket barrier on one 64-bit counter (atomicAdd + acquire spin).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o grid_barrier grid_barrier.cu && ./grid_barrier
#include <cooperative_groups.h>
#include <cstdio>
namespace cg = cooperative_groups;

__device__ __forceinline__ void ticket_barrier(unsigned long long* bar) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long nb = gridDim.x;
        __threadfence();
        const unsigned long long old = atomicAdd(bar, 1ull);
        const unsigned long long target = (old / nb + 1ull) * nb;
        unsigned long long v;
        do {
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(bar) : "memory");
        } while (v < target);
    }
    __syncthreads();
}

__global__ void k_cg(int n, int* sink) {
    cg::grid_group g = cg::this_grid();
    int acc = 0;
    for (int i = 0; i < n; ++i) { acc += i; g.sync(); }
    if (acc == -1) *sink = acc;
}
__global__ void k_ticket(int n, unsigned long long* bar, int* sink) {
    int acc = 0;
    for (int i = 0; i < n; ++i) { acc += i; ticket_barrier(bar); }
    if (acc == -1) *sink = acc;
}

int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    int blocks = prop.multiProcessorCount, n = 2000;
    int* sink; unsigned long long* bar;
    cudaMalloc(&sink, 4); cudaMalloc(&bar, 8); cudaMemset(bar, 0, 8);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int threads : {256, 128}) {
        for (int rep = 0; rep < 2; ++rep) {
            void* a1[] = {&n, &sink};
            cudaEventRecord(e0);
            cudaLaunchCooperativeKernel((void*)k_cg, dim3(blocks), dim3(threads), a1, 0, 0);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1);
            void* a2[] = {&n, &bar, &sink};
            cudaEventRecord(e0);
            cudaLaunchCooperativeKernel((void*)k_ticket, dim3(blocks), dim3(threads), a2, 0, 0);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms2; cudaEventElapsedTime(&ms2, e0, e1);
            printf("blocks %d threads %d: cg grid.sync %.3f us / barrier, ticket barrier %.3f us / barrier  (%s)\n", blocks, threads,
                   ms * 1e3f / n, ms2 * 1e3f / n, cudaGetErrorString(cudaGetLastError()));
        }
    }
    return 0;
}
