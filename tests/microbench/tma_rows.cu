// Microbenchmark behind the staging-pipeline design (DESIGN.md "streamed items"): cost of staging one
// chunk of constraint rows (ROWS rows x cnt slots x 16 B) from an L2-resident pool into shared memory
// with 1-D bulk (TMA) copies, as a function of who issues them and of the source alignment.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_rows tma_rows.cu && ./tma_rows
#include <cstdio>
#include <cuda_runtime.h>
constexpr int ROWS = 36;
__device__ __forceinline__ unsigned su(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, int c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(su(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void expect_tx(unsigned long long* b, unsigned n) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void bulk(void* d, const void* s, unsigned n, unsigned long long* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(su(d)), "l"(s), "r"(n), "r"(su(b)) : "memory");
}
__device__ __forceinline__ void wait(unsigned long long* b, unsigned par) {
    unsigned ok;
    do { asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(su(b)), "r"(par) : "memory"); } while (!ok);
}
// mode 0: thread 0 issues all rows; 1: ROWS threads issue one row each; 2: one contiguous copy of the whole chunk;
// 3: no TMA, every thread copies with LDG.128 + STS.128
__global__ void k(const float4* pool, size_t gstride, int cnt, int off, int mode, int iters, long long* out, float* sink) {
    extern __shared__ __align__(128) float4 buf[];
    __shared__ __align__(8) unsigned long long mb;
    if (threadIdx.x == 0) { mbar_init(&mb, mode == 1 ? ROWS : 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    const float4* src = pool + (size_t)blockIdx.x * 4096 + off;
    long long t0 = clock64();
    float acc = 0.f;
    for (int it = 0; it < iters; ++it) {
        const float4* s = src + (it & 7) * 512;
        if (mode == 0) {
            if (threadIdx.x == 0) { expect_tx(&mb, ROWS * cnt * 16); for (int r = 0; r < ROWS; ++r) bulk(buf + r * cnt, s + r * gstride, cnt * 16, &mb); }
        } else if (mode == 1) {
            if (threadIdx.x < ROWS) { expect_tx(&mb, cnt * 16); bulk(buf + threadIdx.x * cnt, s + threadIdx.x * gstride, cnt * 16, &mb); }
        } else if (mode == 2) {
            if (threadIdx.x == 0) { expect_tx(&mb, ROWS * cnt * 16); bulk(buf, s, ROWS * cnt * 16, &mb); }
        } else {
            for (int i = threadIdx.x; i < ROWS * cnt; i += blockDim.x) buf[i] = s[(i / cnt) * gstride + (i % cnt)];
        }
        if (mode < 3) wait(&mb, it & 1);
        __syncthreads();
        acc += buf[(threadIdx.x * 7) % (ROWS * cnt)].x;
        __syncthreads();
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) out[blockIdx.x] = (t1 - t0) / iters;
    if (acc == 123.456f) *sink = acc;
}
int main() {
    const size_t gstride = 524288;   // float4 per pool row, like cons_cap of the 80x20 scene
    float4* pool; long long* out; float* sink;
    cudaMalloc(&pool, ROWS * gstride * 16); cudaMemset(pool, 0, ROWS * gstride * 16);
    cudaMalloc(&out, 132 * 8); cudaMalloc(&sink, 4);
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    const char* names[] = {"1 thread x 36 row copies", "36 threads x 1 row copy", "1 contiguous copy", "LDG+STS by 384 threads"};
    for (int blocks : {1, 80, 132})   // 132 = one CTA per SM of an H100 SXM
        for (int cnt : {32, 96})
            for (int off : {0, 3})
                for (int mode = 0; mode < 4; ++mode) {
                    if (mode == 2 && off) continue;
                    k<<<blocks, 384, ROWS * cnt * 16>>>(pool, gstride, cnt, off, mode, 8, out, sink);   // warm L2
                    k<<<blocks, 384, ROWS * cnt * 16>>>(pool, gstride, cnt, off, mode, 64, out, sink);
                    long long h[132]; cudaMemcpy(h, out, blocks * 8, cudaMemcpyDeviceToHost);
                    long long mx = 0; for (int i = 0; i < blocks; ++i) mx = h[i] > mx ? h[i] : mx;
                    printf("blocks=%3d cnt=%3d (%5d B/chunk) src_off=%d float4  %-26s : %6lld cycles/chunk  %s\n", blocks, cnt, ROWS * cnt * 16, off, names[mode], mx,
                           cudaGetErrorString(cudaGetLastError()));
                }
    return 0;
}
