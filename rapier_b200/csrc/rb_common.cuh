// rb_common.cuh -- execution-context abstraction shared by every kernel of librapier_b200.
//
// All device work is written as "phase functions": `template <class Ctx> RB_HD void phase(Ctx&, ...)`
// whose loops are strided by the context (grid-wide, CTA-wide or warp-wide) and whose phase
// boundaries are ctx.grid_sync() / ctx.block_sync().  The product build (nvcc, sm_90a) instantiates
// them with the CUDA contexts below inside __global__ kernels.  tests/emul/ compiles the very same
// phase functions with g++ and a one-thread context (RB_EMULATE) so the kernel LOGIC can be checked
// against the oracle on a machine without a GPU; that build is test infrastructure only and is never
// loaded by the product (rapier_b200/_lib.py refuses to load anything but the CUDA library).
#pragma once
#include <cstring>
#include <stdint.h>
#include <math.h>
#include <string.h>

#if defined(__CUDACC__) && !defined(RB_EMULATE)
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#define RB_HD __device__ __forceinline__
#define RB_D __device__ __forceinline__
#define RB_PHASE __device__
#define RB_DEVICE_BUILD 1
#else
#ifndef RB_EMULATE
#error "host-only compilation of the kernels requires -DRB_EMULATE (tests/emul only)"
#endif
#include <driver_types.h>
#include <vector_types.h>
#include <vector_functions.h>
#define RB_HD inline
#define RB_D inline
#define RB_PHASE inline
#define RB_DEVICE_BUILD 0
#endif

namespace rb {

#if RB_DEVICE_BUILD
namespace cg = cooperative_groups;

// Grid-wide context of a cooperative persistent kernel.
struct GridCtx {
    int gtid, gsize, btid, bsize, bid, nblocks, lane, nlanes, gwarp, ngwarps;
    __device__ GridCtx() {
        btid = threadIdx.x; bsize = blockDim.x; bid = blockIdx.x; nblocks = gridDim.x;
        gtid = bid * bsize + btid; gsize = nblocks * bsize;
        lane = btid & 31; nlanes = 32;
        gwarp = gtid >> 5; ngwarps = gsize >> 5;
    }
    __device__ __forceinline__ void grid_sync() const { cg::this_grid().sync(); }
    __device__ __forceinline__ void block_sync() const { __syncthreads(); }
    __device__ __forceinline__ bool warp_any(bool p) const { return __any_sync(0xffffffffu, p); }
};

// CTA-local context (one CTA per work item).
struct BlockCtx {
    int btid, bsize, bid, nblocks, lane, nlanes;
    __device__ BlockCtx() {
        btid = threadIdx.x; bsize = blockDim.x; bid = blockIdx.x; nblocks = gridDim.x;
        lane = btid & 31; nlanes = 32;
    }
    __device__ __forceinline__ void block_sync() const { __syncthreads(); }
};

template <class T> RB_D T atomic_add(T* p, T v) { return atomicAdd(p, v); }
RB_D int atomic_min(int* p, int v) { return atomicMin(p, v); }
RB_D unsigned long long atomic_min64(unsigned long long* p, unsigned long long v) { return atomicMin(p, v); }
RB_D unsigned atomic_and(unsigned* p, unsigned v) { return atomicAnd(p, v); }
RB_D unsigned atomic_max_u(unsigned* p, unsigned v) { return atomicMax(p, v); }
RB_D unsigned atomic_or(unsigned* p, unsigned v) { return atomicOr(p, v); }
RB_D int atomic_cas(int* p, int cmp, int v) { return atomicCAS(p, cmp, v); }
RB_D void thread_fence() { __threadfence(); }
#define RB_SHARED __shared__

#else  // ---------------- host emulation: one thread plays every role ----------------

struct GridCtx {
    int gtid = 0, gsize = 1, btid = 0, bsize = 1, bid = 0, nblocks = 1, lane = 0, nlanes = 1, gwarp = 0, ngwarps = 1;
    void grid_sync() const {}
    void block_sync() const {}
    bool warp_any(bool p) const { return p; }
};
struct BlockCtx {
    int btid = 0, bsize = 1, bid = 0, nblocks = 1, lane = 0, nlanes = 1;
    void block_sync() const {}
};
template <class T> inline T atomic_add(T* p, T v) { T o = *p; *p = o + v; return o; }
inline int atomic_min(int* p, int v) { int o = *p; if (v < o) *p = v; return o; }
inline unsigned long long atomic_min64(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; if (v < o) *p = v; return o; }
inline unsigned atomic_and(unsigned* p, unsigned v) { unsigned o = *p; *p = o & v; return o; }
inline unsigned atomic_max_u(unsigned* p, unsigned v) { unsigned o = *p; if (v > o) *p = v; return o; }
inline unsigned atomic_or(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
inline int atomic_cas(int* p, int cmp, int v) { int o = *p; if (o == cmp) *p = v; return o; }
inline void thread_fence() {}
#define RB_SHARED static

#endif

// Raise a device-side status (capacity overflow, non-finite state): sticky in State::error and mirrored into the
// host-mapped status word so that every synchronising call of the C ABI sees it, also after asynchronous steps.
#define RB_RAISE(w, code) do { (w).st->error = (code); if ((w).host_hint[1] == 0) (w).host_hint[1] = (code); } while (0)

RB_HD float as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
RB_HD uint32_t as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
RB_HD float as_float_i(int i) { float f; memcpy(&f, &i, 4); return f; }
RB_HD int as_int(float f) { int i; memcpy(&i, &f, 4); return i; }


#if RB_DEVICE_BUILD
RB_D long long rb_clock() { return clock64(); }
#else
inline long long rb_clock() { return 0; }
#endif

// ---- bulk staging: 1-D TMA copies global -> shared completing on an mbarrier (emulation: memcpy) ----
#if RB_DEVICE_BUILD
RB_D unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
RB_D void mbar_init(unsigned long long* b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
RB_D void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
RB_D void mbar_expect_tx(unsigned long long* b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
RB_D void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
}
RB_D void mbar_wait(unsigned long long* b, unsigned parity) {
    unsigned ok;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok)
                     : "r"(smem_u32(b)), "r"(parity)
                     : "memory");
    } while (!ok);
}
// Orders this thread's earlier generic-proxy writes before later async-proxy (TMA) reads of them.
RB_D void fence_async_proxy() { asm volatile("fence.proxy.async;" ::: "memory"); }
#else
inline void mbar_init(unsigned long long*, int) {}
inline void mbar_init_fence() {}
inline void mbar_expect_tx(unsigned long long*, unsigned) {}
inline void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long*) { memcpy(dst, src, bytes); }
inline void mbar_wait(unsigned long long*, unsigned) {}
inline void fence_async_proxy() {}
#endif

}  // namespace rb
