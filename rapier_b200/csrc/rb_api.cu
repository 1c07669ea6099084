// rb_api.cu -- kernels + the extern "C" boundary of librapier_b200.so (include/rapier_b200.h).
//
// Per step the host enqueues two launches on one stream, with no host synchronisation:
//   k_collide       cooperative persistent kernel: collider refresh, [broad phase], narrow phase,
//                   [colouring + islands + schedule]   (rb_collide.cuh); then the solves that are not
//                   shared-memory items (items with joints, the grid-wide "large" item 0)
//   k_solve_coop /  one CTA per shared-memory item from a cost-ordered queue: bodies + impulses in shared
//   k_solve_coop_big  memory, the whole generate -> 4 x (warmstart, biased, integrate, relax) -> writeback
//                   chain fused; constant constraint rows resident or streamed from L2 by bulk (TMA) copies
// All sizes that change at run time (pairs, manifolds, items) live in device memory (rb::State).
//
// With -DRB_EMULATE (tests/emul only) the same kernels and the same host code run on the host with malloc'd
// tables: launch() calls each kernel as one CTA of one thread.  A logic check of the kernels and of the
// step's launch sequence for machines without a GPU, never part of the product library.  It differs from
// the device in two places: the 4-lane kernels run 1 lane per constraint (CONS_LANES), and
// RB_EMU_COOP_SMEM_FLOATS can lower the shared-memory budget of both k_solve_coop launch shapes.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <array>
#include <type_traits>
#include <vector>

#include "rb_solver.cuh"
#include "rb_hull.h"
#include "../../include/rapier_b200.h"

using namespace rb;

// ------------------------------------------------------------------------------------------------
// error handling + memory backend
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static void set_err(const char* fmt, const char* a = "", int code = 0) { snprintf(g_err, sizeof(g_err), fmt, a, code); }

#if RB_DEVICE_BUILD
#define CK(call)                                                                 \
    do {                                                                         \
        cudaError_t e_ = (call);                                                 \
        if (e_ != cudaSuccess) {                                                 \
            set_err("CUDA error %s (%d) at " #call, cudaGetErrorString(e_), (int)e_); \
            return RB_ERR_CUDA;                                                  \
        }                                                                        \
    } while (0)
static cudaError_t dev_alloc(void** p, size_t n) { cudaError_t e = cudaMalloc(p, n ? n : 16); if (e == cudaSuccess) e = cudaMemset(*p, 0, n ? n : 16); return e; }
static cudaError_t dev_free(void* p) { return cudaFree(p); }
static cudaError_t h2d(void* d, const void* h, size_t n) { return n ? cudaMemcpy(d, h, n, cudaMemcpyHostToDevice) : cudaSuccess; }
static cudaError_t d2h(void* h, const void* d, size_t n) { return n ? cudaMemcpy(h, d, n, cudaMemcpyDeviceToHost) : cudaSuccess; }
static cudaError_t dev_set(void* d, int v, size_t n) { return n ? cudaMemset(d, v, n) : cudaSuccess; }
static cudaError_t set_device(int d) { return cudaSetDevice(d); }
static cudaError_t stream_sync(cudaStream_t s) { return cudaStreamSynchronize(s); }
static cudaError_t memset_async(void* d, int v, size_t n, cudaStream_t s) { return cudaMemsetAsync(d, v, n, s); }
static cudaError_t copy_async(void* d, const void* h, size_t n, cudaMemcpyKind k, cudaStream_t s) { return cudaMemcpyAsync(d, h, n, k, s); }
#else
#define CK(call)                                 \
    do {                                         \
        if ((call) != 0) { set_err("emulated allocation failed%s", ""); return RB_ERR_CUDA; } \
    } while (0)
static cudaError_t dev_alloc(void** p, size_t n) { *p = calloc(n ? n : 16, 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static cudaError_t dev_free(void* p) { free(p); return cudaSuccess; }
static cudaError_t h2d(void* d, const void* h, size_t n) { if (n) memcpy(d, h, n); return cudaSuccess; }
static cudaError_t d2h(void* h, const void* d, size_t n) { if (n) memcpy(h, d, n); return cudaSuccess; }
static cudaError_t dev_set(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static cudaError_t set_device(int) { return cudaSuccess; }
static cudaError_t stream_sync(cudaStream_t) { return cudaSuccess; }
static cudaError_t memset_async(void* d, int v, size_t n, cudaStream_t) { return dev_set(d, v, n); }
static cudaError_t copy_async(void* d, const void* h, size_t n, cudaMemcpyKind, cudaStream_t) { return h2d(d, h, n); }
#endif

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
constexpr int COLLIDE_THREADS = 256;
constexpr int ITEM_SMEM_BYTES = ITEM_MAX_BODIES * SB_STRIDE * 4;
// k_solve_coop launch shapes.  Small: two CTAs per SM, items resident in shared memory (many small
// islands).  Big: one CTA per SM with all its shared memory, four times the lanes (islands whose
// constraints are streamed from the L2 pool, or that only fit resident here).
constexpr int COOP_SMALL_THREADS = 128, COOP_SMALL_SMEM_BYTES = 108 * 1024;
constexpr int COOP_BIG_THREADS = 256, COOP_BIG_SMEM_BYTES = 220 * 1024;
// Lanes per constraint of the lane-cooperative kernels (k_collide's inline item-0 solve, k_solve_large, k_solve_coop).
// The emulation's one thread has no lane groups: it runs them with one lane.
constexpr int CONS_LANES = RB_DEVICE_BUILD ? 4 : 1;

struct Grav { float x, y, z; };

template <class Ctx>
RB_PHASE void init_bodies_phase(const Ctx& ctx, const World& w, int first) {
    for (int b = first + ctx.gtid; b < w.nb; b += ctx.gsize) {
        pose p = body_pose(w, b);
        update_world_mass(w, b, p);
        float* s = w.state13 + (size_t)b * 13;
        vec3 l = xyz(w.b_linvel[b]), a = xyz(w.b_angvel[b]);
        s[0] = p.t.x; s[1] = p.t.y; s[2] = p.t.z; s[3] = p.q.x; s[4] = p.q.y; s[5] = p.q.z; s[6] = p.q.w;
        s[7] = l.x; s[8] = l.y; s[9] = l.z; s[10] = a.x; s[11] = a.y; s[12] = a.z;
    }
}

// Scatter of externally provided body states (multi-GPU boundary all-gather): 13 floats per body.
template <class Ctx>
RB_PHASE void import_states_phase(const Ctx& ctx, const World& w, const int* idx, const float* src, int n, int table) {
    for (int k = ctx.gtid; k < n; k += ctx.gsize) {
        int b = idx[k];
        float* d = w.state13 + (size_t)b * 13;
        // src == NULL: the rows were gathered in place into the state buffer; table: src is a whole [nb][13] table
        const float* s = src ? src + (size_t)(table ? b : k) * 13 : d;
        w.b_pos_t[b] = make_float4(s[0], s[1], s[2], 0.f);
        w.b_pos_q[b] = make_float4(s[3], s[4], s[5], s[6]);
        w.b_linvel[b] = make_float4(s[7], s[8], s[9], 0.f);
        w.b_angvel[b] = make_float4(s[10], s[11], s[12], 0.f);
        if (s != d && !table)   // (table mode: the current buffer's rows of these bodies belong to an in-flight gather)
            for (int i = 0; i < 13; ++i) d[i] = s[i];
        update_world_mass(w, b, body_pose(w, b));
    }
}

// Unit-level known-answer evaluation: ONE device function of the path on literal inputs (rb_debug_kat;
// float layouts in tests/golden/make_ref_vectors.py).  Runs as a single thread; `w` is a one-pair, one-slot
// scratch world for the functions that read the pair / constraint tables.
enum { KAT_POSE_DRIFT = 0, KAT_REDUCE, KAT_NORMAL_SOLVE, KAT_TANGENT_SOLVE, KAT_GENERATE };
RB_PHASE void kat_phase(const World& w, int which, const float* in, float* out) {
    auto v3at = [&](int o) { return mk3(in[o], in[o + 1], in[o + 2]); };
    auto put3 = [&](int o, vec3 v) { out[o] = v.x; out[o + 1] = v.y; out[o + 2] = v.z; };
    if (which == KAT_POSE_DRIFT) {
        quat qb, qc;
        qb.x = in[3]; qb.y = in[4]; qb.z = in[5]; qb.w = in[6];
        qc.x = in[10]; qc.y = in[11]; qc.z = in[12]; qc.w = in[13];
        out[0] = pose_drift(mkpose(qb, v3at(0)), mkpose(qc, v3at(7)), in[14]);
    } else if (which == KAT_REDUCE) {
        RawManifold m;
        m.n = (int)in[0];
        m.n1 = v3at(2);
        for (int i = 0; i < m.n; ++i) { m.pt[i].p1 = v3at(5 + 4 * i); m.pt[i].dist = in[8 + 4 * i]; }
        int sel[4] = {0, 1, 2, 3};
        int nsel = m.n < MAX_PTS ? m.n : MAX_PTS;
        reduce_manifold(m, sel, nsel, in[1]);
        out[0] = (float)nsel;
        for (int i = 0; i < 4; ++i) out[1 + i] = i < nsel ? (float)sel[i] : -1.0f;
    } else if (which == KAT_NORMAL_SOLVE) {
        const vec3 dir = v3at(0), im1 = v3at(3), im2 = v3at(6);
        PointPre pp;
        pp.td1 = v3at(9); pp.td2 = v3at(12); pp.itd1 = v3at(15); pp.itd2 = v3at(18);
        pp.rhs = in[22]; pp.cfm = in[24];
        vec3 v1 = v3at(25), w1 = v3at(28), v2 = v3at(31), w2 = v3at(34);
        float nl;
        const float dl = point_solve(pp, in[21], in[23], dir, v1, w1, v2, w2, nl);
        apply_normal(had(dir, im1), had(dir, im2), pp.itd1, pp.itd2, dl, v1, w1, v2, w2);
        out[0] = nl;
        put3(1, v1); put3(4, w1); put3(7, v2); put3(10, w2);
    } else if (which == KAT_TANGENT_SOLVE) {
        Params P = w.prm;
        P.sub_inv_dt = 1.0f;
        BodyState g1, g2;
        g1.p = pident(); g2.p = pident(); g1.ii = sym_zero(); g2.ii = sym_zero();
        g1.im = v3at(9); g2.im = v3at(12);
        FrictionJac j;
        j.td10 = v3at(15); j.td11 = v3at(18); j.td20 = v3at(21); j.td21 = v3at(24);
        j.i10 = v3at(27); j.i11 = v3at(30); j.i20 = v3at(33); j.i21 = v3at(36);
        j.tw1 = zero3(); j.tw2 = zero3();
        FrictionState f;
        f.ti0 = in[45]; f.ti1 = in[46]; f.wi = 0.0f;
        vec3 v1 = v3at(48), w1 = v3at(51), v2 = v3at(54), w2 = v3at(57);
        g1.lin = v1; g1.ang = w1; g2.lin = v2; g2.ang = w2;
        friction_solve_jac(P, g1, g2, v3at(0), v3at(3), v3at(6), 1, in[47], 0.0f, 0.0f, j, in[39], in[40], in[41], false, v3at(42),
                           zero3(), f, v1, w1, v2, w2);
        out[0] = f.ti0; out[1] = f.ti1;
        put3(2, v1); put3(5, w1); put3(8, v2); put3(11, w2);
    } else if (which == KAT_GENERATE) {
        const int n = (int)in[5];
        for (int r = 0; r < PR_ROWS; ++r) prow(w, 0, r, 0) = make_float4(0.f, 0.f, 0.f, 0.f);
        prow(w, 0, PR_INFO, 0) = make_float4(as_float_i(0), as_float_i(n), as_float_i(n), as_float_i(0));
        prow(w, 0, PR_NORMAL, 0) = make_float4(in[0], in[1], in[2], in[3]);
        prow(w, 0, PR_LN2, 0) = make_float4(0.f, 0.f, 0.f, in[4]);
        for (int k = 0; k < n; ++k) {
            const int o = 6 + 19 * k, cid = (int)in[o + 6];
            prow(w, 0, PR_A1 + k, 0) = make_float4(in[o], in[o + 1], in[o + 2], as_float_i(cid));
            prow(w, 0, PR_A2 + k, 0) = make_float4(in[o + 3], in[o + 4], in[o + 5], 0.f);
            prow(w, 0, PR_PD + cid, 0) = make_float4(in[o + 7], in[o + 8], in[o + 9], 0.f);
            prow(w, 0, PR_TW + cid, 0) = make_float4(in[o + 10], in[o + 11], in[o + 12], 0.f);
            prow(w, 0, PR_DP1 + cid, 0) = make_float4(in[o + 13], in[o + 14], in[o + 15], 0.f);
            prow(w, 0, PR_DP2 + cid, 0) = make_float4(in[o + 16], in[o + 17], in[o + 18], 0.f);
        }
        w.cons_hdr[0] = make_int4(0, NO_BODY, NO_BODY, 0);
        GlobalBodies gb;
        gb.w = &w;
        Cons c;
        cons_generate(w, gb, 0, 0, 0, c);
        for (int i = 0; i < 39; ++i) out[i] = 0.0f;
        out[0] = (float)c.nc; put3(1, c.dir); put3(4, c.t1); out[7] = c.fric;
        for (int k = 0; k < MAX_PTS; ++k) {
            out[8 + k] = c.imp[k]; out[12 + k] = c.acc[k]; out[16 + k] = k < c.nc ? c.r[k] : 0.0f;
            out[20 + k] = k < c.nc ? c.dist0[k] : 0.0f; out[24 + k] = c.twd[k];
            out[35 + k] = k < c.nc ? (float)c.cid[k] : 255.0f;
        }
        out[28] = c.ti0; out[29] = c.ti1; out[30] = c.ta0; out[31] = c.ta1; out[32] = c.wi; out[33] = c.wa; out[34] = c.wr;
    }
}

// Halo bodies (b_owned == 2): take their state from the packed state table (filled by the exchange).
template <class Ctx>
RB_PHASE void import_halo_phase(const Ctx& ctx, const World& w) {
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize) {
        if (w.b_owned[b] != 2) continue;
        const float* s = w.state13 + (size_t)b * 13;
        w.b_pos_t[b] = make_float4(s[0], s[1], s[2], 0.f);
        w.b_pos_q[b] = make_float4(s[3], s[4], s[5], s[6]);
        w.b_linvel[b] = make_float4(s[7], s[8], s[9], 0.f);
        w.b_angvel[b] = make_float4(s[10], s[11], s[12], 0.f);
        update_world_mass(w, b, body_pose(w, b));
    }
}
// Wake the islands of the listed bodies (idx == NULL: every sleeping body), timers reset.
template <class Ctx>
RB_PHASE void wake_phase(const Ctx& ctx, const World& w, const int* idx, int n) {
    if (!idx) {
        for (int b = ctx.gtid; b < w.nb; b += ctx.gsize)
            if (w.b_sleeping[b]) { w.b_sleeping[b] = 0; w.b_sleep_time[b] = 0.0f; w.st->sched_dirty = 1; }
        return;
    }
    for (int k = ctx.gtid; k < n; k += ctx.gsize) {
        const int b = idx[k];
        if (b < 0 || b >= w.nb || !type_is_solver(w.b_type[b])) continue;
        w.wake_req[w.isl_label[b]] = 1;   // (labels are roots; wake_apply_phase wakes the whole island right away, the
        w.st->wake_any = 1;               //  next step's wake pass clears the requests)
        if (w.b_sleeping[b]) { w.b_sleeping[b] = 0; w.b_sleep_time[b] = 0.0f; w.st->sched_dirty = 1; }
    }
}
template <class Ctx>
RB_PHASE void wake_apply_phase(const Ctx& ctx, const World& w) {
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize)
        if (type_is_solver(w.b_type[b]) && w.b_sleeping[b] && w.wake_req[w.isl_label[b]]) {
            w.b_sleeping[b] = 0;
            w.b_sleep_time[b] = 0.0f;
            w.st->sched_dirty = 1;
        }
}

// New halo flags (device array, 0 / 2 for foreign bodies; entries of owned bodies are ignored).
template <class Ctx>
RB_PHASE void set_halo_phase(const Ctx& ctx, const World& w, const unsigned char* flags) {
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize) {
        if (w.b_owned[b] == 1) continue;
        const unsigned char f = flags[b] ? 2 : 0;
        if (w.b_owned[b] != f) { w.b_owned[b] = f; w.st->lists_dirty |= 1; w.st->bp_dirty = 1; }
    }
}

// Collision pipeline, then every solve that is NOT shared-memory resident: work items streamed from
// HBM (one CTA each) and the grid-wide "large" item 0.  Those touch bodies / constraints disjoint from
// the items k_solve_coop handles next, so the order between the two kernels does not matter.
// `do_solve` = 0 runs only the collision pipeline (the general path, whose solves have kernels of their own);
// bit 1 set: k_solve_large follows and solves the grid-wide item 0.
// SHAPES = 1: the variant for worlds with capsules (rb_geom.cuh); the ball / cuboid kernel is SHAPES = 0.
template <int SHAPES>
RB_KERNEL RB_BOUNDS(COLLIDE_THREADS) k_collide(World w, Grav g, int do_solve) {
    RB_DYNAMIC_SMEM(smem);
    GridCtx ctx;
    if (ctx.gtid == 0) {   // publish last step's launch hints to the host (read without synchronising)
        w.host_hint[0] = w.st->need_big;
        w.host_hint[2] = w.st->nlarge_bodies > 0 ? 1 : 0;   // a grid-wide island exists: launch k_solve_large
        w.st->need_big = 0;
        w.st->coop_streamed = 0;
        w.st->coop_resident = 0;
        w.st->cursor_rest = 0;
        w.st->cursor_coop = 0;
    }
    {   // CCD clamps queued by the last step's body writeback (rb_solver.cuh): applied before anything reads the poses.
        // Every CTA reads the count before the barrier, thread 0 resets it after it.
        const int nccd = w.st->nccd;
        if (nccd > 0) {
            const int npass = w.st->nccd_bullets > 0 ? 2 : 1;
#pragma unroll 1
            for (int pass = 0; pass < npass; ++pass) {   // (one inlined copy of the sweep: the kernel's stack frame stays small)
                phase_ccd_pending(ctx, w, nccd, pass == 1);
                ctx.grid_sync();
            }
            if (ctx.gtid == 0) { w.st->nccd = 0; w.st->nccd_bullets = 0; w.host_hint[3] = 0; }
        }
    }
    collide_pipeline<SHAPES>(ctx, w);   // (ends with a grid barrier: after the narrow phase, or after the last optional section)
    if (!do_solve) return;
    {
        BlockCtx bctx;
        SmemBodies bd;
        bd.s = smem;
        BlockExec ex;
        ex.c = &bctx;
        RB_SHARED int s_next;
        const int n = w.st->norder;
        for (;;) {   // items that are not shared-memory items, most expensive first
            if (bctx.btid == 0) s_next = atomic_add(&w.st->cursor_rest, 1);
            bctx.block_sync();
            const int k = s_next;
            bctx.block_sync();
            if (k >= n) break;
            const int item = w.item_order[k];
            if (item_is_coop(w, item)) continue;
            solve_item<HbmRows<0, 0>>(ex, w, bd, item, mk3(g.x, g.y, g.z));
            ex.sync();
        }
    }
    // The grid-wide "large" item 0 normally has its own launch (k_solve_large, register budget and work placement of
    // its own).  The host decides that launch from a hint that is one step old, so the step in which a large island
    // first appears is solved here instead (do_solve bit 1 clear = no k_solve_large follows).
    if (w.st->nlarge_bodies == 0 || (do_solve & 2)) return;
    GlobalBodies gb;
    gb.w = &w;
    GridSpreadExec gex;
    gex.c = &ctx;
    solve_item<PoolRows<CONS_LANES>>(gex, w, gb, 0, mk3(g.x, g.y, g.z));
}
// The grid-wide item 0: islands too large for one CTA (pyramid3, keva3, joint grids).  Cooperative, one CTA per SM;
// bodies in the global solver-body tables, constant rows in the L2-resident large pool, one grid barrier per colour
// stage; consecutive warps of a stage's constraints go to different SMs (GridSpreadExec).
RB_KERNEL RB_BOUNDS(COLLIDE_THREADS, 1) k_solve_large(World w, Grav g) {
    GridCtx ctx;
    if (w.st->nlarge_bodies == 0) return;
    GlobalBodies gb;
    gb.w = &w;
    GridSpreadExec gex;
    gex.c = &ctx;
    solve_item<PoolRows<CONS_LANES>>(gex, w, gb, 0, mk3(g.x, g.y, g.z));
}
// The general solve path, compiled per (friction model FM, joint model JM):
//   FM = 1  FrictionModel::Coulomb (integration_parameters.rs:26-29): one coupled tangent part per contact point
//   JM = 1  some joint has limits or motors (joint_velocity_constraint.rs:145-357): generic joint rows
// Every work item takes the streaming solve (solve_item<HbmRows<FM, JM>>: bodies in shared memory, rows in HBM/L2), the
// grid-wide item 0 the same code with grid barriers.  The twist / locked-axes kernels carry none of this code.
template <int FM, int JM>
RB_KERNEL RB_BOUNDS(COLLIDE_THREADS) k_solve_items_x(World w, Grav g) {
    RB_DYNAMIC_SMEM(smem);
    BlockCtx bctx;
    SmemBodies bd;
    bd.s = smem;
    BlockExec ex;
    ex.c = &bctx;
    RB_SHARED int s_next;
    const int n = w.st->norder;
    for (;;) {
        if (bctx.btid == 0) s_next = atomic_add(&w.st->cursor_rest, 1);
        bctx.block_sync();
        const int k = s_next;
        bctx.block_sync();
        if (k >= n) break;
        solve_item<HbmRows<FM, JM>>(ex, w, bd, w.item_order[k], mk3(g.x, g.y, g.z));
        ex.sync();
    }
}
template <int FM, int JM>
RB_KERNEL RB_BOUNDS(COLLIDE_THREADS, 1) k_solve_large_x(World w, Grav g) {
    GridCtx ctx;
    if (w.st->nlarge_bodies == 0) return;
    GlobalBodies gb;
    gb.w = &w;
    GridExec gex;
    gex.c = &ctx;
    solve_item<HbmRows<FM, JM>>(gex, w, gb, 0, mk3(g.x, g.y, g.z));
}
// Shared-memory items: one CTA per item, bodies (and, when they fit, constraints) staged in shared memory,
// four lanes per constraint (rb_solver.cuh "lane-cooperative path").
// Either launch shape takes every shared-memory item (the small one streams what does not fit), so the
// host's choice between them -- a hint read without synchronising -- only affects speed.
template <int L>
RB_D void solve_coop_items(const World& w, const Grav& g, int smem_floats) {
    RB_DYNAMIC_SMEM(smem);
    RB_SHARED __align__(8) unsigned long long s_mbar[2];
    BlockCtx ctx;
    if (ctx.btid == 0) {
        mbar_init(&s_mbar[0], 1);
        mbar_init(&s_mbar[1], 1);
        mbar_init_fence();
    }
    ctx.block_sync();
    CoopPipe pp;
    pp.mbar = s_mbar;
    pp.t = 0;
    pp.sweep_threads = ctx.bsize;   // (set per item)
    RB_SHARED int s_next;
    const int n = w.st->norder;
    int* cursor = &w.st->cursor_coop;
    for (;;) {   // dynamic queue over the cost-ordered items
        if (ctx.btid == 0) s_next = atomic_add(cursor, 1);
        ctx.block_sync();
        const int k = s_next;
        ctx.block_sync();
        if (k >= n) break;
        const int item = w.item_order[k];
        if (!item_is_coop(w, item)) continue;
        solve_item_coop<L>(ctx, w, smem, smem_budget(smem_floats), pp, item, mk3(g.x, g.y, g.z));
        ctx.block_sync();
    }
}
// The two launch shapes (COOP_SMALL_* / COOP_BIG_*): same code, different register budgets.
RB_KERNEL RB_BOUNDS(COOP_SMALL_THREADS, 2) k_solve_coop(World w, Grav g) { solve_coop_items<CONS_LANES>(w, g, COOP_SMALL_SMEM_BYTES / 4); }
RB_KERNEL RB_BOUNDS(COOP_BIG_THREADS, 1) k_solve_coop_big(World w, Grav g) { solve_coop_items<1>(w, g, COOP_BIG_SMEM_BYTES / 4); }
RB_KERNEL k_kat(World w, int which, const float* in, float* out) { kat_phase(w, which, in, out); }
// Contact force events of the step just solved (launched only for worlds in which a collider asks for them).
RB_KERNEL k_force_events(World w) {
    GridCtx ctx;
    phase_force_events(ctx, w);
}
// The CCD clamps queued by the last step's body writeback (rb_solver.cuh) when NO further step follows: a synchronising
// call launches this (one CTA: fast bodies are rare) if the device flagged any; otherwise the next k_collide applies them.
RB_KERNEL k_ccd_pending(World w) {
    GridCtx ctx;
    const int n = w.st->nccd;
    if (n == 0) return;
    const int npass = w.st->nccd_bullets > 0 ? 2 : 1;
#pragma unroll 1
    for (int pass = 0; pass < npass; ++pass) {
        phase_ccd_pending(ctx, w, n, pass == 1);
        ctx.block_sync();
    }
    if (ctx.gtid == 0) { w.st->nccd = 0; w.st->nccd_bullets = 0; w.host_hint[3] = 0; }
}
RB_KERNEL k_init_bodies(World w, int first) {
    GridCtx ctx;
    init_bodies_phase(ctx, w, first);
}
RB_KERNEL k_wake(World w, const int* idx, int n) {
    GridCtx ctx;
    wake_phase(ctx, w, idx, n);
}
RB_KERNEL k_wake_apply(World w) {
    GridCtx ctx;
    wake_apply_phase(ctx, w);
}
RB_KERNEL k_import_halo(World w) {
    GridCtx ctx;
    import_halo_phase(ctx, w);
}
RB_KERNEL k_set_halo(World w, const unsigned char* flags) {
    GridCtx ctx;
    set_halo_phase(ctx, w, flags);
}
RB_KERNEL k_import_states(World w, const int* idx, const float* src, int n, int table) {
    GridCtx ctx;
    import_states_phase(ctx, w, idx, src, n, table);
}

// ------------------------------------------------------------------------------------------------
// host-side world
// ------------------------------------------------------------------------------------------------
struct RbWorld {
    World w{};
    RbIntegrationParameters params{};
    std::vector<RbBodyDesc> bodies;
    std::vector<RbColliderDesc> colliders;
    std::vector<RbJointDesc> joints;
    std::vector<void*> allocs;
    int reserve_bodies = 0, reserve_colliders = 0;   // rb_world_reserve: room for later insertions
    int body_cap = 0, collider_cap = 0;               // allocated table lengths of the current scene
    int device = 0;
    int num_sms = 1;
    int collide_blocks = 1, coop_blocks = 1;
    int coop_blocks_big = 1;
    float* state_buf[2] = {nullptr, nullptr};   // double-buffered packed state (rb_world_state_buffers), else unused
    int state_next = 0;
    bool ext_shapes = false;     // some collider is a capsule or a convex polyhedron: the SHAPES = 1 collision kernel
    std::vector<rbhull::Hull> hulls;   // convex polyhedra (rb_world_add_hull); hull 0 = the unit cube
    int hulls_uploaded = 0;            // how many of them the device tables hold
    bool force_events = false;   // some collider has RB_EVENT_CONTACT_FORCE: run k_force_events after every step
    std::vector<unsigned char> joint_removed;   // tombstones of rb_world_remove_joints (slots stay allocated)
    int reserve_joints = 0, reserve_generic = 0;   // rb_world_reserve_joints
    std::vector<int> extra_keys; // distinct additional_solver_iterations of the bodies, descending (substep solve-groups); {0} = none
    int steps_since_scene = 0;   // the launch-shape hint of a new scene is awaited once (see rb_world_step)
    int coop_shape = -1;   // RB_COOP_SHAPE debugging override: 0 small, 1 big, -1 automatic
    int* host_hint = nullptr;
    long long kernels = 0, steps = 0;
    bool profiling = false;
    float ms_collide = 0, ms_solve = 0, ms_step = 0;
    int njused = 0;
    float* stage_dev = nullptr;      // [nb*13] device staging for bulk state import
    int* ident_dev = nullptr;        // [nb] identity index list
    float* stage_host = nullptr;     // pinned host staging (2 * nb * 13 floats: in, out)
    cudaStream_t stream = nullptr;   // (the emulation has none)
#if RB_DEVICE_BUILD
    bool own_stream = true;
    std::vector<cudaEvent_t> prof_ev;   // 3 events per profiled step
    int prof_steps = 0;
#else
    std::vector<float> emu_smem;   // dynamic shared memory of the emulated kernels
    int emu_coop_floats = COOP_BIG_SMEM_BYTES / 4, emu_hint[4] = {0, 0, 0, 0};
#endif
};

template <class T> struct same_type { using type = T; };
// Launches `kernel` on the world's stream and counts it.  The emulation calls it as one CTA of one thread, with
// `smem_bytes` of host memory as its dynamic shared memory, of which it may plan with at most emu_coop_floats.
template <class... P>
static cudaError_t launch(RbWorld* W, void (*kernel)(P...), int grid, int block, size_t smem_bytes, bool cooperative,
                          typename same_type<P>::type... args) {
#if RB_DEVICE_BUILD
    void* argv[] = {(void*)&args...};
    const cudaError_t e = cooperative ? cudaLaunchCooperativeKernel((void*)kernel, dim3(grid), dim3(block), argv, smem_bytes, W->stream)
                                      : cudaLaunchKernel((void*)kernel, dim3(grid), dim3(block), argv, smem_bytes, W->stream);
    const cudaError_t last = cudaGetLastError();
    if (e != cudaSuccess || last != cudaSuccess) return e != cudaSuccess ? e : last;
#else
    (void)grid; (void)block; (void)cooperative;
    const int floats = (int)(smem_bytes / 4);
    if ((int)W->emu_smem.size() < floats) W->emu_smem.resize(floats);
    emu_smem.p = W->emu_smem.data();
    emu_smem.budget = std::min(floats, W->emu_coop_floats);
    kernel(args...);
#endif
    W->kernels++;
    return cudaSuccess;
}

template <class T>
static int alloc_arr(RbWorld* W, T** p, size_t count) {
    void* v = nullptr;
    if (dev_alloc(&v, count * sizeof(T)) != cudaSuccess) { set_err("device allocation failed%s", ""); return RB_ERR_CUDA; }
    W->allocs.push_back(v);
    *p = (T*)v;
    return RB_OK;
}
#define ALLOC(ptr, count)                                   \
    do {                                                    \
        int rc_ = alloc_arr(W, &(ptr), (size_t)(count));    \
        if (rc_ != RB_OK) return rc_;                       \
    } while (0)

static void free_all(RbWorld* W) {
    for (void* p : W->allocs) dev_free(p);
    W->allocs.clear();
}

static int next_pow2_host(int n) { int p = 1; while (p < n) p <<= 1; return p; }

// The general solve path: every item, the grid-wide item 0 included, through solve_item<HbmRows<FM, JM>>.
static bool general_path(const World& w) { return w.prm.friction_model == 1 || w.generic_joints != 0 || w.any_extra != 0; }
// Calls f(FM, JM) with the compile-time variant of the general path as std::integral_constant values:
// FM = 1 FrictionModel::Coulomb, JM = 1 generic joints.
template <class F>
static auto with_variant(bool fm, bool jm, F&& f) {
    using I0 = std::integral_constant<int, 0>;
    using I1 = std::integral_constant<int, 1>;
    if (fm && jm) return f(I1(), I1());
    if (fm) return f(I1(), I0());
    if (jm) return f(I0(), I1());
    return f(I0(), I0());
}
template <class F>
static auto with_variant(const World& w, F&& f) { return with_variant(w.prm.friction_model == 1, w.generic_joints != 0, f); }

// Derived solver coefficients (integration_parameters.rs:85-149, :305-377; init.rs:96-101).
static void derive_params(const RbIntegrationParameters& p_in, Params& o, int extra_substeps = 0) {
    RbIntegrationParameters p = p_in;   // a substep solve-group: num_solver_iterations + extra at dt / that count (init.rs:64-66)
    p.num_solver_iterations += extra_substeps;
    auto erp_inv_dt = [](float f, float z, float dt) { float w = f * 6.283185307179586f; return w / (dt * w + 2.0f * z); };
    auto cfm_factor = [&](float f, float z, float dt) {
        float e = dt * erp_inv_dt(f, z, dt);
        float c = 0.0f;
        if (e != 0.0f) {
            float e1 = 1.0f / e - 1.0f;
            c = e1 * e1 / ((1.0f + e1) * 4.0f * z * z);
        }
        return 1.0f / (1.0f + c);
    };
    o.dt = p.dt;
    o.inv_dt_full = p.dt == 0.0f ? 0.0f : 1.0f / p.dt;
    o.num_substeps = p.num_solver_iterations;
    o.sub_dt = p.dt / (float)p.num_solver_iterations;
    o.sub_inv_dt = o.sub_dt == 0.0f ? 0.0f : 1.0f / o.sub_dt;
    o.dyn_cfm = cfm_factor(p.contact_natural_frequency, p.contact_damping_ratio, o.sub_dt);
    o.static_cfm = cfm_factor(p.static_contact_natural_frequency, p.static_contact_damping_ratio, o.sub_dt);
    o.dyn_erp = erp_inv_dt(p.contact_natural_frequency, p.contact_damping_ratio, o.sub_dt);
    o.static_erp = erp_inv_dt(p.static_contact_natural_frequency, p.static_contact_damping_ratio, o.sub_dt);
    o.max_corrective_velocity = p.normalized_max_corrective_velocity * p.length_unit;
    o.warmstart_coeff = p.warmstart_coefficient;
    o.prediction = p.normalized_prediction_distance * p.length_unit;
    o.recycle_dist = p.normalized_contact_recycle_distance * p.length_unit;
    o.length_unit = p.length_unit;
    o.fat_skin = 4.0e-2f * p.length_unit;   // BroadPhaseBvh::CHANGE_DETECTION_FACTOR (broad_phase_bvh/mod.rs:175)
    o.max_lin_vel = p.normalized_max_linear_velocity * p.length_unit;
    o.max_ang_vel = 0.7853981633974483f * o.inv_dt_full;   // MAX_ROTATION * inv_dt (worker.rs:573-580)
    o.num_pgs = p.num_internal_pgs_iterations;
    o.num_relax = p.num_internal_stabilization_iterations;
    o.friction_in_bias = p.friction_in_bias_pass;
    o.contact_recycling = p.contact_recycling;
    o.friction_model = p.friction_model;
    o.warmstart_joints = p.warmstart_joints != 0 ? 1 : 0;
    o.ccd = p.max_ccd_substeps != 0 ? 1 : 0;
    o.linear_slop = p.normalized_allowed_linear_error * p.length_unit;
}

// Substep solve-groups: the distinct additional_solver_iterations among the bodies (an island's key is the max over its
// members, so it is always one of these), descending as the reference orders its groups (substep_groups.rs:18-20).
static void refresh_extra_keys(RbWorld* W) {
    bool seen[256] = {false};
    seen[0] = true;
    for (const RbBodyDesc& d : W->bodies) seen[RB_BODY_EXTRA_ITERS_OF(d.flags)] = true;
    W->extra_keys.clear();
    for (int k = 255; k >= 0; --k)
        if (seen[k]) W->extra_keys.push_back(k);
    W->w.any_extra = W->extra_keys.size() > 1 ? 1 : 0;
    W->w.pass_key = 0;
}

static int validate_params(const RbIntegrationParameters* p) {
    if (!p) { set_err("null parameters%s", ""); return RB_ERR_INVALID; }
    if (p->friction_model != 0 && p->friction_model != 1) { set_err("friction_model must be 0 (Simplified) or 1 (Coulomb)%s", ""); return RB_ERR_INVALID; }
    if (p->warmstart_joints != 0 && p->warmstart_joints != 1) { set_err("warmstart_joints must be 0 or 1%s", ""); return RB_ERR_INVALID; }
    if (p->max_ccd_substeps < 0 || p->max_ccd_substeps > 1) { set_err("max_ccd_substeps must be 0 (CCD off) or 1 (motion clamping); the multi-substep splitter is not supported%s", ""); return RB_ERR_INVALID; }
    if (p->num_solver_iterations < 1 || p->num_solver_iterations > 64) { set_err("num_solver_iterations out of range%s", ""); return RB_ERR_INVALID; }
    return RB_OK;
}

// parry MassProperties::{from_cuboid, from_ball} (see oracle/oracle_world.cpp for the citation chain).
static void collider_mass_props(const RbColliderDesc& c, float& mass, float pi[3]) {
    if (c.shape == RB_SHAPE_CUBOID) {
        float hx = c.half_extents[0], hy = c.half_extents[1], hz = c.half_extents[2];
        float vol = hx * hy * hz * 8.0f;
        float sx = hx * hx, sy = hy * hy, sz = hz * hz;
        float third = 1.0f / 3.0f;
        float ux = (sy + sz) * third, uy = (sx + sz) * third, uz = (sx + sy) * third;
        mass = vol * c.density;
        pi[0] = ux * mass; pi[1] = uy * mass; pi[2] = uz * mass;
    } else if (c.shape == RB_SHAPE_CAPSULE) {
        // parry MassProperties::from_capsule: a cylinder plus the two half balls (restated from the published formulas)
        const float hh = c.half_extents[0], r = c.half_extents[1];
        const int ax = (int)c.half_extents[2];
        const float pi_ = 3.14159265358979323846f;
        const float cyl_vol = hh * r * r * pi_ * 2.0f, ball_vol = pi_ * r * r * r * 4.0f / 3.0f;
        const float sq_r = r * r, sq_h = hh * hh * 4.0f;
        const float cyl_off = (sq_r * 3.0f + sq_h) / 12.0f, cyl_axis = sq_r / 2.0f, ball_unit = sq_r * 2.0f / 5.0f;
        const float h = hh * 2.0f;
        const float extra = (h * h * 0.25f + h * r * 3.0f / 8.0f) * ball_vol * c.density;
        const float i_off = (cyl_off * cyl_vol + ball_unit * ball_vol) * c.density + extra;
        const float i_axis = (cyl_axis * cyl_vol + ball_unit * ball_vol) * c.density;
        mass = (cyl_vol + ball_vol) * c.density;
        pi[0] = pi[1] = pi[2] = i_off;
        pi[ax] = i_axis;
    } else {
        float r = c.half_extents[0];
        float vol = 3.14159265358979323846f * r * r * r * 4.0f / 3.0f;
        float unit = r * r * 2.0f / 5.0f;
        mass = vol * c.density;
        pi[0] = pi[1] = pi[2] = unit * mass;
    }
}
static inline float inv0(float x) { return x == 0.0f ? 0.0f : 1.0f / x; }
static inline bool type_moves(int t) { return t == RB_BODY_DYNAMIC || t == RB_BODY_KINEMATIC_POSITION_BASED || t == RB_BODY_KINEMATIC_VELOCITY_BASED; }

struct HostMass { float lcom[3], inv_mass, ipi[3], pi[3], pframe[4], max_extent, ccd_thickness; };

// General composite mass properties (MassProperties sum + from_inertia_tensor / symmetric eigen-decomposition [parry],
// restated): parts with mass m_i, principal inertia pi_i in their own frame (rotation q_i, centre t_i).  Sums the world
// tensors about the common centre of mass (parallel-axis theorem) in double precision and diagonalises the sum with cyclic
// Jacobi rotations.  Outputs the centre of mass, the principal inertia and the principal frame (x, y, z, w).
static void composite_inertia(int n, const float* mass, const float (*pi)[3], const float (*q)[4], const float (*t)[3],
                              float com_out[3], float pi_out[3], float frame_out[4]) {
    double M = 0.0, com[3] = {0.0, 0.0, 0.0};
    for (int i = 0; i < n; ++i) {
        M += (double)mass[i];
        for (int k = 0; k < 3; ++k) com[k] += (double)t[i][k] * (double)mass[i];
    }
    for (int k = 0; k < 3; ++k) com[k] /= M;
    double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = 0; i < n; ++i) {
        const double x = q[i][0], y = q[i][1], z = q[i][2], w = q[i][3];
        const double R[3][3] = {{1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w), 2.0 * (x * z + y * w)},
                                {2.0 * (x * y + z * w), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w)},
                                {2.0 * (x * z - y * w), 2.0 * (y * z + x * w), 1.0 - 2.0 * (x * x + y * y)}};
        double d[3];
        for (int k = 0; k < 3; ++k) d[k] = (double)t[i][k] - com[k];
        const double d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) {
                double v = 0.0;
                for (int k = 0; k < 3; ++k) v += R[r][k] * (double)pi[i][k] * R[c][k];
                v += (double)mass[i] * ((r == c ? d2 : 0.0) - d[r] * d[c]);
                A[r][c] += v;
            }
    }
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 64; ++sweep) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        const double diag = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
        if (off <= 1.0e-30 * diag || off == 0.0) break;
        for (int p = 0; p < 2; ++p)
            for (int r = p + 1; r < 3; ++r) {
                if (A[p][r] == 0.0) continue;
                const double theta = (A[r][r] - A[p][p]) / (2.0 * A[p][r]);
                const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
                for (int k = 0; k < 3; ++k) {   // A <- A J
                    const double akp = A[k][p], akr = A[k][r];
                    A[k][p] = c * akp - s * akr;
                    A[k][r] = s * akp + c * akr;
                }
                for (int k = 0; k < 3; ++k) {   // A <- J^T A
                    const double apk = A[p][k], ark = A[r][k];
                    A[p][k] = c * apk - s * ark;
                    A[r][k] = s * apk + c * ark;
                }
                for (int k = 0; k < 3; ++k) {   // V <- V J
                    const double vkp = V[k][p], vkr = V[k][r];
                    V[k][p] = c * vkp - s * vkr;
                    V[k][r] = s * vkp + c * vkr;
                }
            }
    }
    // a proper rotation: flip the third axis if the eigenvectors came out left-handed
    const double det = V[0][0] * (V[1][1] * V[2][2] - V[1][2] * V[2][1]) - V[0][1] * (V[1][0] * V[2][2] - V[1][2] * V[2][0]) +
                       V[0][2] * (V[1][0] * V[2][1] - V[1][1] * V[2][0]);
    if (det < 0.0)
        for (int k = 0; k < 3; ++k) V[k][2] = -V[k][2];
    // rotation matrix -> quaternion (largest-component branch)
    double qw, qx, qy, qz;
    const double tr = V[0][0] + V[1][1] + V[2][2];
    if (tr > 0.0) {
        const double s = sqrt(tr + 1.0) * 2.0;
        qw = 0.25 * s; qx = (V[2][1] - V[1][2]) / s; qy = (V[0][2] - V[2][0]) / s; qz = (V[1][0] - V[0][1]) / s;
    } else if (V[0][0] > V[1][1] && V[0][0] > V[2][2]) {
        const double s = sqrt(1.0 + V[0][0] - V[1][1] - V[2][2]) * 2.0;
        qw = (V[2][1] - V[1][2]) / s; qx = 0.25 * s; qy = (V[0][1] + V[1][0]) / s; qz = (V[0][2] + V[2][0]) / s;
    } else if (V[1][1] > V[2][2]) {
        const double s = sqrt(1.0 + V[1][1] - V[0][0] - V[2][2]) * 2.0;
        qw = (V[0][2] - V[2][0]) / s; qx = (V[0][1] + V[1][0]) / s; qy = 0.25 * s; qz = (V[1][2] + V[2][1]) / s;
    } else {
        const double s = sqrt(1.0 + V[2][2] - V[0][0] - V[1][1]) * 2.0;
        qw = (V[1][0] - V[0][1]) / s; qx = (V[0][2] + V[2][0]) / s; qy = (V[1][2] + V[2][1]) / s; qz = 0.25 * s;
    }
    const double qn = sqrt(qx * qx + qy * qy + qz * qz + qw * qw);
    frame_out[0] = (float)(qx / qn); frame_out[1] = (float)(qy / qn); frame_out[2] = (float)(qz / qn); frame_out[3] = (float)(qw / qn);
    for (int k = 0; k < 3; ++k) { com_out[k] = (float)com[k]; pi_out[k] = (float)A[k][k]; }
}


// RigidBodyMassProps::recompute_mass_properties_from_colliders (rigid_body_components.rs:421).
// `first_body` / `first_collider`: only the bodies from first_body on are computed, from the colliders from
// first_collider on (rb_world_insert: appended bodies carry appended colliders only).
static int host_mass_props(const RbWorld* W, std::vector<HostMass>& out, int first_body = 0, int first_collider = 0) {
    int nb = (int)W->bodies.size();
    out.assign(nb, HostMass{});
    std::vector<int> count(nb, 0), first(nb, -1);
    for (int ci = first_collider; ci < (int)W->colliders.size(); ++ci) {
        int p = W->colliders[ci].parent;
        if (W->colliders[ci].sensor && W->colliders[ci].density == 0.0f) continue;   // a massless sensor adds nothing (and must not force the composite path)
        if (p >= 0) { if (count[p] == 0) first[p] = ci; count[p]++; }
    }
    for (int b = first_body; b < nb; ++b) {
        HostMass& m = out[b];
        m.pframe[3] = 1.0f;
        if (count[b] == 1) {
            const RbColliderDesc& c = W->colliders[first[b]];
            float mass, pi[3];
            if (c.shape == RB_SHAPE_CONVEX) {
                // MassProperties::from_convex_polyhedron [parry]: the hull's unit-density properties scaled by the density,
                // centre of mass and principal frame carried through the collider's pose (double arithmetic, rounded once)
                const rbhull::Hull& h = W->hulls[(int)c.half_extents[0]];
                mass = h.volume * c.density;
                for (int k = 0; k < 3; ++k) pi[k] = h.principal_inertia[k] * c.density;
                const double q[4] = {c.pos_wrt_parent_q[0], c.pos_wrt_parent_q[1], c.pos_wrt_parent_q[2], c.pos_wrt_parent_q[3]};
                const double v[3] = {h.com[0], h.com[1], h.com[2]};
                double t[3], u[3];
                rbhull::cross3d(q, v, t);
                for (int k = 0; k < 3; ++k) t[k] *= 2.0;
                rbhull::cross3d(q, t, u);
                for (int k = 0; k < 3; ++k) m.lcom[k] = (float)((double)c.pos_wrt_parent_t[k] + (v[k] + q[3] * t[k] + u[k]));
                const double g[4] = {h.principal_frame[0], h.principal_frame[1], h.principal_frame[2], h.principal_frame[3]};
                m.pframe[0] = (float)(q[3] * g[0] + q[0] * g[3] + q[1] * g[2] - q[2] * g[1]);
                m.pframe[1] = (float)(q[3] * g[1] - q[0] * g[2] + q[1] * g[3] + q[2] * g[0]);
                m.pframe[2] = (float)(q[3] * g[2] + q[0] * g[1] - q[1] * g[0] + q[2] * g[3]);
                m.pframe[3] = (float)(q[3] * g[3] - q[0] * g[0] - q[1] * g[1] - q[2] * g[2]);
                for (int k = 0; k < 3; ++k) m.ipi[k] = inv0(pi[k]);
                m.inv_mass = inv0(mass);
            } else {
            collider_mass_props(c, mass, pi);
            for (int k = 0; k < 3; ++k) { m.lcom[k] = c.pos_wrt_parent_t[k]; m.ipi[k] = inv0(pi[k]); }
            m.inv_mass = inv0(mass);
            for (int k = 0; k < 4; ++k) m.pframe[k] = c.pos_wrt_parent_q[k];
            }
        } else if (count[b] > 1) {
            float M = 0.0f, com[3] = {0, 0, 0};
            bool simple = true;   // axis-aligned parts whose offsets from the centre of mass lie along one axis: the summed tensor is diagonal
            for (size_t ci = (size_t)first_collider; ci < W->colliders.size(); ++ci) {
                const RbColliderDesc& c = W->colliders[ci];
                if (c.parent != b || (c.sensor && c.density == 0.0f)) continue;
                if (c.shape == RB_SHAPE_CONVEX) { set_err("multi-collider bodies with convex polyhedra are not supported%s", ""); return RB_ERR_INVALID; }
                float mass, pi[3];
                collider_mass_props(c, mass, pi);
                M = M + mass;
                for (int k = 0; k < 3; ++k) com[k] = com[k] + c.pos_wrt_parent_t[k] * mass;
            }
            if (M != 0.0f) {
                float invM = 1.0f / M;
                for (int k = 0; k < 3; ++k) com[k] = com[k] * invM;
                for (size_t ci = (size_t)first_collider; ci < W->colliders.size(); ++ci) {
                    const RbColliderDesc& c = W->colliders[ci];
                    if (c.parent != b || (c.sensor && c.density == 0.0f)) continue;
                    if (!(c.pos_wrt_parent_q[0] == 0.0f && c.pos_wrt_parent_q[1] == 0.0f && c.pos_wrt_parent_q[2] == 0.0f)) simple = false;
                    float d[3];
                    for (int k = 0; k < 3; ++k) d[k] = c.pos_wrt_parent_t[k] - com[k];
                    if ((d[0] != 0.0f) + (d[1] != 0.0f) + (d[2] != 0.0f) > 1) simple = false;
                }
                if (simple) {
                    float I[3] = {0, 0, 0};
                    for (size_t ci = (size_t)first_collider; ci < W->colliders.size(); ++ci) {
                        const RbColliderDesc& c = W->colliders[ci];
                        if (c.parent != b || (c.sensor && c.density == 0.0f)) continue;
                        float mass, pi[3];
                        collider_mass_props(c, mass, pi);
                        float d[3];
                        for (int k = 0; k < 3; ++k) d[k] = c.pos_wrt_parent_t[k] - com[k];
                        float d2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
                        for (int k = 0; k < 3; ++k) I[k] = I[k] + pi[k] + (d2 - d[k] * d[k]) * mass;
                    }
                    for (int k = 0; k < 3; ++k) { m.lcom[k] = com[k]; m.ipi[k] = inv0(I[k]); }
                } else {   // compound bodies in general (e.g. stress_tests/compound3.rs): full tensor, principal axes by eigen-decomposition
                    std::vector<float> pm;
                    std::vector<std::array<float, 3>> ppi, pt;
                    std::vector<std::array<float, 4>> pq;
                    for (size_t ci = (size_t)first_collider; ci < W->colliders.size(); ++ci) {
                        const RbColliderDesc& c = W->colliders[ci];
                        if (c.parent != b || (c.sensor && c.density == 0.0f)) continue;
                        float mass, pi[3];
                        collider_mass_props(c, mass, pi);
                        pm.push_back(mass);
                        ppi.push_back({pi[0], pi[1], pi[2]});
                        pt.push_back({c.pos_wrt_parent_t[0], c.pos_wrt_parent_t[1], c.pos_wrt_parent_t[2]});
                        pq.push_back({c.pos_wrt_parent_q[0], c.pos_wrt_parent_q[1], c.pos_wrt_parent_q[2], c.pos_wrt_parent_q[3]});
                    }
                    float I[3];
                    composite_inertia((int)pm.size(), pm.data(), reinterpret_cast<const float(*)[3]>(ppi.data()), reinterpret_cast<const float(*)[4]>(pq.data()),
                                      reinterpret_cast<const float(*)[3]>(pt.data()), m.lcom, I, m.pframe);
                    for (int k = 0; k < 3; ++k) m.ipi[k] = inv0(I[k]);
                }
                m.inv_mass = inv0(M);
            }
        }
        // RigidBodyAdditionalMassProps::Mass (rigid_body_components.rs:454-486); MassProperties::set_mass(m, true)
        // [parry] rescales the angular inertia by new_mass / old_mass, i.e. its inverse by inv(new) * old.
        const float add = W->bodies[b].additional_mass;
        if (add > 0.0f) {
            const float prev = inv0(m.inv_mass);
            if (prev > 0.0f) {
                const float inv_new = inv0(prev + add);
                for (int k = 0; k < 3; ++k) m.ipi[k] = m.ipi[k] * (inv_new * prev);
                m.inv_mass = inv_new;
            } else if (count[b] == 1 && W->colliders[first[b]].shape == RB_SHAPE_CONVEX) {
                set_err("additional mass on a massless convex polyhedron is not supported%s", "");
                return RB_ERR_INVALID;
            } else if (count[b] == 1) {
                // massless collider: inertia and centre of mass of the shape at unit density, rescaled to the mass
                RbColliderDesc u = W->colliders[first[b]];
                u.density = 1.0f;
                float um, upi[3];
                collider_mass_props(u, um, upi);
                const float inv_new = inv0(add);
                for (int k = 0; k < 3; ++k) { m.lcom[k] = u.pos_wrt_parent_t[k]; m.ipi[k] = inv0(upi[k]) * (inv_new * um); }
                for (int k = 0; k < 4; ++k) m.pframe[k] = u.pos_wrt_parent_q[k];
                m.inv_mass = inv_new;
            } else if (count[b] == 0) {
                m.inv_mass = inv0(add);   // no shape to derive an inertia from: just the mass
            } else {
                set_err("additional mass on a massless multi-collider body is not supported%s", "");
                return RB_ERR_INVALID;
            }
        }
        for (int k = 0; k < 3; ++k) m.pi[k] = inv0(m.ipi[k]);
        // recompute_max_extent (rigid_body_components.rs:491-515): bounding spheres about the local centre of mass
        m.max_extent = 0.0f;
        m.ccd_thickness = 3.4028235e38f;   // RigidBodyCcd::default (rigid_body_components.rs:1076), min over the colliders (:1224-1228)
        for (size_t ci = (size_t)first_collider; ci < W->colliders.size(); ++ci) {
            const RbColliderDesc& c = W->colliders[ci];
            if (c.parent != b) continue;
            const float hx = c.half_extents[0], hy = c.half_extents[1], hz = c.half_extents[2];
            if (c.shape != RB_SHAPE_CAPSULE && c.shape != RB_SHAPE_CONVEX)   // (capsules and polyhedra are never swept here, like the reference's never-swept shapes: they do not count, rigid_body_components.rs:1224-1228)
                m.ccd_thickness = std::min(m.ccd_thickness, c.shape == RB_SHAPE_BALL ? hx : std::min(hx, std::min(hy, hz)));   // parry Shape::ccd_thickness
            const float radius = c.shape == RB_SHAPE_CONVEX ? W->hulls[(int)hx].radius + hy
                               : c.shape == RB_SHAPE_BALL ? hx : (c.shape == RB_SHAPE_CAPSULE ? hx + hy : sqrtf(fmaf(hz, hz, fmaf(hy, hy, hx * hx))));
            const float dx = c.pos_wrt_parent_t[0] - m.lcom[0], dy = c.pos_wrt_parent_t[1] - m.lcom[1], dz = c.pos_wrt_parent_t[2] - m.lcom[2];
            m.max_extent = std::max(m.max_extent, sqrtf(fmaf(dz, dz, fmaf(dy, dy, dx * dx))) + radius);
        }
    }
    return RB_OK;
}

static int launch_init_bodies(RbWorld* W, int first = 0) {
    CK(launch(W, k_init_bodies, std::max((W->w.nb - first + 255) / 256, 1), 256, 0, false, W->w, first));
    return RB_OK;
}

// Waits for the world's stream.  `check`: also report (and clear) a status the device raised since the last check --
// capacity overflow or non-finite state -- so asynchronous stepping (sync = 0, rb_world_step_host) cannot hide it.
static int sync_world(RbWorld* W, bool check = true) {
    CK(stream_sync(W->stream));
    if (W->host_hint && W->w.st && *(volatile int*)(W->host_hint + 3) != 0) {   // CCD clamps queued by the last step: apply them now
        CK(launch(W, k_ccd_pending, 1, 256, 0, false, W->w));
        CK(stream_sync(W->stream));
    }
    if (check && W->host_hint && W->w.st) {
        const int code = *(volatile int*)(W->host_hint + 1);
        if (code != 0) {
            W->host_hint[1] = 0;
            int zero = 0;
            CK(h2d(&W->w.st->error, &zero, sizeof(int)));
            set_err(code == -6 ? "device raised status %s%d (a contact formed between bodies simulated by different ranks: the shards' islands merged, repartition)" : code == RB_ERR_NONFINITE ? "device raised status %s%d (non-finite body state: see rb_world_get_quarantine)"
                                             : "device raised status %s%d (capacity overflow: the step kept the previous pair set / truncated the schedule)", "", code);
            return code;
        }
    }
    return RB_OK;
}

extern "C" { static int wake_impl(RbWorld* W, const int32_t* indices_host, int n); }

static int read_state(RbWorld* W, State& s) {
    int rc = sync_world(W, false);   // (counters / debug reads must stay readable after an overflow; they do not consume the status)
    if (rc != RB_OK) return rc;
    CK(d2h(&s, W->w.st, sizeof(State)));
    return RB_OK;
}

// Upload the static data of bodies [first, first + count) / colliders [first, first + count) from the host copies.
static int upload_bodies(RbWorld* W, const std::vector<HostMass>& mp, int first, int count) {
    World& w = W->w;
    if (count <= 0) return RB_OK;
    std::vector<int> type(count);
    std::vector<unsigned> flags(count);
    std::vector<float4> pt(count), pq(count), lv(count), av(count), lc(count), ipi(count), pi(count), pf(count), misc(count), uf(count), ut(count);
    std::vector<float> ext(count), thick(count);
    std::vector<float4> prev_t(count, make_float4(0.f, 0.f, 0.f, 0.f)), prev_q(count, make_float4(0.f, 0.f, 0.f, 1.f));   // sleep_prev_pose = identity
    for (int k = 0; k < count; ++k) {
        const int i = first + k;
        ext[k] = mp[i].max_extent;
        thick[k] = mp[i].ccd_thickness;
        const RbBodyDesc& d = W->bodies[i];
        type[k] = d.body_type;
        flags[k] = d.body_type == RB_BODY_DYNAMIC ? d.flags : (d.flags & ~(unsigned)RB_BODY_GYROSCOPIC);   // gyroscopic term: dynamic bodies only (worker.rs:86)
        pt[k] = make_float4(d.translation[0], d.translation[1], d.translation[2], 0.f);
        pq[k] = make_float4(d.rotation[0], d.rotation[1], d.rotation[2], d.rotation[3]);
        lv[k] = make_float4(d.linvel[0], d.linvel[1], d.linvel[2], 0.f);
        av[k] = make_float4(d.angvel[0], d.angvel[1], d.angvel[2], 0.f);
        lc[k] = make_float4(mp[i].lcom[0], mp[i].lcom[1], mp[i].lcom[2], mp[i].inv_mass);
        ipi[k] = make_float4(mp[i].ipi[0], mp[i].ipi[1], mp[i].ipi[2], mp[i].max_extent);       // .w: copy of b_max_extent for the CCD test
        pi[k] = make_float4(mp[i].pi[0], mp[i].pi[1], mp[i].pi[2], 0.f);
        pf[k] = make_float4(mp[i].pframe[0], mp[i].pframe[1], mp[i].pframe[2], mp[i].pframe[3]);
        misc[k] = make_float4(d.linear_damping, d.angular_damping, d.gravity_scale, mp[i].ccd_thickness);   // .w: copy of b_ccd_thick
        uf[k] = make_float4(d.user_force[0], d.user_force[1], d.user_force[2], 0.f);
        ut[k] = make_float4(d.user_torque[0], d.user_torque[1], d.user_torque[2], 0.f);
    }
    const size_t n = (size_t)count;
    CK(h2d(w.b_type + first, type.data(), n * sizeof(int)));
    CK(h2d(w.b_flags + first, flags.data(), n * sizeof(unsigned)));
    CK(h2d(w.b_pos_t + first, pt.data(), n * sizeof(float4)));
    CK(h2d(w.b_pos_q + first, pq.data(), n * sizeof(float4)));
    CK(h2d(w.b_next_t + first, pt.data(), n * sizeof(float4)));   // next_position = position until the user sets a target
    CK(h2d(w.b_next_q + first, pq.data(), n * sizeof(float4)));
    CK(h2d(w.b_linvel + first, lv.data(), n * sizeof(float4)));
    CK(h2d(w.b_angvel + first, av.data(), n * sizeof(float4)));
    CK(h2d(w.b_lcom_im + first, lc.data(), n * sizeof(float4)));
    CK(h2d(w.b_ipi + first, ipi.data(), n * sizeof(float4)));
    CK(h2d(w.b_pi + first, pi.data(), n * sizeof(float4)));
    CK(h2d(w.b_pframe + first, pf.data(), n * sizeof(float4)));
    CK(h2d(w.b_misc + first, misc.data(), n * sizeof(float4)));
    CK(h2d(w.b_uforce + first, uf.data(), n * sizeof(float4)));
    CK(h2d(w.b_utorque + first, ut.data(), n * sizeof(float4)));
    CK(h2d(w.b_max_extent + first, ext.data(), n * sizeof(float)));
    CK(h2d(w.b_ccd_thick + first, thick.data(), n * sizeof(float)));
    CK(h2d(w.b_sleep_prev_t + first, prev_t.data(), n * sizeof(float4)));
    CK(h2d(w.b_sleep_prev_q + first, prev_q.data(), n * sizeof(float4)));
    CK(dev_set(w.b_sleeping + first, 0, n));
    CK(dev_set(w.b_sleep_time + first, 0, n * sizeof(float)));
    for (int k = 0; k < count; ++k)
        if (type_moves(type[k]) && !(flags[k] & RB_BODY_NO_SLEEP)) w.sleep_enabled = 1;
    {   // the position-based kinematic bodies, for the velocity interpolation at the start of the solve
        std::vector<int> kin;
        for (int i = 0; i < (int)W->bodies.size(); ++i)
            if (W->bodies[i].body_type == RB_BODY_KINEMATIC_POSITION_BASED) kin.push_back(i);
        w.nkinpos = (int)kin.size();
        if (!kin.empty()) CK(h2d(w.kinpos_list, kin.data(), kin.size() * sizeof(int)));
    }
    return RB_OK;
}
static int upload_colliders(RbWorld* W, int first, int count, int first_body = 0) {
    World& w = W->w;
    if (count <= 0) {
        const int nbn = (int)W->bodies.size() - first_body;
        if (nbn > 0) { std::vector<int> head(nbn, -1); CK(h2d(w.b_col_head + first_body, head.data(), (size_t)nbn * sizeof(int))); }
        return RB_OK;
    }
    std::vector<int> shape(count), parent(count);
    std::vector<float4> he(count), rt(count), rq(count), mat(count);
    std::vector<int2> rules(count);
    std::vector<uint2> groups(count);
    std::vector<int> events(count);
    std::vector<float> thr(count);
    for (int k = 0; k < count; ++k) {
        const RbColliderDesc& c = W->colliders[first + k];
        events[k] = (int)(c.active_events & 3u) | (c.sensor ? 4 : 0);
        if (c.sensor) w.has_sensors = 1;
        thr[k] = c.contact_force_event_threshold;
        if (c.active_events & RB_EVENT_CONTACT_FORCE) W->force_events = true;
        if (c.shape == RB_SHAPE_CAPSULE || c.shape == RB_SHAPE_CONVEX) W->ext_shapes = true;
        shape[k] = c.shape;
        parent[k] = c.parent;
        he[k] = make_float4(c.half_extents[0], c.half_extents[1], c.half_extents[2], 0.f);
        rt[k] = make_float4(c.pos_wrt_parent_t[0], c.pos_wrt_parent_t[1], c.pos_wrt_parent_t[2], 0.f);
        rq[k] = make_float4(c.pos_wrt_parent_q[0], c.pos_wrt_parent_q[1], c.pos_wrt_parent_q[2], c.pos_wrt_parent_q[3]);
        mat[k] = make_float4(c.friction, c.restitution, c.contact_skin, 0.f);
        rules[k] = make_int2(c.friction_combine_rule, c.restitution_combine_rule);
        groups[k] = make_uint2(c.collision_memberships, c.collision_filter);
    }
    const size_t n = (size_t)count;
    CK(h2d(w.c_shape + first, shape.data(), n * sizeof(int)));
    CK(h2d(w.c_parent + first, parent.data(), n * sizeof(int)));
    CK(h2d(w.c_he + first, he.data(), n * sizeof(float4)));
    CK(h2d(w.c_rel_t + first, rt.data(), n * sizeof(float4)));
    CK(h2d(w.c_rel_q + first, rq.data(), n * sizeof(float4)));
    CK(h2d(w.c_mat + first, mat.data(), n * sizeof(float4)));
    CK(h2d(w.c_rules + first, rules.data(), n * sizeof(int2)));
    CK(h2d(w.c_groups + first, groups.data(), n * sizeof(uint2)));
    CK(h2d(w.c_events + first, events.data(), n * sizeof(int)));
    CK(h2d(w.c_force_thr + first, thr.data(), n * sizeof(float)));
    // per-body collider chains (RigidBodyColliders): appended colliders only ever belong to appended bodies
    // (rb_world_insert), so the chains of the bodies from `first_body` on are rebuilt from the colliders from `first` on
    const int nb_all = (int)W->bodies.size();
    std::vector<int> head(std::max(nb_all - first_body, 0), -1), next(count, -1);
    for (int k = count - 1; k >= 0; --k) {
        const int p = parent[k];
        if (p >= first_body) { next[k] = head[p - first_body]; head[p - first_body] = first + k; }
    }
    CK(h2d(w.c_next + first, next.data(), n * sizeof(int)));
    if (!head.empty()) CK(h2d(w.b_col_head + first_body, head.data(), head.size() * sizeof(int)));
    return RB_OK;
}
// Device tables of the convex polyhedra (rb_poly.cuh): rebuilt whenever hulls were added since the last upload.
// Only worlds that hold a convex collider carry them.
static int upload_hulls(RbWorld* W) {
    bool any = false;
    for (const RbColliderDesc& c : W->colliders) any = any || c.shape == RB_SHAPE_CONVEX;
    if (!any || (W->w.hulls.desc && W->hulls_uploaded == (int)W->hulls.size())) return RB_OK;
    const int nh = (int)W->hulls.size();
    std::vector<int4> desc(nh), desc2(nh), edges;
    std::vector<float4> info(nh), verts, planes;
    std::vector<int2> faces;
    std::vector<int> loops;
    for (int h = 0; h < nh; ++h) {
        const rbhull::Hull& H = W->hulls[h];
        desc[h] = make_int4((int)verts.size(), H.nv(), (int)faces.size(), H.nf());
        desc2[h] = make_int4((int)edges.size(), H.ne(), (int)loops.size(), 0);
        info[h] = make_float4(H.aabb[0], H.aabb[1], H.aabb[2], H.radius);
        for (int i = 0; i < H.nv(); ++i) verts.push_back(make_float4(H.verts[3 * i], H.verts[3 * i + 1], H.verts[3 * i + 2], 0.0f));
        for (int f = 0; f < H.nf(); ++f) {
            planes.push_back(make_float4(H.planes[4 * f], H.planes[4 * f + 1], H.planes[4 * f + 2], H.planes[4 * f + 3]));
            faces.push_back(make_int2(H.face_start[f], H.face_count[f]));
        }
        for (int e = 0; e < H.ne(); ++e) edges.push_back(make_int4(H.edges[4 * e], H.edges[4 * e + 1], H.edges[4 * e + 2], H.edges[4 * e + 3]));
        loops.insert(loops.end(), H.loops.begin(), H.loops.end());
    }
    World& w = W->w;
    int4 *d_desc, *d_desc2, *d_edges;
    float4 *d_info, *d_verts, *d_planes;
    int2* d_faces;
    int* d_loops;
    ALLOC(d_desc, nh); ALLOC(d_desc2, nh); ALLOC(d_info, nh); ALLOC(d_verts, verts.size()); ALLOC(d_planes, planes.size());
    ALLOC(d_faces, faces.size()); ALLOC(d_loops, loops.size()); ALLOC(d_edges, edges.size());
    CK(h2d(d_desc, desc.data(), nh * sizeof(int4))); CK(h2d(d_desc2, desc2.data(), nh * sizeof(int4)));
    CK(h2d(d_info, info.data(), nh * sizeof(float4))); CK(h2d(d_verts, verts.data(), verts.size() * sizeof(float4)));
    CK(h2d(d_planes, planes.data(), planes.size() * sizeof(float4))); CK(h2d(d_faces, faces.data(), faces.size() * sizeof(int2)));
    CK(h2d(d_loops, loops.data(), loops.size() * sizeof(int))); CK(h2d(d_edges, edges.data(), edges.size() * sizeof(int4)));
    w.hulls.desc = d_desc; w.hulls.desc2 = d_desc2; w.hulls.info = d_info; w.hulls.verts = d_verts; w.hulls.planes = d_planes;
    w.hulls.faces = d_faces; w.hulls.loops = d_loops; w.hulls.edges = d_edges;
    if (!w.convex_work) { ALLOC(w.convex_work, w.pair_cap); ALLOC(w.convex_raw, (size_t)w.pair_cap * POLY_RAW_STRIDE); }
    W->hulls_uploaded = nh;
    return RB_OK;
}

static int validate_descs(int nb_total, int nb, const RbBodyDesc* bodies, int nc, const RbColliderDesc* colliders, int nhulls) {
    for (int i = 0; i < nc; ++i) {
        const RbColliderDesc& c = colliders[i];
        const bool capsule_ok = c.shape == RB_SHAPE_CAPSULE && (c.half_extents[2] == 0.0f || c.half_extents[2] == 1.0f || c.half_extents[2] == 2.0f);
        const bool convex_ok = c.shape == RB_SHAPE_CONVEX && c.half_extents[0] >= 0.0f && c.half_extents[0] < (float)nhulls &&
                               c.half_extents[0] == (float)(int)c.half_extents[0] && c.half_extents[1] >= 0.0f;
        if ((c.shape != RB_SHAPE_BALL && c.shape != RB_SHAPE_CUBOID && !capsule_ok && !convex_ok) || c.parent >= nb_total) {
            set_err("collider with unsupported shape, unknown hull or bad parent%s", "");
            return RB_ERR_INVALID;
        }
    }
    for (int i = 0; i < nb; ++i)
        if (bodies[i].body_type < RB_BODY_DYNAMIC || bodies[i].body_type > RB_BODY_KINEMATIC_VELOCITY_BASED) {
            set_err("unknown body type%s", "");
            return RB_ERR_INVALID;
        }
    return RB_OK;
}

extern "C" {

int rb_abi_version(void) { return RB_ABI_VERSION; }
const char* rb_last_error(void) { return g_err; }

void rb_integration_parameters_default(RbIntegrationParameters* p) {
    if (!p) return;
    p->dt = 1.0f / 60.0f;
    p->min_ccd_dt = 1.0f / 60.0f / 100.0f;
    p->contact_natural_frequency = 30.0f;
    p->contact_damping_ratio = 10.0f;
    p->static_contact_natural_frequency = 60.0f;
    p->static_contact_damping_ratio = 10.0f;
    p->warmstart_coefficient = 1.0f;
    p->length_unit = 1.0f;
    p->normalized_allowed_linear_error = 0.005f;
    p->normalized_max_corrective_velocity = 3.0f;
    p->normalized_prediction_distance = 0.02f;
    p->normalized_max_linear_velocity = 400.0f;
    p->num_solver_iterations = 4;
    p->num_internal_pgs_iterations = 1;
    p->num_internal_stabilization_iterations = 1;
    p->max_ccd_substeps = 1;
    p->contact_clustering = 1;
    p->contact_recycling = 1;
    p->normalized_contact_recycle_distance = 0.05f;
    p->friction_in_bias_pass = 0;
    p->warmstart_joints = 0;
    p->friction_model = 0;
}

RbWorld* rb_world_create(const RbIntegrationParameters* params, int device) {
    RbIntegrationParameters defp;
    if (!params) { rb_integration_parameters_default(&defp); params = &defp; }
    if (validate_params(params) != RB_OK) return nullptr;
#if RB_DEVICE_BUILD
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
        set_err("no usable CUDA device (%s, code %d): librapier_b200 has no CPU fallback",
                e == cudaSuccess ? "device ordinal out of range" : cudaGetErrorString(e), (int)e);
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) { set_err("cudaSetDevice failed%s", ""); return nullptr; }
#endif
    RbWorld* W = new RbWorld();
    W->params = *params;
    W->device = device;
    W->hulls.emplace_back();
    rbhull::unit_cube(W->hulls[0]);
#if RB_DEVICE_BUILD
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    W->num_sms = prop.multiProcessorCount;
    if (!prop.cooperativeLaunch) { set_err("device lacks cooperative launch%s", ""); delete W; return nullptr; }
    cudaStreamCreateWithFlags(&W->stream, cudaStreamNonBlocking);
    cudaFuncSetAttribute(k_solve_coop, cudaFuncAttributeMaxDynamicSharedMemorySize, COOP_SMALL_SMEM_BYTES);
    cudaFuncSetAttribute(k_solve_coop_big, cudaFuncAttributeMaxDynamicSharedMemorySize, COOP_BIG_SMEM_BYTES);
    if (cudaHostAlloc((void**)&W->host_hint, 4 * sizeof(int), cudaHostAllocMapped) != cudaSuccess) { set_err("cudaHostAlloc failed%s", ""); delete W; return nullptr; }
    for (int i = 0; i < 4; ++i) W->host_hint[i] = 0;
    cudaFuncSetAttribute(k_collide<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, ITEM_SMEM_BYTES);
    cudaFuncSetAttribute(k_collide<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, ITEM_SMEM_BYTES);
    for (int v = 0; v < 4; ++v)   // every variant: the friction model may change after the world is created
        with_variant(v & 1, v & 2, [](auto fm, auto jm) {
            cudaFuncSetAttribute(k_solve_items_x<decltype(fm)::value, decltype(jm)::value>, cudaFuncAttributeMaxDynamicSharedMemorySize, ITEM_SMEM_BYTES);
        });
    int occ = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_collide<1>, COLLIDE_THREADS, ITEM_SMEM_BYTES);
    if (occ < 1) { set_err("k_collide cannot be resident%s", ""); delete W; return nullptr; }
    W->collide_blocks = W->num_sms;   // one CTA per SM: the cheapest grid barrier that still covers the chip
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_solve_coop, COOP_SMALL_THREADS, COOP_SMALL_SMEM_BYTES);
    if (occ < 1) occ = 1;
    W->coop_blocks = W->num_sms * occ;
    W->coop_blocks_big = W->num_sms;
#else
    {   // emulated CTA: a test override of the shared-memory budget of both launch shapes that forces streaming
        const char* v = getenv("RB_EMU_COOP_SMEM_FLOATS");
        if (v) W->emu_coop_floats = atoi(v);
        W->host_hint = W->emu_hint;
    }
#endif
    {   // debugging override (never needed in production): force the launch shape of k_solve_coop
        const char* v = getenv("RB_COOP_SHAPE");
        W->coop_shape = v ? atoi(v) : -1;
    }
    return W;
}

void rb_world_destroy(RbWorld* W) {
    if (!W) return;
    set_device(W->device);
    stream_sync(W->stream);
    free_all(W);
#if RB_DEVICE_BUILD
    for (cudaEvent_t e : W->prof_ev) cudaEventDestroy(e);
    if (W->stage_host) cudaFreeHost(W->stage_host);
    if (W->host_hint) cudaFreeHost(W->host_hint);
    if (W->stream && W->own_stream) cudaStreamDestroy(W->stream);
#else
    free(W->stage_host);
#endif
    delete W;
}

int rb_world_set_params(RbWorld* W, const RbIntegrationParameters* params) {
    if (!W) { set_err("null world%s", ""); return RB_ERR_INVALID; }
    int rc = validate_params(params);
    if (rc != RB_OK) return rc;
    // joint warm starting runs on the generic joint path, whose row tables are sized when the scene is set
    if (params->warmstart_joints && !W->w.generic_joints && !W->joints.empty()) {
        set_err("warmstart_joints must be enabled before the scene is set%s", "");
        return RB_ERR_INVALID;
    }
    W->params = *params;
    derive_params(W->params, W->w.prm);
    return RB_OK;
}

// ImpulseJointSet -> device: static joint data, greedy colouring in joint order (interaction_groups.rs:59-165), stage order
// (joints.rs:318-392), the body pairs whose contacts a joint disables.  Runs at scene upload and again whenever joints are
// inserted or removed (rb_world_insert_joints / rb_world_remove_joints): everything is recomputed from the host's joint list,
// the warm-start impulses of the surviving joints stay where they are.
static int upload_joints(RbWorld* W) {
    World& w = W->w;
    const int NJ = w.joint_cap, NB = W->body_cap, nj = w.nj;
    const RbJointDesc* joints = W->joints.data();
    const RbBodyDesc* bodies = W->bodies.data();
    W->joint_removed.resize(W->joints.size(), 0);
        std::vector<int4> info(NJ, make_int4(-1, -1, 0, -1));
        std::vector<float4> f1t(NJ), f1q(NJ), f2t(NJ), f2q(NJ);
        std::vector<float2> soft(NJ);
        std::vector<unsigned long long> nocontact;
        struct M128 { unsigned m[4] = {0, 0, 0, 0}; bool test(int c) const { return (m[c >> 5] >> (c & 31)) & 1u; } void set(int c) { m[c >> 5] |= 1u << (c & 31); } };
        std::vector<M128> jm(NB);
        std::vector<int> ccount(NUM_COLORS, 0);
        for (int i = 0; i < nj; ++i) {
            const RbJointDesc& j = joints[i];
            if (W->joint_removed[i]) continue;   // a removed joint keeps its slot: bodies -1 (never selected, no island edge), no colour
            bool d1 = type_moves(bodies[j.body1].body_type), d2 = type_moves(bodies[j.body2].body_type);   // (kinematic bodies conflict like dynamic ones)
            int color = -1;
            if (d1 && d2) {
                color = 128;
                for (int c = 0; c < DYN_COLOR_COUNT; ++c)
                    if (!jm[j.body1].test(c) && !jm[j.body2].test(c)) { color = c; break; }
                if (color < 128) { jm[j.body1].set(color); jm[j.body2].set(color); }
            } else if (d1 || d2) {
                int b = d1 ? j.body1 : j.body2;
                color = 128;
                for (int c = 127; c >= 0; --c)
                    if (!jm[b].test(c)) { color = c; break; }
                if (color < 128) jm[b].set(color);
            }
            if (color >= 0) ccount[color]++;
            info[i] = make_int4(j.body1, j.body2, (int)j.locked_axes, color);
            f1t[i] = make_float4(j.local_frame1_t[0], j.local_frame1_t[1], j.local_frame1_t[2], 0.f);
            f1q[i] = make_float4(j.local_frame1_q[0], j.local_frame1_q[1], j.local_frame1_q[2], j.local_frame1_q[3]);
            f2t[i] = make_float4(j.local_frame2_t[0], j.local_frame2_t[1], j.local_frame2_t[2], 0.f);
            f2q[i] = make_float4(j.local_frame2_q[0], j.local_frame2_q[1], j.local_frame2_q[2], j.local_frame2_q[3]);
            soft[i] = make_float2(j.natural_frequency, j.damping_ratio);
            if (!j.contacts_enabled) {
                unsigned lo = (unsigned)std::min(j.body1, j.body2), hi = (unsigned)std::max(j.body1, j.body2);
                nocontact.push_back(((unsigned long long)lo << 32) | hi);
            }
        }
        std::sort(nocontact.begin(), nocontact.end());
        nocontact.erase(std::unique(nocontact.begin(), nocontact.end()), nocontact.end());
        std::vector<int> jpos(NUM_COLORS + 1, -1);
        int pos = 0;
        for (int pass = 0; pass < 2; ++pass)
            for (int c = 0; c < 128; ++c) {
                if (ccount[c] == 0 || (ccount[c] >= BIG_JCOLOR_MIN) != (pass == 0)) continue;
                jpos[c] = pos++;
            }
        if (ccount[128] > 0) jpos[128] = pos++;
        W->njused = pos;
        CK(h2d(w.j_info, info.data(), NJ * sizeof(int4)));
        CK(h2d(w.j_f1_t, f1t.data(), NJ * sizeof(float4)));
        CK(h2d(w.j_f1_q, f1q.data(), NJ * sizeof(float4)));
        CK(h2d(w.j_f2_t, f2t.data(), NJ * sizeof(float4)));
        CK(h2d(w.j_f2_q, f2q.data(), NJ * sizeof(float4)));
        CK(h2d(w.j_soft, soft.data(), NJ * sizeof(float2)));
        if (w.generic_joints) {
            std::vector<uint2> axes(NJ);
            std::vector<float2> lim((size_t)NJ * 6), mb((size_t)NJ * 6);
            std::vector<float4> ma((size_t)NJ * 6), al((size_t)NJ * 3);
            for (int i = 0; i < nj; ++i) {
                const RbJointDesc& j = joints[i];
                axes[i] = make_uint2((j.limit_axes & 63u) | ((j.coupled_axes & 63u) << 8), j.motor_axes);
                for (int k = 0; k < 6; ++k) {
                    lim[(size_t)i * 6 + k] = make_float2(j.limits[k][0], j.limits[k][1]);
                    ma[(size_t)i * 6 + k] = make_float4(j.motors[k].target_vel, j.motors[k].target_pos, j.motors[k].stiffness, j.motors[k].damping);
                    float model_bits;
                    memcpy(&model_bits, &j.motors[k].model, 4);
                    mb[(size_t)i * 6 + k] = make_float2(j.motors[k].max_force, model_bits);
                }
                for (int k = 0; k < 3; ++k) {   // AngularLimitParams::new (joint_constraint_helper.rs:44-73)
                    const float lo = j.limits[3 + k][0], hi = j.limits[3 + k][1];
                    const float half_range = (hi - lo) * 0.5f;
                    if (half_range >= 3.14159265358979323846f || half_range != half_range) al[(size_t)i * 3 + k] = make_float4(1.0f, 0.0f, 10.0f, 0.0f);
                    else {
                        const float center = (lo + hi) * 0.5f;
                        al[(size_t)i * 3 + k] = make_float4(cosf(center * 0.5f), sinf(center * 0.5f), half_range, 0.0f);
                    }
                }
            }
            CK(h2d(w.j_axes, axes.data(), NJ * sizeof(uint2)));
            CK(h2d(w.j_limits, lim.data(), lim.size() * sizeof(float2)));
            CK(h2d(w.j_motor_a, ma.data(), ma.size() * sizeof(float4)));
            CK(h2d(w.j_motor_b, mb.data(), mb.size() * sizeof(float2)));
            CK(h2d(w.j_anglim, al.data(), al.size() * sizeof(float4)));
        }
        CK(h2d(w.jcolor_pos, jpos.data(), (NUM_COLORS + 1) * sizeof(int)));
        w.n_nocontact = (int)nocontact.size();
        CK(h2d(w.nocontact_keys, nocontact.data(), nocontact.size() * sizeof(unsigned long long)));
    return RB_OK;
}

int rb_world_set_scene(RbWorld* W, int32_t nb, const RbBodyDesc* bodies, int32_t nc, const RbColliderDesc* colliders,
                       int32_t nj, const RbJointDesc* joints) {
    if (!W || nb < 0 || nc < 0 || nj < 0 || (nb && !bodies) || (nc && !colliders) || (nj && !joints)) {
        set_err("invalid scene arguments%s", "");
        return RB_ERR_INVALID;
    }
    CK(set_device(W->device));
    CK(stream_sync(W->stream));
    { int vrc = validate_descs(nb, nb, bodies, nc, colliders, (int)W->hulls.size()); if (vrc != RB_OK) return vrc; }
    for (int i = 0; i < nj; ++i) {
        const RbJointDesc& j = joints[i];
        if (j.body1 < 0 || j.body1 >= nb || j.body2 < 0 || j.body2 >= nb || (j.locked_axes & ~63u)) {
            set_err("joint with bad body index or axes%s", "");
            return RB_ERR_INVALID;
        }
        const unsigned ac = (j.coupled_axes >> 3) & 7u;   // limit_angular_coupled asserts exactly two coupled angular axes (joint_constraint_helper.rs:737-739)
        if ((j.coupled_axes & ~63u) || (ac != 0 && ac != 3u && ac != 5u && ac != 6u)) {
            set_err("joint %s%d: coupled_axes must couple exactly two angular axes (or none)", "", i);
            return RB_ERR_INVALID;
        }
    }
    W->steps_since_scene = 0;
    if (W->host_hint) W->host_hint[0] = W->host_hint[1] = W->host_hint[2] = W->host_hint[3] = 0;
    W->state_buf[0] = W->state_buf[1] = nullptr;
    W->bodies.assign(bodies, bodies + nb);
    W->colliders.assign(colliders, colliders + nc);
    W->joints.assign(joints, joints + nj);
    std::vector<HostMass> mp;
    int rc = host_mass_props(W, mp);
    if (rc != RB_OK) return rc;

    free_all(W);
    World& w = W->w;
    W->force_events = false;
    W->ext_shapes = false;
    W->hulls_uploaded = 0;
    memset(&w, 0, sizeof(w));
    derive_params(W->params, w.prm);
    w.nb = nb; w.nc = nc; w.nj = nj;
    refresh_extra_keys(W);
    int ndyn_col = 0;
    for (int i = 0; i < nc; ++i)
        if (colliders[i].parent >= 0 && type_moves(bodies[colliders[i].parent].body_type)) ndyn_col++;
    // capacities: the scene plus what rb_world_reserve asked for (reserved colliders are assumed to be movers)
    const int NB = std::max(std::max(nb, W->reserve_bodies), 1), NC = std::max(std::max(nc, W->reserve_colliders), 1);
    W->body_cap = NB; W->collider_cap = NC;
    ndyn_col += NC - std::max(nc, 1);
    w.pair_cap = next_pow2_host(std::max(4096, 16 * ndyn_col)) + 160;   // (+160: row strides that are no power of two spread the rows of a record over the L2 slices)
    w.cons_cap = w.pair_cap;
    w.joint_cap = std::max(std::max(nj, W->reserve_joints), 1);
    w.item_cap = 4 + (NB + w.pair_cap + nj) / ITEM_TARGET;
    const int NJ = w.joint_cap;
    w.generic_joints = ((nj > 0 && W->params.warmstart_joints) || W->reserve_generic) ? 1 : 0;   // joint warm starting: generic path too
    for (int i = 0; i < nj; ++i) {   // any limit or motor on a free axis: the generic joint path (12 row slots per joint)
        const unsigned free_axes = ~joints[i].locked_axes & 63u;
        if ((joints[i].limit_axes | joints[i].motor_axes) & free_axes) w.generic_joints = 1;   // (coupled axes only act through a limit or a motor)
    }

    ALLOC(w.st, 1);
    ALLOC(w.b_type, NB); ALLOC(w.b_flags, NB);
    ALLOC(w.b_pos_t, NB); ALLOC(w.b_pos_q, NB); ALLOC(w.b_next_t, NB); ALLOC(w.b_next_q, NB); ALLOC(w.kinpos_list, NB); ALLOC(w.b_linvel, NB); ALLOC(w.b_angvel, NB);
    ALLOC(w.b_lcom_im, NB); ALLOC(w.b_ipi, NB); ALLOC(w.b_pi, NB); ALLOC(w.b_pframe, NB); ALLOC(w.b_misc, NB);
    ALLOC(w.b_uforce, NB); ALLOC(w.b_utorque, NB); ALLOC(w.b_wcom, NB); ALLOC(w.b_eim, NB + 2);
    ALLOC(w.b_eii0, NB); ALLOC(w.b_eii1, NB); ALLOC(w.b_owned, NB);
    ALLOC(w.b_sleeping, NB); ALLOC(w.b_sleep_time, NB); ALLOC(w.b_sleep_prev_t, NB); ALLOC(w.b_sleep_prev_q, NB); ALLOC(w.b_max_extent, NB); ALLOC(w.b_ccd_thick, NB); ALLOC(w.b_col_head, NB); ALLOC(w.c_next, NC);
    ALLOC(w.ccd_list, NB); ALLOC(w.ccd_start_t, NB); ALLOC(w.ccd_start_q, NB);
    ALLOC(w.wake_req, NB); ALLOC(w.isl_block, NB); ALLOC(w.quarantine, NB);
    ALLOC(w.s_lin, NB + 2); ALLOC(w.s_ang, NB + 2); ALLOC(w.s_q, NB + 2); ALLOC(w.s_t, NB + 2);   // + world pseudo body, garbage slot
    ALLOC(w.s_incr_lin, NB); ALLOC(w.s_incr_ang, NB);
    ALLOC(w.state13, (size_t)NB * 13);
    ALLOC(w.c_shape, NC); ALLOC(w.c_parent, NC); ALLOC(w.c_he, NC); ALLOC(w.c_rel_t, NC); ALLOC(w.c_rel_q, NC);
    ALLOC(w.c_mat, NC); ALLOC(w.c_rules, NC); ALLOC(w.c_groups, NC); ALLOC(w.c_events, NC); ALLOC(w.c_force_thr, NC); ALLOC(w.c_pos_t, NC); ALLOC(w.c_pos_q, NC);
    ALLOC(w.c_aabb_min, NC); ALLOC(w.c_aabb_max, NC); ALLOC(w.c_fat_min, NC); ALLOC(w.c_fat_max, NC);
    ALLOC(w.dyn_list, NC); ALLOC(w.wide_list, WIDE_CAP); ALLOC(w.dyn_smin, NC); ALLOC(w.dyn_smax, NC);
    for (int k = 0; k < 2; ++k) { ALLOC(w.dyn_key[k], NC); ALLOC(w.stat_key[k], NC); }
    ALLOC(w.radix_hist, (size_t)9 * 1024 * RADIX);   // (grids of up to 1024 CTAs; the collide grid is one CTA per SM)
    ALLOC(w.cand_key, w.pair_cap); ALLOC(w.cand_key2, w.pair_cap);
    ALLOC(w.remap_src, w.pair_cap);
    w.ev_cap = w.pair_cap;
    ALLOC(w.ev_coll, w.ev_cap); ALLOC(w.ev_force, (size_t)3 * w.ev_cap);
    for (int k = 0; k < 2; ++k) { ALLOC(w.pb[k].key, w.pair_cap); ALLOC(w.pb[k].rows, (size_t)PR_ROWS * w.pair_cap); }
    ALLOC(w.todo, 16);
    ALLOC(w.color_mask, (size_t)NB * 4); ALLOC(w.body_min, NB); ALLOC(w.body_minkey, NB);
    ALLOC(w.isl_label, NB); ALLOC(w.isl_nb, NB); ALLOC(w.isl_ncons, NB); ALLOC(w.isl_item, NB);
    ALLOC(w.scan_tmp, (size_t)1 << 20);
    ALLOC(w.item_body_start, w.item_cap + 2); ALLOC(w.item_cons_start, w.item_cap + 2); ALLOC(w.item_joint_start, w.item_cap + 2);
    ALLOC(w.item_cursor, 3 * (w.item_cap + 2));
    ALLOC(w.item_flags, w.item_cap + 2);
    ALLOC(w.adj_off, NB + 2); ALLOC(w.adj_cnt, NB + 2); ALLOC(w.adj_list, (size_t)2 * w.cons_cap + 2);
    ALLOC(w.item_order, w.item_cap + 2); ALLOC(w.dbg_times, 32); ALLOC(w.order_hist, 2 * ORDER_BUCKETS + 2);
    ALLOC(w.item_bodies, NB); ALLOC(w.body_local, NB); ALLOC(w.body_item, NB);
    ALLOC(w.cons_pair_tmp, w.cons_cap); ALLOC(w.cons_pair, w.cons_cap);
    ALLOC(w.item_color_off, (size_t)(w.item_cap + 1) * (NUM_COLORS + 1));
    ALLOC(w.item_jcolor_off, (size_t)(w.item_cap + 1) * (NUM_COLORS + 1));
    ALLOC(w.color_count, NUM_COLORS + 1); ALLOC(w.color_pos, NUM_COLORS + 1); ALLOC(w.jcolor_pos, NUM_COLORS + 1);
    ALLOC(w.joint_tmp, NJ); ALLOC(w.joint_sched, NJ);
    ALLOC(w.cons_hdr, w.cons_cap); ALLOC(w.cons, (size_t)CR_ROWS * w.cons_cap);
    ALLOC(w.isl_key, NB); ALLOC(w.b_key, NB); ALLOC(w.cons_key, w.cons_cap); ALLOC(w.j_key, NJ);
    ALLOC(w.coop_pool, (size_t)2 * COOP_ROWS * w.cons_cap);
    ALLOC(w.large_pool, (size_t)COOP_ROWS * w.cons_cap); ALLOC(w.large_mut, (size_t)MR_COUNT * w.cons_cap);
    w.host_hint = W->host_hint;
    w.coop_small_floats = COOP_SMALL_SMEM_BYTES / 4;
#ifdef RB_DEBUG
    { const char* v = getenv("RB_DEBUG_FLAGS"); w.debug_flags = v ? atoi(v) : 0; }
#endif
#if !RB_DEVICE_BUILD
    w.coop_small_floats = std::min(w.coop_small_floats, W->emu_coop_floats);   // the emulated CTA must fit what it is given
#endif
    ALLOC(w.j_info, NJ); ALLOC(w.j_f1_t, NJ); ALLOC(w.j_f1_q, NJ); ALLOC(w.j_f2_t, NJ); ALLOC(w.j_f2_q, NJ);
    ALLOC(w.j_soft, NJ); ALLOC(w.j_impulses, (size_t)NJ * 6);
    ALLOC(w.j_rows, (size_t)JR_ROWS * (w.generic_joints ? JROWS_GENERIC : 6) * NJ); ALLOC(w.j_sched_ids, NJ);
    if (w.generic_joints) {
        ALLOC(w.j_axes, NJ); ALLOC(w.j_limits, (size_t)NJ * 6); ALLOC(w.j_motor_a, (size_t)NJ * 6); ALLOC(w.j_motor_b, (size_t)NJ * 6);
        ALLOC(w.j_anglim, (size_t)NJ * 3); ALLOC(w.j_bnd, (size_t)JROWS_GENERIC * NJ);
        ALLOC(w.j_limit_impulses, (size_t)NJ * 6); ALLOC(w.j_motor_impulses, (size_t)NJ * 6);
    }

    // ---- bodies + colliders (unused capacity: fixed bodies / parentless nothing, never listed) ----
    {
        std::vector<int> type(NB, RB_BODY_FIXED);
        std::vector<unsigned char> owned(NB, 1);
        std::vector<int> bmin(NB, 0x7fffffff), parent(NC, -1);
        CK(h2d(w.b_type, type.data(), NB * sizeof(int)));
        CK(h2d(w.b_owned, owned.data(), NB));
        CK(h2d(w.body_min, bmin.data(), NB * sizeof(int)));
        CK(dev_set(w.body_minkey, 0xff, NB * sizeof(unsigned long long)));
        CK(h2d(w.c_parent, parent.data(), NC * sizeof(int)));
        rc = upload_bodies(W, mp, 0, nb);
        if (rc != RB_OK) return rc;
        rc = upload_hulls(W);
        if (rc != RB_OK) return rc;
        rc = upload_colliders(W, 0, nc);
        if (rc != RB_OK) return rc;
    }
    // ---- joints ----
    ALLOC(w.nocontact_keys, (size_t)NJ);
    W->joint_removed.assign(W->joints.size(), 0);
    rc = upload_joints(W);
    if (rc != RB_OK) return rc;
    {
        State s;
        memset(&s, 0, sizeof(s));
        s.bp_dirty = 1;
        s.lists_dirty = 3;
        s.sched_dirty = 1;
        s.nitems = 1;
        s.njused_colors = W->njused;
        CK(h2d(w.st, &s, sizeof(s)));
        std::vector<int> cp(NUM_COLORS + 1, -1);
        CK(h2d(w.color_pos, cp.data(), cp.size() * sizeof(int)));
    }
    ALLOC(W->stage_dev, (size_t)NB * 13);
    ALLOC(W->ident_dev, NB);
    {
        std::vector<int> id(NB);
        for (int i = 0; i < NB; ++i) id[i] = i;
        CK(h2d(W->ident_dev, id.data(), NB * sizeof(int)));
    }
#if RB_DEVICE_BUILD
    if (W->stage_host) { cudaFreeHost(W->stage_host); W->stage_host = nullptr; }
    CK(cudaMallocHost((void**)&W->stage_host, (size_t)NB * 26 * sizeof(float)));
#else
    free(W->stage_host);
    W->stage_host = (float*)calloc((size_t)NB * 26, sizeof(float));
#endif
    W->steps = 0;
    rc = launch_init_bodies(W);
    if (rc != RB_OK) return rc;
    return sync_world(W);
}

// ---- incremental changes of the sets (src/pipeline/user_changes.rs:11-46, substep.rs:303-334) ----
// Room for later rb_world_insert calls; takes effect at the next rb_world_set_scene.
int rb_world_reserve(RbWorld* W, int32_t max_bodies, int32_t max_colliders) {
    if (!W || max_bodies < 0 || max_colliders < 0) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    W->reserve_bodies = max_bodies;
    W->reserve_colliders = max_colliders;
    return RB_OK;
}

int rb_world_reserve_joints(RbWorld* W, int32_t max_joints, int32_t generic) {
    if (!W || max_joints < 0) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    W->reserve_joints = max_joints;
    W->reserve_generic = generic ? 1 : 0;
    return RB_OK;
}

static int validate_joint(const RbJointDesc& j, int nb, int index) {
    if (j.body1 < 0 || j.body1 >= nb || j.body2 < 0 || j.body2 >= nb || (j.locked_axes & ~63u)) {
        set_err("joint with bad body index or axes%s", "");
        return RB_ERR_INVALID;
    }
    const unsigned ac = (j.coupled_axes >> 3) & 7u;   // limit_angular_coupled asserts exactly two coupled angular axes (joint_constraint_helper.rs:737-739)
    if ((j.coupled_axes & ~63u) || (ac != 0 && ac != 3u && ac != 5u && ac != 6u)) {
        set_err("joint %s%d: coupled_axes must couple exactly two angular axes (or none)", "", index);
        return RB_ERR_INVALID;
    }
    return RB_OK;
}

// The joint set changed: colours, stage order and the contact-disabling pairs were recomputed (upload_joints); the islands and
// the schedule follow at the next step, the broad phase re-filters its pairs.
static int joints_changed(RbWorld* W) {
    int one = 1;
    CK(h2d(&W->w.st->bp_dirty, &one, sizeof(int)));
    CK(h2d(&W->w.st->sched_dirty, &one, sizeof(int)));
    CK(h2d(&W->w.st->njused_colors, &W->njused, sizeof(int)));
    return RB_OK;
}

// ImpulseJointSet::insert after the world has been uploaded (impulse_joint_set.rs; user_changes.rs): appended joints keep every
// existing index.  Capacity comes from rb_world_reserve_joints (before rb_world_set_scene); joints with limits, motors or coupled
// axes -- and any joint under warmstart_joints -- need the generic joint path, which a world without such joints only has when
// it was reserved with generic = 1.
int rb_world_insert_joints(RbWorld* W, int32_t n, const RbJointDesc* joints, int32_t* first_joint) {
    if (!W || n < 0 || (n && !joints) || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    const int nj0 = W->w.nj;
    if (nj0 + n > W->w.joint_cap) { set_err("rb_world_insert_joints exceeds the reserved capacity (rb_world_reserve_joints before rb_world_set_scene)%s", ""); return RB_ERR_CAPACITY; }
    for (int i = 0; i < n; ++i) {
        int rc = validate_joint(joints[i], W->w.nb, nj0 + i);
        if (rc != RB_OK) return rc;
        const unsigned free_axes = ~joints[i].locked_axes & 63u;
        if ((((joints[i].limit_axes | joints[i].motor_axes) & free_axes) || W->params.warmstart_joints) && !W->w.generic_joints) {
            set_err("this joint needs the generic joint path: reserve it with rb_world_reserve_joints(.., generic = 1)%s", "");
            return RB_ERR_INVALID;
        }
    }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    W->joints.insert(W->joints.end(), joints, joints + n);
    W->w.nj = nj0 + n;
    if ((rc = upload_joints(W)) != RB_OK) return rc;
    if (first_joint) *first_joint = nj0;
    if ((rc = joints_changed(W)) != RB_OK) return rc;
    // insert(.., wake_up = true): the attached bodies' islands are woken -- an island is awake or asleep as a whole here, and a
    // joint between a sleeping and an awake body would otherwise merge the two states into one island
    std::vector<int32_t> wake;
    for (int i = 0; i < n; ++i) { wake.push_back(joints[i].body1); wake.push_back(joints[i].body2); }
    return wake.empty() ? RB_OK : wake_impl(W, wake.data(), (int)wake.size());
}

// ImpulseJointSet::remove: the slot stays allocated (indices of the other joints are unchanged), the joint is neither solved
// nor an island edge any more, and contacts it disabled come back.
int rb_world_remove_joints(RbWorld* W, int32_t n, const int32_t* indices) {
    if (!W || n < 0 || (n && !indices) || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    for (int k = 0; k < n; ++k)
        if (indices[k] < 0 || indices[k] >= W->w.nj) { set_err("joint index out of range%s", ""); return RB_ERR_INVALID; }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    W->joint_removed.resize(W->joints.size(), 0);
    for (int k = 0; k < n; ++k) W->joint_removed[indices[k]] = 1;
    if ((rc = upload_joints(W)) != RB_OK) return rc;
    return joints_changed(W);
}

// Registers a convex polyhedron (closed convex mesh: vertices + polygonal faces) that RB_SHAPE_CONVEX colliders refer to
// by the id returned (>= 1; 0 is the unit cube).  Negative = RB_ERR_*.  Hulls persist across rb_world_set_scene.
int32_t rb_world_add_hull(RbWorld* W, int32_t nv, const float* verts, int32_t nf, const int32_t* face_sizes, const int32_t* face_indices) {
    if (!W || !verts || !face_sizes || !face_indices) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    rbhull::Hull h;
    const char* why = rbhull::from_mesh(nv, verts, nf, face_sizes, face_indices, h);
    if (why) { set_err("convex mesh rejected: %s", why); return RB_ERR_INVALID; }
    W->hulls.push_back(h);
    return (int32_t)W->hulls.size() - 1;
}

// ColliderBuilder::convex_hull's hull computation (parry transformation::convex_hull) for at most 32 points: writes the
// hull's vertices (a subset of the points, in input order), face sizes and face vertex indices.  Host code only.
int32_t rb_convex_hull(int32_t npoints, const float* points, int32_t* nv, float* verts, int32_t* nf, int32_t* face_sizes, int32_t* face_indices) {
    if (!points || !nv || !verts || !nf || !face_sizes || !face_indices) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    std::vector<float> v;
    std::vector<int32_t> sizes, idx;
    const char* why = rbhull::convex_hull(npoints, points, v, sizes, idx);
    if (why) { set_err("convex hull failed: %s", why); return RB_ERR_INVALID; }
    *nv = (int32_t)v.size() / 3; *nf = (int32_t)sizes.size();
    memcpy(verts, v.data(), v.size() * sizeof(float));
    memcpy(face_sizes, sizes.data(), sizes.size() * sizeof(int32_t));
    memcpy(face_indices, idx.data(), idx.size() * sizeof(int32_t));
    return RB_OK;
}

// Appends bodies and colliders to the world (RigidBodySet::insert / ColliderSet::insert_with_parent): indices of
// existing bodies, colliders and contact pairs do not change, so warm-start data, colours and islands persist.
// New colliders may only be attached to the new bodies (or to none).  Joints cannot be inserted this way.
int rb_world_insert(RbWorld* W, int32_t nb, const RbBodyDesc* bodies, int32_t nc, const RbColliderDesc* colliders,
                    int32_t* first_body, int32_t* first_collider) {
    if (!W || nb < 0 || nc < 0 || (nb && !bodies) || (nc && !colliders) || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    const int nb0 = W->w.nb, nc0 = W->w.nc;
    if (nb0 + nb > W->body_cap || nc0 + nc > W->collider_cap) {
        set_err("rb_world_insert exceeds the reserved capacity (rb_world_reserve before rb_world_set_scene)%s", "");
        return RB_ERR_CAPACITY;
    }
    int rc = validate_descs(nb0 + nb, nb, bodies, nc, colliders, (int)W->hulls.size());
    if (rc != RB_OK) return rc;
    for (int i = 0; i < nc; ++i)
        if (colliders[i].parent >= 0 && colliders[i].parent < nb0) { set_err("new colliders may only be attached to new bodies%s", ""); return RB_ERR_INVALID; }
    rc = sync_world(W);
    if (rc != RB_OK) return rc;
    W->bodies.insert(W->bodies.end(), bodies, bodies + nb);
    W->colliders.insert(W->colliders.end(), colliders, colliders + nc);
    std::vector<HostMass> mp;
    rc = host_mass_props(W, mp, nb0, nc0);
    if (rc != RB_OK) { W->bodies.resize(nb0); W->colliders.resize(nc0); return rc; }
    W->w.nb = nb0 + nb;
    W->w.nc = nc0 + nc;
    refresh_extra_keys(W);
    if ((rc = upload_hulls(W)) != RB_OK) return rc;
    if ((rc = upload_bodies(W, mp, nb0, nb)) != RB_OK) return rc;
    if ((rc = upload_colliders(W, nc0, nc, nb0)) != RB_OK) return rc;
    int one = 1, lists = 1;   // lists: 1 = only movers were added, 3 = static colliders too (re-sort them)
    for (int i = 0; i < nc; ++i)
        if (colliders[i].parent < 0 || !type_moves(W->bodies[colliders[i].parent].body_type)) lists = 3;
    CK(h2d(&W->w.st->lists_dirty, &lists, sizeof(int)));
    CK(h2d(&W->w.st->bp_dirty, &one, sizeof(int)));
    CK(h2d(&W->w.st->sched_dirty, &one, sizeof(int)));
    if (first_body) *first_body = nb0;
    if (first_collider) *first_collider = nc0;
    rc = launch_init_bodies(W, nb0);
    if (rc != RB_OK) return rc;
    return sync_world(W);
}

// Removes bodies with their colliders (RigidBodySet::remove with remove_attached_colliders): the slots stay
// allocated (indices of everything else are unchanged), the colliders leave the broad phase, so their contact
// pairs end at the next step.
int rb_world_remove_bodies(RbWorld* W, int32_t n, const int32_t* indices) {
    if (!W || n < 0 || (n && !indices) || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    for (int k = 0; k < n; ++k)
        if (indices[k] < 0 || indices[k] >= W->w.nb) { set_err("body index out of range%s", ""); return RB_ERR_INVALID; }
    const int removed_type = BODY_REMOVED, removed_shape = SHAPE_REMOVED;
    for (int k = 0; k < n; ++k) {
        const int b = indices[k];
        W->bodies[b].body_type = BODY_REMOVED;
        CK(h2d(W->w.b_type + b, &removed_type, sizeof(int)));
        for (int c = 0; c < (int)W->colliders.size(); ++c)
            if (W->colliders[c].parent == b) CK(h2d(W->w.c_shape + c, &removed_shape, sizeof(int)));
    }
    int one = 1, lists = 3;
    CK(h2d(&W->w.st->lists_dirty, &lists, sizeof(int)));
    CK(h2d(&W->w.st->bp_dirty, &one, sizeof(int)));
    CK(h2d(&W->w.st->sched_dirty, &one, sizeof(int)));
    return wake_impl(W, nullptr, 0);   // (the reference wakes what touched the removed body; here: everything asleep)
}

// Quarantine::bodies (quarantine.rs:34-37): bodies disabled because their state went non-finite since the last call.
int rb_world_get_quarantine(RbWorld* W, int32_t* bodies, int32_t cap) {
    if (!W || !W->w.st) return RB_ERR_INVALID;
    State st;
    int rc = read_state(W, st);
    if (rc != RB_OK) return rc;
    const int n = std::min(st.nquarantine, W->w.nb);
    if (bodies && cap > 0 && n > 0) {
        std::vector<int> q(n);
        CK(d2h(q.data(), W->w.quarantine, (size_t)n * sizeof(int)));
        std::sort(q.begin(), q.end());
        for (int i = 0; i < n && i < cap; ++i) {
            bodies[i] = q[i];
            if (q[i] >= 0 && q[i] < (int)W->bodies.size()) W->bodies[q[i]].body_type = BODY_REMOVED;
        }
        int zero = 0;
        CK(h2d(&W->w.st->nquarantine, &zero, sizeof(int)));
    }
    return n;
}

int rb_world_get_sleeping(RbWorld* W, uint8_t* sleeping) {
    if (!W || !sleeping || !W->w.st) return RB_ERR_INVALID;
    int rc = sync_world(W, false);
    if (rc != RB_OK) return rc;
    CK(d2h(sleeping, W->w.b_sleeping, (size_t)W->w.nb));
    return RB_OK;
}

static int wake_impl(RbWorld* W, const int32_t* indices_host, int n) {
    int* idx_dev = nullptr;
    if (indices_host) {
        if (dev_alloc((void**)&idx_dev, (size_t)std::max(n, 1) * sizeof(int)) != cudaSuccess) { set_err("device allocation failed%s", ""); return RB_ERR_CUDA; }
        CK(h2d(idx_dev, indices_host, (size_t)n * sizeof(int)));
    }
    CK(set_device(W->device));
    const int work = indices_host ? n : W->w.nb;
    CK(launch(W, k_wake, (std::max(work, 1) + 255) / 256, 256, 0, false, W->w, idx_dev, n));
    if (indices_host) CK(launch(W, k_wake_apply, (std::max(W->w.nb, 1) + 255) / 256, 256, 0, false, W->w));
    CK(stream_sync(W->stream));
    if (idx_dev) dev_free(idx_dev);
    return RB_OK;
}
// RigidBody::wake_up(strong = true) through IslandManager::wake_up: the bodies' whole islands.
int rb_world_wake_up(RbWorld* W, int32_t n, const int32_t* indices) {
    if (!W || n < 0 || (n && !indices) || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    if (n == 0) return RB_OK;
    return wake_impl(W, indices, n);
}

// ImpulseJointSet::get_mut(handle, wake_up) followed by edits of the joint (motor targets, limits, frames, softness ...): the
// listed joints take the new descriptors in place.  Their bodies must stay the same (otherwise remove + insert); impulses carried
// for warm starting are kept; with wake_up the islands of the attached bodies are woken (issue_692_joint_get_mut_wakes_bodies.rs).
int rb_world_update_joints(RbWorld* W, int32_t n, const int32_t* indices, const RbJointDesc* joints, int32_t wake_up) {
    if (!W || n < 0 || (n && (!indices || !joints)) || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    W->joint_removed.resize(W->joints.size(), 0);
    for (int k = 0; k < n; ++k) {
        const int i = indices[k];
        if (i < 0 || i >= W->w.nj || W->joint_removed[i]) { set_err("joint index out of range (or removed)%s", ""); return RB_ERR_INVALID; }
        int rc = validate_joint(joints[k], W->w.nb, i);
        if (rc != RB_OK) return rc;
        if (joints[k].body1 != W->joints[i].body1 || joints[k].body2 != W->joints[i].body2) {
            set_err("rb_world_update_joints cannot move a joint to other bodies: remove it and insert a new one%s", "");
            return RB_ERR_INVALID;
        }
        const unsigned free_axes = ~joints[k].locked_axes & 63u;
        if (((joints[k].limit_axes | joints[k].motor_axes) & free_axes) && !W->w.generic_joints) {
            set_err("this joint needs the generic joint path: reserve it with rb_world_reserve_joints(.., generic = 1)%s", "");
            return RB_ERR_INVALID;
        }
    }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    std::vector<int32_t> wake;
    for (int k = 0; k < n; ++k) {
        W->joints[indices[k]] = joints[k];
        wake.push_back(joints[k].body1);
        wake.push_back(joints[k].body2);
    }
    if ((rc = upload_joints(W)) != RB_OK) return rc;
    if ((rc = joints_changed(W)) != RB_OK) return rc;
    if (wake_up && !wake.empty()) return wake_impl(W, wake.data(), (int)wake.size());
    return RB_OK;
}

int rb_world_set_body_states(RbWorld* W, int32_t n, const int32_t* indices, const float* pose7, const float* vel6) {
    if (!W || n < 0 || (n && !indices)) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    for (int k = 0; k < n; ++k) {
        int i = indices[k];
        if (i < 0 || i >= W->w.nb) { set_err("body index out of range%s", ""); return RB_ERR_INVALID; }
        if (pose7) {
            float4 t = make_float4(pose7[k * 7], pose7[k * 7 + 1], pose7[k * 7 + 2], 0.f);
            float4 q = make_float4(pose7[k * 7 + 3], pose7[k * 7 + 4], pose7[k * 7 + 5], pose7[k * 7 + 6]);
            CK(h2d(W->w.b_pos_t + i, &t, sizeof(t)));
            CK(h2d(W->w.b_pos_q + i, &q, sizeof(q)));
            CK(h2d(W->w.b_next_t + i, &t, sizeof(t)));
            CK(h2d(W->w.b_next_q + i, &q, sizeof(q)));
        }
        if (vel6) {
            float4 l = make_float4(vel6[k * 6], vel6[k * 6 + 1], vel6[k * 6 + 2], 0.f);
            float4 a = make_float4(vel6[k * 6 + 3], vel6[k * 6 + 4], vel6[k * 6 + 5], 0.f);
            CK(h2d(W->w.b_linvel + i, &l, sizeof(l)));
            CK(h2d(W->w.b_angvel + i, &a, sizeof(a)));
        }
    }
    {   // a teleported FIXED body moves static colliders: rebuild the broad-phase lists (and re-sort the static ones)
        bool moved_static = false;
        if (pose7)
            for (int k = 0; k < n; ++k) moved_static = moved_static || !type_moves(W->bodies[indices[k]].body_type);
        if (moved_static) {
            int one = 1, lists = 3;
            CK(h2d(&W->w.st->lists_dirty, &lists, sizeof(int)));
            CK(h2d(&W->w.st->bp_dirty, &one, sizeof(int)));
        }
    }
    rc = launch_init_bodies(W);
    if (rc != RB_OK) return rc;
    if (n > 0 && (rc = wake_impl(W, indices, n)) != RB_OK) return rc;   // a user change wakes the body's island (user_changes.rs)
    return sync_world(W);
}

int rb_world_set_body_forces(RbWorld* W, int32_t n, const int32_t* indices, const float* force3, const float* torque3) {
    if (!W || n < 0 || (n && !indices)) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    for (int k = 0; k < n; ++k) {
        const int i = indices[k];
        if (i < 0 || i >= W->w.nb) { set_err("body index out of range%s", ""); return RB_ERR_INVALID; }
        if (force3) {
            float4 f = make_float4(force3[k * 3], force3[k * 3 + 1], force3[k * 3 + 2], 0.f);
            CK(h2d(W->w.b_uforce + i, &f, sizeof(f)));
            for (int a = 0; a < 3; ++a) W->bodies[i].user_force[a] = force3[k * 3 + a];
        }
        if (torque3) {
            float4 t = make_float4(torque3[k * 3], torque3[k * 3 + 1], torque3[k * 3 + 2], 0.f);
            CK(h2d(W->w.b_utorque + i, &t, sizeof(t)));
            for (int a = 0; a < 3; ++a) W->bodies[i].user_torque[a] = torque3[k * 3 + a];
        }
    }
    if (n > 0 && (rc = wake_impl(W, indices, n)) != RB_OK) return rc;   // add_force(.., wake_up = true)
    return sync_world(W);
}

int rb_world_set_next_kinematic_positions(RbWorld* W, int32_t n, const int32_t* indices, const float* pose7) {
    if (!W || n < 0 || (n && (!indices || !pose7))) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    for (int k = 0; k < n; ++k) {
        const int i = indices[k];
        if (i < 0 || i >= W->w.nb || W->bodies[i].body_type != RB_BODY_KINEMATIC_POSITION_BASED) {
            set_err("rb_world_set_next_kinematic_positions: not a position-based kinematic body%s", "");
            return RB_ERR_INVALID;
        }
        float4 t = make_float4(pose7[k * 7], pose7[k * 7 + 1], pose7[k * 7 + 2], 0.f);
        float4 q = make_float4(pose7[k * 7 + 3], pose7[k * 7 + 4], pose7[k * 7 + 5], pose7[k * 7 + 6]);
        CK(h2d(W->w.b_next_t + i, &t, sizeof(t)));
        CK(h2d(W->w.b_next_q + i, &q, sizeof(q)));
    }
    if (n > 0 && (rc = wake_impl(W, indices, n)) != RB_OK) return rc;
    return sync_world(W);
}

int rb_world_drain_collision_events(RbWorld* W, int32_t cap, RbCollisionEvent* out) {
    if (!W || cap < 0 || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    State st;
    int rc = read_state(W, st);
    if (rc != RB_OK) return rc;
    const int n = std::min(st.nev_coll, W->w.ev_cap);
    std::vector<int4> ev(std::max(n, 1));
    CK(d2h(ev.data(), W->w.ev_coll, (size_t)n * sizeof(int4)));
    std::sort(ev.begin(), ev.begin() + n, [](const int4& a, const int4& b) {
        if (a.w != b.w) return a.w < b.w;
        if (a.x != b.x) return a.x < b.x;
        if (a.y != b.y) return a.y < b.y;
        return a.z < b.z;
    });
    auto is_sensor = [&](int c) { return c >= 0 && c < (int)W->colliders.size() && W->colliders[c].sensor != 0; };
    for (int i = 0; i < n && i < cap && out; ++i)
        out[i] = RbCollisionEvent{ev[i].x, ev[i].y, ev[i].z, ev[i].w, (is_sensor(ev[i].x) || is_sensor(ev[i].y)) ? RB_COLLISION_EVENT_SENSOR : 0};
    int zero = 0;
    CK(h2d(&W->w.st->nev_coll, &zero, sizeof(int)));
    return n;
}

int rb_world_drain_contact_force_events(RbWorld* W, int32_t cap, RbContactForceEvent* out) {
    if (!W || cap < 0 || !W->w.st) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    State st;
    int rc = read_state(W, st);
    if (rc != RB_OK) return rc;
    const int n = std::min(st.nev_force, W->w.ev_cap), ec = W->w.ev_cap;
    std::vector<float4> r0(std::max(n, 1)), r1(std::max(n, 1)), r2(std::max(n, 1));
    CK(d2h(r0.data(), W->w.ev_force, (size_t)n * sizeof(float4)));
    CK(d2h(r1.data(), W->w.ev_force + ec, (size_t)n * sizeof(float4)));
    CK(d2h(r2.data(), W->w.ev_force + 2 * (size_t)ec, (size_t)n * sizeof(float4)));
    std::vector<RbContactForceEvent> ev(n);
    for (int i = 0; i < n; ++i) {
        RbContactForceEvent& e = ev[i];
        memcpy(&e.collider1, &r0[i].x, 4); memcpy(&e.collider2, &r0[i].y, 4); memcpy(&e.started, &r0[i].z, 4); memcpy(&e.step, &r0[i].w, 4);
        e.total_force[0] = r1[i].x; e.total_force[1] = r1[i].y; e.total_force[2] = r1[i].z; e.total_force_magnitude = r1[i].w;
        e.max_force_direction[0] = r2[i].x; e.max_force_direction[1] = r2[i].y; e.max_force_direction[2] = r2[i].z; e.max_force_magnitude = r2[i].w;
    }
    std::sort(ev.begin(), ev.end(), [](const RbContactForceEvent& a, const RbContactForceEvent& b) {
        if (a.step != b.step) return a.step < b.step;
        if (a.collider1 != b.collider1) return a.collider1 < b.collider1;
        return a.collider2 < b.collider2;
    });
    for (int i = 0; i < n && i < cap && out; ++i) out[i] = ev[i];
    int zero = 0;
    CK(h2d(&W->w.st->nev_force, &zero, sizeof(int)));
    return n;
}

int rb_world_step(RbWorld* W, const float gravity[3], int32_t nsteps, int32_t sync) {
    if (!W || !gravity || nsteps < 0) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    if (W->w.nb == 0 && W->w.nc == 0) return RB_OK;
    Grav g{gravity[0], gravity[1], gravity[2]};
    CK(set_device(W->device));
#if RB_DEVICE_BUILD
    if (W->profiling) {
        while ((int)W->prof_ev.size() < 3 * nsteps) { cudaEvent_t e; CK(cudaEventCreate(&e)); W->prof_ev.push_back(e); }
        W->prof_steps = nsteps;
    }
    // event i of step s: 0 before k_collide, 1 after it, 2 after the solves
    auto mark = [&](int s, int i) { return W->profiling ? cudaEventRecord(W->prof_ev[3 * s + i], W->stream) : cudaSuccess; };
#else
    auto mark = [](int, int) { return cudaSuccess; };
#endif
    for (int s = 0; s < nsteps; ++s) {
        CK(mark(s, 0));
        // a grid-wide island existed after the last schedule the host knows of: it gets its own launch
        const bool general = general_path(W->w);
        const bool large = *(volatile int*)(W->host_hint + 2) != 0;
        const int do_solve = general ? 0 : (large ? 3 : 1);
        if (W->state_buf[1]) { W->w.state13 = W->state_buf[W->state_next]; W->state_next ^= 1; }
        // A new scene's islands are only known after its first schedule.  A caller that enqueues many steps in
        // one asynchronous call would otherwise run all of them in the launch shape chosen before that, so the
        // first call after a scene upload waits ONCE, after its second step, for the device hint.
        if (W->steps_since_scene == 2 && nsteps > 3) CK(stream_sync(W->stream));
        W->steps_since_scene++;
        // launch shape of k_solve_coop for this step (both kernels must agree on it): device hint of the last step
        const bool big = W->coop_shape >= 0 ? W->coop_shape == 1 : (*(volatile int*)W->host_hint != 0);
        W->w.step_index = (int)(W->steps + s + 1);
        CK(launch(W, W->ext_shapes ? k_collide<1> : k_collide<0>, W->collide_blocks, COLLIDE_THREADS, ITEM_SMEM_BYTES, true, W->w, g, do_solve));
        CK(mark(s, 1));
        if (general) {   // every item through the streaming solve; the grid-wide item's kernel returns at once when there is none
            // substep solve-groups: one pass of both kernels per distinct key, each with the parameters of its cadence
            const size_t npass = W->w.any_extra ? W->extra_keys.size() : 1;
            for (size_t ki = 0; ki < npass; ++ki) {
                if (W->w.any_extra) {
                    W->w.pass_key = W->extra_keys[ki];
                    derive_params(W->params, W->w.prm, W->w.pass_key);
                    if (ki > 0) CK(memset_async(&W->w.st->cursor_rest, 0, sizeof(int), W->stream));
                }
                CK(with_variant(W->w, [&](auto fm, auto jm) {
                    constexpr int FM = decltype(fm)::value, JM = decltype(jm)::value;
                    const cudaError_t e = launch(W, k_solve_items_x<FM, JM>, W->collide_blocks, COLLIDE_THREADS, ITEM_SMEM_BYTES, false, W->w, g);
                    return e != cudaSuccess ? e : launch(W, k_solve_large_x<FM, JM>, W->collide_blocks, COLLIDE_THREADS, 0, true, W->w, g);
                }));
            }
            if (W->w.any_extra) { W->w.pass_key = 0; derive_params(W->params, W->w.prm); }
        } else {
            if (large) CK(launch(W, k_solve_large, W->collide_blocks, COLLIDE_THREADS, 0, true, W->w, g));
            if (big) CK(launch(W, k_solve_coop_big, W->coop_blocks_big, COOP_BIG_THREADS, COOP_BIG_SMEM_BYTES, false, W->w, g));
            else CK(launch(W, k_solve_coop, W->coop_blocks, COOP_SMALL_THREADS, COOP_SMALL_SMEM_BYTES, false, W->w, g));
        }
        if (W->force_events) CK(launch(W, k_force_events, W->collide_blocks, 256, 0, false, W->w));
        CK(mark(s, 2));
    }
    W->steps += nsteps;
    if (!sync) return RB_OK;
    CK(stream_sync(W->stream));
#if RB_DEVICE_BUILD
    if (W->profiling && nsteps > 0) {  // mean per-step device time of each launch group over this call
        float c = 0.f, v = 0.f;
        for (int s = 0; s < W->prof_steps; ++s) {
            float a = 0.f, b = 0.f;
            cudaEventElapsedTime(&a, W->prof_ev[3 * s], W->prof_ev[3 * s + 1]);
            cudaEventElapsedTime(&b, W->prof_ev[3 * s + 1], W->prof_ev[3 * s + 2]);
            c += a; v += b;
        }
        W->ms_collide = c / W->prof_steps;
        W->ms_solve = v / W->prof_steps;
        W->ms_step = W->ms_collide + W->ms_solve;
    }
#endif
    return sync_world(W);
}

int rb_world_synchronize(RbWorld* W) {
    if (!W) return RB_ERR_INVALID;
    return sync_world(W);
}

int rb_world_num_bodies(RbWorld* W) { return W ? W->w.nb : RB_ERR_INVALID; }

int rb_world_get_body_states(RbWorld* W, float* pose7, float* vel6) {
    if (!W) return RB_ERR_INVALID;
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    int nb = W->w.nb;
    std::vector<float> s((size_t)nb * 13);
    CK(d2h(s.data(), W->w.state13, s.size() * sizeof(float)));
    for (int i = 0; i < nb; ++i) {
        if (pose7) memcpy(pose7 + (size_t)i * 7, &s[(size_t)i * 13], 7 * sizeof(float));
        if (vel6) memcpy(vel6 + (size_t)i * 6, &s[(size_t)i * 13 + 7], 6 * sizeof(float));
    }
    return RB_OK;
}

int rb_world_enable_profiling(RbWorld* W, int32_t enabled) {
    if (!W) return RB_ERR_INVALID;
    W->profiling = enabled != 0;
    return RB_OK;
}

int rb_world_get_counters(RbWorld* W, RbCounters* out) {
    if (!W || !out) return RB_ERR_INVALID;
    State st;
    int rc = read_state(W, st);
    if (rc != RB_OK) return rc;
    memset(out, 0, sizeof(*out));
    out->step_ms = W->ms_step;
    out->collision_detection_ms = W->ms_collide;
    out->solver_ms = W->ms_solve;
    out->num_bodies = W->w.nb;
    out->num_colliders = W->w.nc;
    out->num_joints = W->w.nj;
    out->num_pairs = st.npairs;
    out->num_active_manifolds = st.ncons;
    out->num_islands = st.nitems;
    out->num_colors = st.nused_colors;
    out->broad_phase_ran = st.bp_ran;
    out->schedule_rebuilt = st.sched_ran;
    out->kernels_launched = W->kernels;
    out->steps = W->steps;
    return RB_OK;
}

static int fetch_rows(RbWorld* W, const State& st, int row, int count, std::vector<float4>& out) {
    out.resize((size_t)count * std::max(st.npairs, 1));
    for (int r = 0; r < count; ++r)
        CK(d2h(out.data() + (size_t)r * st.npairs, W->w.pb[st.cur].rows + (size_t)(row + r) * W->w.pair_cap, (size_t)st.npairs * sizeof(float4)));
    return RB_OK;
}

int rb_world_get_contact_pairs(RbWorld* W, int32_t cap, int32_t* pair_colliders, int32_t* num_contacts, int32_t* color,
                               float* normal, float* impulses) {
    if (!W) return RB_ERR_INVALID;
    State st;
    int rc = read_state(W, st);
    if (rc != RB_OK) return rc;
    int n = st.npairs;
    if (cap <= 0 || n == 0) return n;
    std::vector<unsigned long long> keys(n);
    CK(d2h(keys.data(), W->w.pb[st.cur].key, (size_t)n * 8));
    std::vector<float4> info, nrm, pd, a1;
    if ((rc = fetch_rows(W, st, PR_INFO, 1, info)) != RB_OK) return rc;
    if ((rc = fetch_rows(W, st, PR_NORMAL, 1, nrm)) != RB_OK) return rc;
    if ((rc = fetch_rows(W, st, PR_PD, MAX_PTS, pd)) != RB_OK) return rc;
    if ((rc = fetch_rows(W, st, PR_A1, MAX_PTS, a1)) != RB_OK) return rc;
    for (int i = 0; i < n && i < cap; ++i) {
        int nsc, col;
        memcpy(&nsc, &info[i].z, 4);
        memcpy(&col, &info[i].w, 4);
        if (pair_colliders) { pair_colliders[2 * i] = (int)(keys[i] >> 32); pair_colliders[2 * i + 1] = (int)(keys[i] & 0xffffffffu); }
        if (num_contacts) num_contacts[i] = nsc;
        if (color) color[i] = col;
        if (normal) { normal[3 * i] = nrm[i].x; normal[3 * i + 1] = nrm[i].y; normal[3 * i + 2] = nrm[i].z; }
        if (impulses)
            for (int k = 0; k < 4; ++k) {
                float v = 0.0f;
                if (k < nsc) {
                    int cid;
                    memcpy(&cid, &a1[(size_t)k * n + i].w, 4);
                    v = pd[(size_t)cid * n + i].x;
                }
                impulses[4 * i + k] = v;
            }
    }
    return n;
}

int64_t rb_world_debug_read(RbWorld* W, const char* table, void* dst, int64_t cap) {
    if (!W || !table) return RB_ERR_INVALID;
    State st;
    int rc = read_state(W, st);
    if (rc != RB_OK) return rc;
    std::string t(table);
    std::vector<unsigned char> out;
    auto put = [&](const void* p, size_t n) { size_t o = out.size(); out.resize(o + n); memcpy(out.data() + o, p, n); };
    const int n = st.npairs;
    std::vector<float4> info;
    if (t.rfind("pair_", 0) == 0 && n > 0) { if ((rc = fetch_rows(W, st, PR_INFO, 1, info)) != RB_OK) return rc; }
    auto geti = [](float f) { int i; memcpy(&i, &f, 4); return i; };
    if (t == "pair_keys") {
        std::vector<unsigned long long> keys(std::max(n, 1));
        CK(d2h(keys.data(), W->w.pb[st.cur].key, (size_t)n * 8));
        put(keys.data(), (size_t)n * 8);
    } else if (t == "pair_nsc" || t == "pair_npts" || t == "pair_color") {
        for (int i = 0; i < n; ++i) { int v = t == "pair_nsc" ? geti(info[i].z) : (t == "pair_npts" ? geti(info[i].y) : geti(info[i].w)); put(&v, 4); }
    } else if (t == "pair_normal") {
        std::vector<float4> r;
        if (n > 0 && (rc = fetch_rows(W, st, PR_NORMAL, 1, r)) != RB_OK) return rc;
        for (int i = 0; i < n; ++i) put(&r[i], 12);
    } else if (t == "pair_points") {
        std::vector<float4> pa, pb, pd;
        if (n > 0) { fetch_rows(W, st, PR_PA, MAX_PTS, pa); fetch_rows(W, st, PR_PB, MAX_PTS, pb); fetch_rows(W, st, PR_PD, MAX_PTS, pd); }
        for (int i = 0; i < n; ++i)
            for (int k = 0; k < 4; ++k) {
                float rec[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
                if (k < geti(info[i].y)) {
                    float4 a = pa[(size_t)k * n + i], b = pb[(size_t)k * n + i], d = pd[(size_t)k * n + i];
                    rec[0] = a.x; rec[1] = a.y; rec[2] = a.z; rec[3] = b.x; rec[4] = b.y; rec[5] = b.z; rec[6] = a.w; rec[7] = b.w; rec[8] = d.w;
                }
                put(rec, 36);
            }
    } else if (t == "pair_data") {
        std::vector<float4> pd, tw, d1, d2;
        if (n > 0) { fetch_rows(W, st, PR_PD, MAX_PTS, pd); fetch_rows(W, st, PR_TW, MAX_PTS, tw); fetch_rows(W, st, PR_DP1, MAX_PTS, d1); fetch_rows(W, st, PR_DP2, MAX_PTS, d2); }
        for (int i = 0; i < n; ++i)
            for (int k = 0; k < 4; ++k) {
                float rec[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
                if (k < geti(info[i].y)) {
                    float4 a = pd[(size_t)k * n + i], b = tw[(size_t)k * n + i], c = d1[(size_t)k * n + i], d = d2[(size_t)k * n + i];
                    rec[0] = a.x; rec[1] = a.y; rec[2] = a.z; rec[3] = b.x; rec[4] = b.y; rec[5] = b.z;
                    rec[6] = c.x; rec[7] = c.y; rec[8] = c.z; rec[9] = d.x; rec[10] = d.y; rec[11] = d.z;
                }
                put(rec, 48);
            }
    } else if (t == "pair_sc") {
        std::vector<float4> a1, a2;
        if (n > 0) { fetch_rows(W, st, PR_A1, MAX_PTS, a1); fetch_rows(W, st, PR_A2, MAX_PTS, a2); }
        for (int i = 0; i < n; ++i)
            for (int k = 0; k < 4; ++k) {
                float rec[6] = {0, 0, 0, 0, 0, 0};
                int cid = -1;
                if (k < geti(info[i].z)) {
                    float4 a = a1[(size_t)k * n + i], b = a2[(size_t)k * n + i];
                    rec[0] = a.x; rec[1] = a.y; rec[2] = a.z; rec[3] = b.x; rec[4] = b.y; rec[5] = b.z;
                    cid = geti(a.w);
                }
                put(rec, 24);
                put(&cid, 4);
            }
    } else if (t == "collider_aabb" || t == "collider_fat") {
        int nc = W->w.nc;
        std::vector<float4> lo(std::max(nc, 1)), hi(std::max(nc, 1));
        CK(d2h(lo.data(), t == "collider_aabb" ? W->w.c_aabb_min : W->w.c_fat_min, (size_t)nc * 16));
        CK(d2h(hi.data(), t == "collider_aabb" ? W->w.c_aabb_max : W->w.c_fat_max, (size_t)nc * 16));
        for (int i = 0; i < nc; ++i) { put(&lo[i], 12); put(&hi[i], 12); }
    } else if (t == "body_mprops") {
        int nb = W->w.nb;
        std::vector<float4> lc(std::max(nb, 1)), ipi(std::max(nb, 1)), wc(std::max(nb, 1)), e0(std::max(nb, 1));
        std::vector<float2> e1(std::max(nb, 1));
        CK(d2h(lc.data(), W->w.b_lcom_im, (size_t)nb * 16)); CK(d2h(ipi.data(), W->w.b_ipi, (size_t)nb * 16));
        CK(d2h(wc.data(), W->w.b_wcom, (size_t)nb * 16)); CK(d2h(e0.data(), W->w.b_eii0, (size_t)nb * 16));
        CK(d2h(e1.data(), W->w.b_eii1, (size_t)nb * 8));
        for (int i = 0; i < nb; ++i) { put(&lc[i], 16); put(&ipi[i], 12); put(&wc[i], 12); put(&e0[i], 16); put(&e1[i], 8); }
    } else if (t == "joint_impulses") {
        std::vector<float> v((size_t)std::max(W->w.nj, 1) * 6);
        CK(d2h(v.data(), W->w.j_impulses, (size_t)W->w.nj * 24));
        put(v.data(), (size_t)W->w.nj * 24);
    } else if (t == "joint_color") {
        std::vector<int4> v(std::max(W->w.nj, 1));
        CK(d2h(v.data(), W->w.j_info, (size_t)W->w.nj * 16));
        for (int i = 0; i < W->w.nj; ++i) put(&v[i].w, 4);
    } else if (t == "body_item" || t == "isl_label") {
        std::vector<int> v(std::max(W->w.nb, 1));
        CK(d2h(v.data(), t == "body_item" ? W->w.body_item : W->w.isl_label, (size_t)W->w.nb * 4));
        put(v.data(), (size_t)W->w.nb * 4);
    } else if (t == "sched_cons_pair" || t == "sched_item_cons_start" || t == "sched_item_color_off" || t == "sched_color_pos" || t == "sched_cons_hdr") {
        // the constraint schedule (solver_contact_graph.rs analogue): pair index per schedule slot, slot range per item,
        // colour-stage offsets per item, stage position of each colour, (pair, id1, id2, n) headers
        const int ni = st.nitems;
        if (t == "sched_cons_pair") { std::vector<int> v(std::max(st.ncons, 1)); CK(d2h(v.data(), W->w.cons_pair, (size_t)st.ncons * 4)); put(v.data(), (size_t)st.ncons * 4); }
        else if (t == "sched_cons_hdr") { std::vector<int4> v(std::max(st.ncons, 1)); CK(d2h(v.data(), W->w.cons_hdr, (size_t)st.ncons * 16)); put(v.data(), (size_t)st.ncons * 16); }
        else if (t == "sched_item_cons_start") { std::vector<int> v(ni + 1); CK(d2h(v.data(), W->w.item_cons_start, (size_t)(ni + 1) * 4)); put(v.data(), (size_t)(ni + 1) * 4); }
        else if (t == "sched_item_color_off") { std::vector<int> v((size_t)ni * (NUM_COLORS + 1)); CK(d2h(v.data(), W->w.item_color_off, v.size() * 4)); put(v.data(), v.size() * 4); }
        else { std::vector<int> v(NUM_COLORS + 1); CK(d2h(v.data(), W->w.color_pos, v.size() * 4)); put(v.data(), v.size() * 4); }
    } else if (t == "dbg_times") {
        long long v[32];
        CK(d2h(v, W->w.dbg_times, sizeof(v)));
        put(v, sizeof(v));
    } else if (t == "state") {
        put(&st, sizeof(st));
    } else {
        set_err("unknown debug table %s", table);
        return RB_ERR_INVALID;
    }
    int64_t total = (int64_t)out.size();
    int64_t ncopy = total < cap ? total : cap;
    if (dst && ncopy > 0) memcpy(dst, out.data(), (size_t)ncopy);
    return total;
}

// Unit-level known-answer entry point (parity tests): evaluates one device function on literal inputs.
int rb_debug_kat(const char* name, const float* in, int32_t n_in, float* out, int32_t n_out) {
    if (!name || !in || !out || n_in <= 0 || n_out <= 0) { set_err("invalid arguments%s", ""); return RB_ERR_INVALID; }
    static const struct { const char* n; int id, nin, nout; } T[] = {
        {"pose_drift", KAT_POSE_DRIFT, 15, 1}, {"reduce_manifold", KAT_REDUCE, 5, 5}, {"normal_solve", KAT_NORMAL_SOLVE, 37, 13},
        {"tangent_solve", KAT_TANGENT_SOLVE, 59, 14}, {"generate", KAT_GENERATE, 25, 39}};
    int which = -1, nout = 0;
    for (auto& t : T)
        if (!strcmp(t.n, name)) {
            if (n_in < t.nin || n_out < t.nout) { set_err("buffer too small for %s", name); return RB_ERR_INVALID; }
            which = t.id; nout = t.nout;
        }
    if (which < 0) { set_err("unknown function %s", name); return RB_ERR_INVALID; }
    if (which == KAT_REDUCE && ((int)in[0] < 0 || (int)in[0] > MAX_RAW || n_in < 5 + 4 * (int)in[0])) return RB_ERR_INVALID;
    if (which == KAT_GENERATE && ((int)in[5] < 1 || (int)in[5] > MAX_PTS || n_in < 6 + 19 * (int)in[5])) return RB_ERR_INVALID;
    RbWorld tmp;
    RbWorld* W = &tmp;
    World& w = W->w;
    w.pair_cap = 1; w.cons_cap = 1;
    RbIntegrationParameters dp;
    rb_integration_parameters_default(&dp);
    derive_params(dp, w.prm);
    float *din = nullptr, *dout = nullptr;
    int rc = RB_OK;
    auto body = [&]() -> int {
        ALLOC(w.pb[0].rows, PR_ROWS); ALLOC(w.cons_hdr, 1); ALLOC(w.cons, CR_ROWS); ALLOC(w.item_flags, 2);
        ALLOC(din, n_in); ALLOC(dout, nout);
        CK(h2d(din, in, (size_t)n_in * sizeof(float)));
        CK(launch(W, k_kat, 1, 1, 0, false, w, which, din, dout));
        CK(stream_sync(W->stream));
        CK(d2h(out, dout, (size_t)nout * sizeof(float)));
        return RB_OK;
    };
    rc = body();
    free_all(W);
    return rc;
}

// ---- multi-GPU sharding ----
int rb_world_label_components(RbWorld* W, int32_t* component_of_body) {
    if (!W || !component_of_body) return RB_ERR_INVALID;
    // Run the collision pipeline once (it leaves poses untouched) so the island labels are current.
    CK(set_device(W->device));
    int one = 1;
    CK(stream_sync(W->stream));
    CK(h2d(&W->w.st->sched_dirty, &one, sizeof(int)));
    CK(launch(W, W->ext_shapes ? k_collide<1> : k_collide<0>, W->collide_blocks, COLLIDE_THREADS, ITEM_SMEM_BYTES, true, W->w, Grav{0.f, 0.f, 0.f}, 0));
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    CK(d2h(component_of_body, W->w.isl_label, (size_t)W->w.nb * sizeof(int)));
    for (int i = 0; i < W->w.nb; ++i)
        if (!type_moves(W->bodies[i].body_type)) component_of_body[i] = -1;
    return RB_OK;
}

int rb_world_set_owned_bodies(RbWorld* W, const uint8_t* owned) {
    if (!W || !owned) return RB_ERR_INVALID;
    if (W->steps > 0) {   // the partition drops the pair table (warm start, colours): only before the first step
        set_err("rb_world_set_owned_bodies must be called before the world is stepped%s", "");
        return RB_ERR_INVALID;
    }
    int rc = sync_world(W);
    if (rc != RB_OK) return rc;
    CK(h2d(W->w.b_owned, owned, (size_t)W->w.nb));
    // Ownership changes the pair filter: drop the pair table and every derived structure.
    State st;
    CK(d2h(&st, W->w.st, sizeof(st)));
    st.npairs = 0; st.bp_dirty = 1; st.lists_dirty = 3; st.sched_dirty = 1; st.ntodo = 0; st.ncons = 0; st.nitems = 1; st.nlarge_bodies = 0;
    CK(h2d(W->w.st, &st, sizeof(st)));
    CK(dev_set(W->w.color_mask, 0, (size_t)std::max(W->w.nb, 1) * 16));
    CK(dev_set(W->w.c_fat_min, 0, (size_t)std::max(W->w.nc, 1) * 16));
    CK(dev_set(W->w.c_fat_max, 0, (size_t)std::max(W->w.nc, 1) * 16));
    return RB_OK;
}

// Halo bodies: which bodies of OTHER ranks this rank tracks (flags_dev: device array [num_bodies], non-zero = track).
// Stream-ordered, no host synchronisation; contact state of everything else is untouched.
int rb_world_set_halo_bodies(RbWorld* W, const uint8_t* flags_dev) {
    if (!W || !flags_dev) return RB_ERR_INVALID;
    CK(set_device(W->device));
    CK(launch(W, k_set_halo, (W->w.nb + 255) / 256, 256, 0, false, W->w, flags_dev));
    return RB_OK;
}
// Imports the states of the halo bodies from the packed state table (after an exchange wrote their rows).
int rb_world_import_halo(RbWorld* W) {
    if (!W) return RB_ERR_INVALID;
    CK(set_device(W->device));
    CK(launch(W, k_import_halo, (W->w.nb + 255) / 256, 256, 0, false, W->w));
    return RB_OK;
}

int rb_world_state_buffer(RbWorld* W, void** device_ptr, int64_t* bytes) {
    if (!W || !device_ptr || !bytes) return RB_ERR_INVALID;
    *device_ptr = W->w.state13;
    *bytes = (int64_t)W->w.nb * 13 * 4;
    return RB_OK;
}

static int import_states_impl(RbWorld* W, const int32_t* idx_dev, const float* src_dev, int32_t n, int table) {
    if (!W || n < 0) return RB_ERR_INVALID;
    if (n == 0) return RB_OK;
    CK(set_device(W->device));
    CK(launch(W, k_import_states, (n + 255) / 256, 256, 0, false, W->w, idx_dev, src_dev, n, table));
    return RB_OK;
}
// Imports externally simulated body states (device pointers): idx[n] body indices, src[n*13].
int rb_world_import_states(RbWorld* W, const int32_t* idx_dev, const float* src_dev, int32_t n) {
    return import_states_impl(W, idx_dev, src_dev, n, 0);
}
// ... from a whole [num_bodies][13] state table (one of the two buffers of rb_world_state_buffers).
int rb_world_import_states_from(RbWorld* W, const int32_t* idx_dev, const float* table_dev, int32_t n) {
    if (!table_dev) return RB_ERR_INVALID;
    return import_states_impl(W, idx_dev, table_dev, n, 1);
}
// Turns on double buffering of the packed state: step k writes buffer (k & 1) counted from this call, so an
// asynchronous in-place all-gather of the buffer just written can run under the next step.
int rb_world_state_buffers(RbWorld* W, void** ptr0, void** ptr1, int64_t* bytes) {
    if (!W || !ptr0 || !ptr1 || !bytes) return RB_ERR_INVALID;
    const size_t n = (size_t)std::max(W->w.nb, 1) * 13;
    if (!W->state_buf[1]) {
        float* second = nullptr;
        int rc = alloc_arr(W, &second, n);
        if (rc != RB_OK) return rc;
        W->state_buf[0] = W->w.state13;
        W->state_buf[1] = second;
        CK(set_device(W->device));
        CK(copy_async(second, W->w.state13, n * sizeof(float), cudaMemcpyDeviceToDevice, W->stream));
        CK(stream_sync(W->stream));
        W->state_next = 0;
    }
    *ptr0 = W->state_buf[0]; *ptr1 = W->state_buf[1];
    *bytes = (int64_t)W->w.nb * 13 * 4;
    return RB_OK;
}

// CUDA stream of the world (for callers that enqueue NCCL work behind the step).
void* rb_world_stream(RbWorld* W) { return W ? (void*)W->stream : nullptr; }


// Use a caller-provided CUDA stream (e.g. torch's current stream) for all of this world's work.
int rb_world_set_stream(RbWorld* W, void* stream) {
    if (!W) return RB_ERR_INVALID;
#if RB_DEVICE_BUILD
    CK(cudaStreamSynchronize(W->stream));
    if (W->own_stream && W->stream) cudaStreamDestroy(W->stream);
    W->stream = (cudaStream_t)stream;
    W->own_stream = false;
#else
    (void)stream;
#endif
    return RB_OK;
}

// End-to-end step with HOST buffers (the call a host-side RigidBodySet owner makes every step):
// uploads all body states (13 floats/body: t3 q4 lin3 ang3) from host memory, runs one step, and
// downloads the resulting states.  Copies go through an internal pinned staging buffer.
int rb_world_step_host(RbWorld* W, const float gravity[3], const float* in_state13, float* out_state13) {
    if (!W || !gravity) return RB_ERR_INVALID;
    const size_t n = (size_t)W->w.nb * 13;
    CK(set_device(W->device));
    // Page-locked caller buffers (cudaHostAlloc / cudaHostRegister / torch pin_memory) are DMA'd directly;
    // pageable ones are staged through the library's pinned buffer.  (The emulation stages every buffer.)
    auto is_pinned = [](const void* p) {
#if RB_DEVICE_BUILD
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return a.type == cudaMemoryTypeHost;
#else
        (void)p;
        return false;
#endif
    };
    if (in_state13) {
        const float* src = in_state13;
        if (!is_pinned(in_state13)) { memcpy(W->stage_host, in_state13, n * sizeof(float)); src = W->stage_host; }
        CK(copy_async(W->stage_dev, src, n * sizeof(float), cudaMemcpyHostToDevice, W->stream));
        int rc = rb_world_import_states(W, W->ident_dev, W->stage_dev, W->w.nb);
        if (rc != RB_OK) return rc;
    }
    int rc = rb_world_step(W, gravity, 1, 0);
    if (rc != RB_OK) return rc;
    if (out_state13) {
        float* dst = is_pinned(out_state13) ? out_state13 : W->stage_host + n;
        auto fetch = [&]() {
            const cudaError_t e = copy_async(dst, W->w.state13, n * sizeof(float), cudaMemcpyDeviceToHost, W->stream);
            return e != cudaSuccess ? e : stream_sync(W->stream);
        };
        CK(fetch());
        if (*(volatile int*)(W->host_hint + 3) != 0) {   // CCD clamps were queued by this step: apply them and fetch the state again
            if ((rc = sync_world(W, false)) != RB_OK) return rc;
            CK(fetch());
        }
        if (dst != out_state13) memcpy(out_state13, dst, n * sizeof(float));
    }
    return sync_world(W);   // (the stream is idle by now: this only reports a status the device raised)
}

}  // extern "C"
