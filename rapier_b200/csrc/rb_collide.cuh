// rb_collide.cuh -- collision-detection and scheduling phases of the step, executed by ONE
// cooperative persistent kernel (k_collide): collider refresh -> [broad phase] -> narrow phase ->
// [colouring, islands, schedule].  Bracketed sections run only when a device-side flag says the
// fat-AABB set / touching set changed (the reference does the same work incrementally on the CPU).
//
// Reference path replaced (SURVEY.md 8a rows a2-a6):
//   a2 Collider::compute_broad_phase_aabb           src/geometry/collider.rs:553-599
//   a3 BroadPhaseBvh::update / set_aabb             src/geometry/broad_phase_bvh/update.rs:35-602, mod.rs:235-263
//   a4 NarrowPhase::compute_contacts / process_pair src/geometry/narrow_phase/contacts.rs:22-293, pair_update.rs:67-680
//   a5 apply_pair_transitions + colouring           contacts.rs:300-385, narrow_phase/mod.rs:87-172
//   a6 maintain_solver_contact_graph                narrow_phase/solver_graph.rs:129-361 (here: islands + schedule)
#pragma once
#include "rb_geom.cuh"

namespace rb {

// -DRB_DEBUG build with RB_DEBUG_FLAGS & 4: thread 0 stamps the end of every section (tests/prof_collide_phases.py)
#ifdef RB_DEBUG
#define RB_CSTAMP(k) do { if ((w.debug_flags & 4) && ctx.gtid == 0) w.dbg_times[16 + (k)] = rb_clock(); } while (0)
#else
#define RB_CSTAMP(k) do { } while (0)
#endif


constexpr int ITEM_TARGET = 128;   // cost (max(bodies, constraints)) packed into one CTA work item
constexpr int ITEM_BODY_CAP = 256; // islands above either cap go to the grid-wide "large" item 0
constexpr int ITEM_CONS_CAP = 3072;
constexpr int ITEM_MAX_BODIES = ITEM_BODY_CAP + ITEM_TARGET;  // shared-memory sizing of the item kernel
constexpr int BIG_COLOR_MIN = 125;   // ceil(n/4) >= 32 chunks (init.rs:169: CHUNK_BATCH*LAYOUT_REF_WORKERS/2)
constexpr int BIG_JCOLOR_MIN = 64;   // joints.rs:340: JOINT_BATCH*LAYOUT_REF_WORKERS/2

// Multi-GPU sharding (b_owned): 1 = simulated by this rank, 2 = "halo": simulated by another rank but close enough to
// be tracked here (its state is imported every step, its colliders take part in proximity detection), 0 = simulated
// by another rank and far away (ignored until the next halo refresh).
// Kinematic bodies are solver bodies like dynamic ones -- zero effective inverse mass, velocities read by their
// contacts, poses integrated by the substeps (solver_body.rs:112-120; is_dynamic_or_kinematic) -- and are coloured
// like them (narrow_phase/mod.rs:105-106: "conflicting" = not fixed).  DEVIATION: here they are also island members
// (the reference keeps them as singleton islands, substep_groups.rs:64-66), so what a platform carries shares its
// island: same solve, coarser sleeping and scheduling granularity.
RB_HD bool type_is_solver(int t) { return t == BODY_DYNAMIC || t == BODY_KIN_POS || t == BODY_KIN_VEL; }
RB_HD bool body_is_dyn(const World& w, int b) {  // dynamic or kinematic, and simulated by this rank (awake or asleep)
    return b >= 0 && type_is_solver(w.b_type[b]) && w.b_owned[b] == 1;
}
RB_HD bool body_is_strict_dyn(const World& w, int b) { return b >= 0 && w.b_type[b] == BODY_DYNAMIC && w.b_owned[b] == 1; }
// ... and awake: a member of the active set (island_manager: sleeping bodies are neither solved nor integrated)
RB_HD bool body_is_sim(const World& w, int b) { return body_is_dyn(w, b) && !w.b_sleeping[b]; }
// ContactManifoldData::relative_dominance (pair_update.rs:381-382; effective_group rigid_body_components.rs:1267-1275):
// > 0 = body 1 dominates and is world-attached in this contact, < 0 = body 2.  The group is a signed byte in b_flags.
RB_HD int body_dominance(const World& w, int b) {
    return (b >= 0 && type_is_solver(w.b_type[b])) ? (int)(signed char)((w.b_flags[b] >> 16) & 0xffu) : 128;
}
RB_HD int relative_dominance(const World& w, int b1, int b2) { return body_dominance(w, b1) - body_dominance(w, b2); }
RB_HD pose body_pose(const World& w, int b) { return mkpose(mkq(w.b_pos_q[b]), xyz(w.b_pos_t[b])); }
RB_HD pose collider_pose(const World& w, int c) { return mkpose(mkq(w.c_pos_q[c]), xyz(w.c_pos_t[c])); }

// ------------------------------------------------------------------------------------------------
// P0: collider world poses, broad-phase AABBs and fat-AABB change detection
// (substep.rs:103-146 + refresh_moved_collider_aabbs substep.rs:229-240 -> BroadPhaseBvh::set_aabb).
// Static colliders (no parent, or a parent that is not dynamic) never move: once the static / dynamic lists
// exist only the dynamic list is refreshed (a 10^6-tile floor costs nothing per step).
// ------------------------------------------------------------------------------------------------
template <int SHAPES = 0>
RB_HD void refresh_collider(const World& w, int c) {
    int parent = w.c_parent[c];
    pose rel = mkpose(mkq(w.c_rel_q[c]), xyz(w.c_rel_t[c]));
    pose p = parent >= 0 ? pmul(body_pose(w, parent), rel) : rel;
    w.c_pos_t[c] = f4(p.t, 0.0f);
    w.c_pos_q[c] = f4(p.q);
    vec3 lo, hi;
    if (SHAPES && w.c_shape[c] == SHAPE_CONVEX) convex_aabb(w.hulls, xyz(w.c_he[c]), p, lo, hi);
    else shape_aabb(w.c_shape[c], xyz(w.c_he[c]), p, lo, hi);
    float l = w.c_mat[c].z + w.prm.prediction / 2.0f;
    lo = mk3(lo.x - l, lo.y - l, lo.z - l);
    hi = mk3(hi.x + l, hi.y + l, hi.z + l);
    w.c_aabb_min[c] = f4(lo, 0.0f);
    w.c_aabb_max[c] = f4(hi, 0.0f);
    float4 fmin = w.c_fat_min[c], fmax = w.c_fat_max[c];
    bool valid = fmin.w != 0.0f;
    bool contains = valid && fmin.x <= lo.x && fmin.y <= lo.y && fmin.z <= lo.z && fmax.x >= hi.x && fmax.y >= hi.y &&
                    fmax.z >= hi.z;
    if (!contains) {
        float s = w.prm.fat_skin;
        w.c_fat_min[c] = make_float4(lo.x - s, lo.y - s, lo.z - s, 1.0f);
        w.c_fat_max[c] = make_float4(hi.x + s, hi.y + s, hi.z + s, 1.0f);
        w.st->bp_dirty = 1;
    }
}
template <int SHAPES = 0, class Ctx>
RB_PHASE void phase_refresh_colliders(const Ctx& ctx, const World& w) {
    if (w.st->lists_dirty) {
        for (int c = ctx.gtid; c < w.nc; c += ctx.gsize) {
            const int parent = w.c_parent[c];
            if (parent >= 0 && w.b_type[parent] == BODY_REMOVED) w.c_shape[c] = SHAPE_REMOVED;   // (removed or quarantined body)
            if (w.c_shape[c] != SHAPE_REMOVED) refresh_collider<SHAPES>(w, c);
        }
    } else {
        const int nd = w.st->ndyn;
        for (int i = ctx.gtid; i < nd; i += ctx.gsize) refresh_collider<SHAPES>(w, w.dyn_list[i]);
    }
}

RB_HD int next_pow2(int n) {
    int p = 1;
    while (p < n) p <<= 1;
    return p;
}

RB_HD unsigned sortable_float(float f) {
    unsigned u = as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

RB_HD int bsearch_u64(const unsigned long long* a, int n, unsigned long long key) {
    int lo = 0, hi = n - 1;
    while (lo <= hi) {
        int mid = (lo + hi) >> 1;
        unsigned long long v = a[mid];
        if (v == key) return mid;
        if (v < key) lo = mid + 1; else hi = mid - 1;
    }
    return -1;
}
RB_HD int lower_bound_u64(const unsigned long long* a, int n, unsigned long long key) {   // first index with a[i] >= key
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// ------------------------------------------------------------------------------------------------
// Grid-wide stable LSD radix sort of 64-bit keys on the bits [lo, hi), 8 bits per pass, ONE grid barrier per
// pass (the north star's "device radix sort"; it replaced a bitonic network with log^2 n barriers).
//   * every CTA owns a contiguous chunk of the array, every warp a contiguous part of that chunk, so "block,
//     warp, position" order is index order and the scatter is stable;
//   * the per-(block, digit) counts of pass p+1 are accumulated with global atomics WHILE pass p scatters
//     (the destination block of a key is known then), so a pass needs no counting sweep of its own;
//   * offsets: each CTA sums the small [blocks][256] count table itself (no grid-wide scan).
// `hist` holds (passes + 1) tables of nblocks x 256 ints and must be ZERO on entry, the keys must be in `a`,
// and a grid barrier must separate both from this call.  Returns the buffer that holds the result.
// ------------------------------------------------------------------------------------------------
constexpr int RADIX = 256;
constexpr int RADIX_MAX_WARPS = 8;
RB_HD int radix_passes(int lo, int hi) { return (hi - lo + 7) / 8; }
RB_HD int bits_for(int n) { int b = 1; while ((1 << b) < n && b < 31) ++b; return b; }

#if RB_DEVICE_BUILD
RB_D unsigned warp_match_any(int v) { return __match_any_sync(0xffffffffu, v); }
RB_D void warp_sync() { __syncwarp(); }
RB_D int popc(unsigned x) { return __popc(x); }
#else
inline unsigned warp_match_any(int) { return 1u; }
inline void warp_sync() {}
inline int popc(unsigned x) { return __builtin_popcount(x); }
#endif

template <class Ctx>
RB_PHASE void grid_radix_zero(const Ctx& ctx, int* hist, int passes) {
    const int n = (passes + 1) * ctx.nblocks * RADIX;
    for (int i = ctx.gtid; i < n; i += ctx.gsize) hist[i] = 0;
}

template <class Ctx>
RB_PHASE unsigned long long* grid_radix_sort(const Ctx& ctx, unsigned long long* a, unsigned long long* b, int n, int lo, int hi,
                                             int* hist) {
    RB_SHARED int s_warp[RADIX_MAX_WARPS][RADIX];   // per-warp digit counts, then running scatter offsets
    RB_SHARED int s_tot[RADIX];
    const int passes = radix_passes(lo, hi);
    // CTAs that take part: at least 1024 keys each (a handful of keys spread over every CTA only lengthens the
    // per-digit walk over the CTAs' histograms below: one dependent L2 read per CTA per pass); the others hold empty chunks
    const int nblocks = ctx.nblocks < (n + 1023) / 1024 ? ctx.nblocks : ((n + 1023) / 1024 > 0 ? (n + 1023) / 1024 : 1);
    const int chunk = (n + nblocks - 1) / nblocks > 0 ? (n + nblocks - 1) / nblocks : 1;
    const int nwarps = ctx.bsize / ctx.nlanes < RADIX_MAX_WARPS ? ctx.bsize / ctx.nlanes : RADIX_MAX_WARPS;
    const int wchunk = (chunk + nwarps - 1) / nwarps;
    const int warp = ctx.btid / ctx.nlanes;
    const int b0 = ctx.bid * chunk, b1 = b0 + chunk < n ? b0 + chunk : n;
    // counts of the first pass
    for (int i = b0 + ctx.btid; i < b1; i += ctx.bsize) atomic_add(&hist[ctx.bid * RADIX + (int)((a[i] >> lo) & 255)], 1);
    ctx.grid_sync();
    for (int p = 0; p < passes; ++p) {
        const int shift = lo + 8 * p;
        const int* h = hist + (size_t)p * ctx.nblocks * RADIX;
        int* hn = hist + (size_t)(p + 1) * ctx.nblocks * RADIX;
        // per digit: total over all blocks, and the part of it that precedes this block
        for (int d = ctx.btid; d < RADIX; d += ctx.bsize) {
            int tot = 0, before = 0;
            for (int k = 0; k < nblocks; ++k) {
                int v = h[k * RADIX + d];
                tot += v;
                if (k < ctx.bid) before += v;
            }
            s_tot[d] = tot;
            s_warp[0][d] = before;   // (parked here until the exclusive scan below)
        }
        ctx.block_sync();
        if (ctx.btid == 0) {
            int run = 0;
            for (int d = 0; d < RADIX; ++d) { int v = s_tot[d]; s_tot[d] = run + s_warp[0][d]; run += v; }   // s_tot = first slot of (digit, this block)
        }
        ctx.block_sync();
        for (int i = ctx.btid; i < nwarps * RADIX; i += ctx.bsize) s_warp[i / RADIX][i % RADIX] = 0;
        ctx.block_sync();
        // per-warp counts over the warp's own part of the chunk
        const int w0 = b0 + warp * wchunk, w1 = (w0 + wchunk < b1 ? w0 + wchunk : b1);
        if (warp < nwarps)
            for (int i = w0 + ctx.lane; i < w1; i += ctx.nlanes) atomic_add(&s_warp[warp][(int)((a[i] >> shift) & 255)], 1);
        ctx.block_sync();
        for (int d = ctx.btid; d < RADIX; d += ctx.bsize) {   // counts -> first slot of (digit, this warp)
            int run = s_tot[d];
            for (int k = 0; k < nwarps; ++k) { int v = s_warp[k][d]; s_warp[k][d] = run; run += v; }
        }
        ctx.block_sync();
        // stable scatter, a warp-load at a time in index order
        if (warp < nwarps)
            for (int base = w0; base < w1; base += ctx.nlanes) {
                const int i = base + ctx.lane;
                const bool valid = i < w1;
                unsigned long long key = valid ? a[i] : 0ull;
                const int d = valid ? (int)((key >> shift) & 255) : 0x1000 + ctx.lane;
                const unsigned peers = warp_match_any(d);
                const int rank = popc(peers & ((1u << ctx.lane) - 1u));
                int dest = 0;
                if (valid) {
                    dest = s_warp[warp][d] + rank;
                    b[dest] = key;
                    if (p + 1 < passes) atomic_add(&hn[(dest / chunk) * RADIX + (int)((key >> (shift + 8)) & 255)], 1);
                }
                warp_sync();
                if (valid && rank == 0) s_warp[warp][d] += popc(peers);
                warp_sync();
            }
        ctx.grid_sync();
        unsigned long long* t = a; a = b; b = t;
    }
    return a;
}

// InteractionGroups::test (interaction_groups.rs:136-154): Or applies only when both sides use it, And takes priority.
RB_HD bool groups_test(unsigned m1, unsigned f1, unsigned or1, unsigned m2, unsigned f2, unsigned or2) {
    const bool a = (m1 & f2) != 0, b = (m2 & f1) != 0;
    return (or1 & or2) ? (a || b) : (a && b);
}
// ActiveCollisionTypes::test (collider_components.rs:300-334) on body types numbered like RigidBodyType.
RB_HD bool collision_types_test(unsigned bits, int t1, int t2) {
    return (((bits >> (t1 * 4)) & 15u) & (1u << t2)) != 0 || (((bits >> (t2 * 4)) & 15u) & (1u << t1)) != 0;
}
RB_HD int filter_body_type(const World& w, int b) { return b < 0 ? BODY_FIXED : w.b_type[b]; }   // (a parentless collider is fixed)
// The solver groups fail, or neither body is dynamic: the pair keeps its contacts and touch events but computes no force
// (SolverFlags without COMPUTE_IMPULSES, pair_update.rs:279-281).  Worlds with collider filters only.
RB_HD bool pair_forceless(const World& w, int c1, int c2, int b1, int b2) {
    if (filter_body_type(w, b1) != BODY_DYNAMIC && filter_body_type(w, b2) != BODY_DYNAMIC) return true;
    const uint4 f1 = w.c_filter[c1], f2 = w.c_filter[c2];
    return !groups_test(f1.x, f1.y, f1.w >> 1, f2.x, f2.y, f2.w >> 1);
}

// update.rs:334-396 filter_new
RB_HD bool pair_allowed(const World& w, int c1, int c2) {
    int p1 = w.c_parent[c1], p2 = w.c_parent[c2];
    if (p1 >= 0 && p1 == p2) return false;
    bool d1 = body_is_strict_dyn(w, p1), d2 = body_is_strict_dyn(w, p2);   // (sleeping bodies keep their pairs)
    uint2 g1 = w.c_groups[c1], g2 = w.c_groups[c2];
    if (w.has_filters) {   // (a kernel parameter: uniform)
        // the collision types of either collider (update.rs:361-385; solver groups are not tested here, :365-366), then the
        // mode-aware collision groups.  Which rank keeps the pair (multi-GPU sharding): a pair with a dynamic body simulated
        // here is kept as without filters; a pair whose only dynamic bodies belong to other ranks is not; a pair without a
        // dynamic body is kept by the rank that simulates its lower-indexed body (every rank, for two parentless colliders).
        const int t1 = filter_body_type(w, p1), t2 = filter_body_type(w, p2);
        if (!d1 && !d2) {
            if (t1 == BODY_DYNAMIC || t2 == BODY_DYNAMIC) return false;
            const int lo = p1 < 0 ? p2 : (p2 < 0 ? p1 : (p1 < p2 ? p1 : p2));
            if (lo >= 0 && w.b_owned[lo] != 1) return false;
        }
        const uint4 f1 = w.c_filter[c1], f2 = w.c_filter[c2];
        if (!collision_types_test(f1.z, t1, t2) && !collision_types_test(f2.z, t1, t2)) return false;
        if (!groups_test(g1.x, g1.y, f1.w & 1u, g2.x, g2.y, f2.w & 1u)) return false;
    } else {
        if (!d1 && !d2) return false;   // ActiveCollisionTypes::default(): DYNAMIC_DYNAMIC | DYNAMIC_KINEMATIC | DYNAMIC_FIXED
        if (!((g1.x & g2.y) != 0 && (g2.x & g1.y) != 0)) return false;
    }
    if (w.n_nocontact > 0 && p1 >= 0 && p2 >= 0) {
        unsigned lo = (unsigned)(p1 < p2 ? p1 : p2), hi = (unsigned)(p1 < p2 ? p2 : p1);
        if (bsearch_u64(w.nocontact_keys, w.n_nocontact, ((unsigned long long)lo << 32) | hi) >= 0) return false;
    }
    return true;
}

RB_HD void clear_color_bits(const World& w, int color, int cb0, int cb1) {
    if (color < COLOR_OVERFLOW) {
        unsigned bit = ~(1u << (color & 31));
        if (cb0 >= 0) atomic_and(&w.color_mask[cb0 * 4 + (color >> 5)], bit);
        if (cb1 >= 0) atomic_and(&w.color_mask[cb1 * 4 + (color >> 5)], bit);
    }
}

// EventHandler::handle_collision_event (contacts.rs:312-324): buffered for the host when either collider asks for it.
RB_HD void emit_collision_event(const World& w, int c1, int c2, bool started) {
    if (!((w.c_events[c1] | w.c_events[c2]) & 1)) return;
    const int slot = atomic_add(&w.st->nev_coll, 1);
    if (slot < w.ev_cap) w.ev_coll[slot] = make_int4(c1, c2, started ? 1 : 0, w.step_index);
    else RB_RAISE(w, -4);
}

RB_HD bool collider_is_static(const World& w, int c) {   // never moves: no parent, or a parent that is neither dynamic nor kinematic
    const int p = w.c_parent[c];
    return p < 0 || !type_is_solver(w.b_type[p]);
}
RB_HD bool fat_overlap(float4 amin, float4 amax, float4 bmin, float4 bmax) {
    return amin.x <= bmax.x && amin.y <= bmax.y && amin.z <= bmax.z && amax.x >= bmin.x && amax.y >= bmin.y && amax.z >= bmin.z;
}
RB_HD void emit_candidate(const World& w, int ci, int cj) {
    const int c1 = ci < cj ? ci : cj, c2 = ci < cj ? cj : ci;
    if (!pair_allowed(w, c1, c2)) return;
    const int slot = atomic_add(&w.st->ncand, 1);
    if (slot < w.pair_cap) w.cand_key[slot] = ((unsigned long long)(unsigned)c1 << 32) | (unsigned)c2;
}

constexpr int WIDE_CAP = 1024;   // static colliders much wider than the rest (a ground slab under a tiled floor): tested by every mover

// Fixed-fixed pairs (ActiveCollisionTypes::FIXED_FIXED, broad_phase_bvh/update.rs:361-385): the sweep below starts from the
// movers only, so two static colliders never meet there.  When the static lists are rebuilt, every static collider that opts in
// is searched, one thread each, against the sorted static keys and the wide list; the pairs found stay in ff_keys and join
// every later candidate set (section_broad_phase).
constexpr unsigned ACT_FIXED_FIXED = 0x0020u;
template <class Ctx>
RB_PHASE void section_fixed_pairs(const Ctx& ctx, const World& w, const unsigned long long* skey) {
    State* st = w.st;
    const int ns = st->nstat, nwide = st->nwide < WIDE_CAP ? st->nwide : WIDE_CAP;
    const float wn = as_float(st->stat_wn_bits) * 1.0001f + 1.0e-6f;   // widest narrow static collider (with rounding slack)
    unsigned long long* ff = ff_keys(w);
    for (int c = ctx.gtid; c < w.nc; c += ctx.gsize) {
        if (w.c_shape[c] == SHAPE_REMOVED || !collider_is_static(w, c) || !(w.c_filter[c].z & ACT_FIXED_FIXED)) continue;
        const float4 amin = w.c_fat_min[c], amax = w.c_fat_max[c];
        auto test = [&](int j) {
            if (j == c || (j < c && (w.c_filter[j].z & ACT_FIXED_FIXED))) return;   // (two opted-in colliders: found from the lower one)
            if (!fat_overlap(amin, amax, w.c_fat_min[j], w.c_fat_max[j])) return;
            const int c1 = c < j ? c : j, c2 = c < j ? j : c;
            if (!pair_allowed(w, c1, c2)) return;
            const int slot = atomic_add(&st->nff, 1);
            if (slot < w.pair_cap) ff[slot] = ((unsigned long long)(unsigned)c1 << 32) | (unsigned)c2;
        };
        const unsigned amax_key = sortable_float(amax.x);
        for (int j = lower_bound_u64(skey, ns, (unsigned long long)sortable_float(amin.x - wn) << 32); j < ns; ++j) {
            const unsigned long long kj = skey[j];
            if ((unsigned)(kj >> 32) > amax_key) break;
            test((int)(kj & 0xffffffffu));
        }
        for (int k = 0; k < nwide; ++k) test(w.wide_list[k]);
    }
    ctx.grid_sync();
    if (ctx.gtid == 0 && st->nff > w.pair_cap) RB_RAISE(w, -4);   // (the list keeps what fits; the status reports the rest)
}

// P1 (lists): split the colliders into the movers (sorted every time an AABB changes) and the static ones (sorted
// here, once): the reference keeps all leaves in one tree and only re-tests CHANGED leaves (broad_phase_bvh/
// update.rs:441-601), which static leaves never are.  Static colliders much wider along x than the average go to a
// short list every mover tests, so that one big slab does not defeat the interval search over the narrow ones.
template <class Ctx>
RB_PHASE void section_build_lists(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const bool statics = (st->lists_dirty & 2) != 0;   // bit 1: the static colliders changed too (else only movers were added)
    if (ctx.gtid == 0) {
        st->ndyn = 0;
        if (statics) { st->nstat = 0; st->nwide = 0; st->stat_count = 0; st->stat_wsum = 0.0f; st->stat_wn_bits = 0u; st->nff = 0; }
    }
    if (statics) grid_radix_zero(ctx, w.radix_hist, 4);
    ctx.grid_sync();
    if (statics) {
        for (int c = ctx.gtid; c < w.nc; c += ctx.gsize)
            if (w.c_shape[c] != SHAPE_REMOVED && collider_is_static(w, c)) {
                atomic_add(&st->stat_count, 1);
                atomic_add(&st->stat_wsum, w.c_fat_max[c].x - w.c_fat_min[c].x);
            }
        ctx.grid_sync();
    }
    const float wide_thr = st->stat_count > 0 ? 4.0f * (st->stat_wsum / (float)st->stat_count) : 0.0f;
    for (int c = ctx.gtid; c < w.nc; c += ctx.gsize) {
        if (w.c_shape[c] == SHAPE_REMOVED) continue;   // collider of a removed body: in no list, so its pairs end
        if (!collider_is_static(w, c)) {
            if (w.b_owned[w.c_parent[c]] != 0) w.dyn_list[atomic_add(&st->ndyn, 1)] = c;   // (far foreign bodies are not tracked)
            continue;
        }
        if (!statics) continue;
        const float4 lo = w.c_fat_min[c], hi = w.c_fat_max[c];
        const float width = hi.x - lo.x;
        bool wide = width > wide_thr;
        if (wide) {
            const int k = atomic_add(&st->nwide, 1);
            if (k < WIDE_CAP) w.wide_list[k] = c; else wide = false;   // (the count is clamped where it is read)
        }
        if (!wide) {
            w.stat_key[0][atomic_add(&st->nstat, 1)] = ((unsigned long long)sortable_float(lo.x) << 32) | (unsigned)c;
            atomic_max_u(&st->stat_wn_bits, as_uint(width > 0.0f ? width : 0.0f));   // (non-negative floats order like their bits)
        }
    }
    ctx.grid_sync();
    if (statics) {
        unsigned long long* sorted = grid_radix_sort(ctx, w.stat_key[0], w.stat_key[1], st->nstat, 32, 64, w.radix_hist);
        if (ctx.gtid == 0) st->stat_sorted = sorted == w.stat_key[0] ? 0 : 1;
        if (w.has_filters) section_fixed_pairs(ctx, w, sorted);   // (a kernel parameter: uniform)
    }
    if (ctx.gtid == 0) { st->lists_dirty = 0; st->bp_dirty = 1; }
    ctx.grid_sync();
}

// P1: sort-and-sweep broad phase over the movers + interval search into the sorted static colliders, then the
// merge with the persistent pair table (skipped when the pair set did not change).
// The movers are binned into STRIPS along z as wide as the widest mover, and sorted by (strip, quantised min-x): a
// mover can only touch movers of its own strip and the next one, so a dense 3-D pile costs its neighbours in x of
// two strips, not of the whole x column (a plain 1-axis sweep of a 50 x 50 x 50 brick pyramid tests 2 500 candidates
// per brick).  The sorted AABBs are gathered into contiguous arrays, so the sweep reads coalesced rows.
constexpr int STRIP_BITS = 12, STRIP_COUNT = 1 << STRIP_BITS, XQ_BITS = 32 - STRIP_BITS;
RB_HD unsigned strip_key(float minz, float minx, float inv_wz) {
    float f = floorf(minz * inv_wz) + (float)(STRIP_COUNT / 2);
    f = f < 0.0f ? 0.0f : (f > (float)(STRIP_COUNT - 1) ? (float)(STRIP_COUNT - 1) : f);   // (far strips merge: more tests, never fewer)
    return ((unsigned)f << XQ_BITS) | (sortable_float(minx) >> STRIP_BITS);
}
template <class Ctx>
RB_PHASE void section_broad_phase(const Ctx& ctx, const World& w) {
    State* st = w.st;
    if (st->lists_dirty) section_build_lists(ctx, w);
    const int nd = st->ndyn, ns = st->nstat;
    const int nwide = st->nwide < WIDE_CAP ? st->nwide : WIDE_CAP;
    const unsigned long long* skey = w.stat_key[st->stat_sorted];
    if (ctx.gtid == 0) { st->mov_wz_bits = 0u; st->mov_wx_bits = 0u; st->ncand = 0; }
    grid_radix_zero(ctx, w.radix_hist, 4);
    ctx.grid_sync();
    for (int i = ctx.gtid; i < nd; i += ctx.gsize) {   // widest mover along z (strip width) and x (search reach)
        const int c = w.dyn_list[i];
        const float4 lo = w.c_fat_min[c], hi = w.c_fat_max[c];
        atomic_max_u(&st->mov_wz_bits, as_uint(hi.z - lo.z > 0.0f ? hi.z - lo.z : 0.0f));
        atomic_max_u(&st->mov_wx_bits, as_uint(hi.x - lo.x > 0.0f ? hi.x - lo.x : 0.0f));
    }
    ctx.grid_sync();
    const float wz = as_float(st->mov_wz_bits) * 1.01f + 1.0e-3f, wx = as_float(st->mov_wx_bits) * 1.0001f + 1.0e-6f;   // (1 %: strips of overlapping movers differ by at most one, also after rounding)
    const float inv_wz = 1.0f / wz;
    for (int i = ctx.gtid; i < nd; i += ctx.gsize) {
        const int c = w.dyn_list[i];
        const float4 lo = w.c_fat_min[c];
        w.dyn_key[0][i] = ((unsigned long long)strip_key(lo.z, lo.x, inv_wz) << 32) | (unsigned)c;
    }
    ctx.grid_sync();
    const unsigned long long* dkey = grid_radix_sort(ctx, w.dyn_key[0], w.dyn_key[1], nd, 32, 64, w.radix_hist);
    for (int i = ctx.gtid; i < nd; i += ctx.gsize) {   // the sorted movers' AABBs, contiguous
        const int c = (int)(dkey[i] & 0xffffffffu);
        w.dyn_smin[i] = w.c_fat_min[c];
        w.dyn_smax[i] = w.c_fat_max[c];
    }
    ctx.grid_sync();
    // sweep: one warp per mover, lanes stride over what follows it
    const float wn = as_float(st->stat_wn_bits) * 1.0001f + 1.0e-6f;   // widest narrow static collider (with rounding slack)
    for (int wi = ctx.gwarp; wi < nd; wi += ctx.ngwarps) {
        const unsigned long long ki = dkey[wi];
        const int ci = (int)(ki & 0xffffffffu);
        const float4 amin = w.dyn_smin[wi], amax = w.dyn_smax[wi];
        const unsigned strip = (unsigned)(ki >> 32) >> XQ_BITS;
        const unsigned own_end = (strip << XQ_BITS) | (sortable_float(amax.x) >> STRIP_BITS);   // last key of the own strip that can overlap in x
        for (int base = wi + 1; base < nd; base += ctx.nlanes) {   // own strip: movers that follow in (quantised) x
            const int j = base + ctx.lane;
            bool stop = true;
            if (j < nd) {
                const unsigned long long kj = dkey[j];
                stop = (unsigned)(kj >> 32) > own_end;
                if (!stop && fat_overlap(amin, amax, w.dyn_smin[j], w.dyn_smax[j])) emit_candidate(w, ci, (int)(kj & 0xffffffffu));
            }
            if (ctx.warp_any(stop)) break;
        }
        if (strip + 1 < (unsigned)STRIP_COUNT) {   // next strip: movers whose x interval can reach ours
            const unsigned nlo = ((strip + 1) << XQ_BITS) | (sortable_float(amin.x - wx) >> STRIP_BITS);
            const unsigned nhi = ((strip + 1) << XQ_BITS) | (sortable_float(amax.x) >> STRIP_BITS);
            const int first = lower_bound_u64(dkey, nd, (unsigned long long)nlo << 32);
            for (int base = first; base < nd; base += ctx.nlanes) {
                const int j = base + ctx.lane;
                bool stop = true;
                if (j < nd) {
                    const unsigned long long kj = dkey[j];
                    stop = (unsigned)(kj >> 32) > nhi;
                    if (!stop && fat_overlap(amin, amax, w.dyn_smin[j], w.dyn_smax[j])) emit_candidate(w, ci, (int)(kj & 0xffffffffu));
                }
                if (ctx.warp_any(stop)) break;
            }
        }
        // narrow static colliders whose x interval can reach [amin.x, amax.x]: min-x in [amin.x - wn, amax.x]
        const unsigned amax_key = sortable_float(amax.x);
        const int first = lower_bound_u64(skey, ns, (unsigned long long)sortable_float(amin.x - wn) << 32);
        for (int base = first; base < ns; base += ctx.nlanes) {
            const int j = base + ctx.lane;
            bool stop = true;
            if (j < ns) {
                const unsigned long long kj = skey[j];
                stop = (unsigned)(kj >> 32) > amax_key;
                if (!stop) {
                    const int cj = (int)(kj & 0xffffffffu);
                    if (fat_overlap(amin, amax, w.c_fat_min[cj], w.c_fat_max[cj])) emit_candidate(w, ci, cj);
                }
            }
            if (ctx.warp_any(stop)) break;
        }
        for (int k = ctx.lane; k < nwide; k += ctx.nlanes) {       // the few wide ones
            const int cj = w.wide_list[k];
            if (fat_overlap(amin, amax, w.c_fat_min[cj], w.c_fat_max[cj])) emit_candidate(w, ci, cj);
        }
    }
    if (w.has_filters) {   // the fixed-fixed pairs of the last static rebuild (section_fixed_pairs), filtered again
        const int nff = st->nff < w.pair_cap ? st->nff : w.pair_cap;
        const unsigned long long* ff = ff_keys(w);
        for (int k = ctx.gtid; k < nff; k += ctx.gsize) emit_candidate(w, (int)(ff[k] >> 32), (int)(ff[k] & 0xffffffffu));
    }
    const int cbits = bits_for(w.nc > 2 ? w.nc : 2);
    const int p_lo = radix_passes(0, cbits), p_hi = radix_passes(32, 32 + cbits);
    grid_radix_zero(ctx, w.radix_hist, p_lo > p_hi ? p_lo : p_hi);
    ctx.grid_sync();
    const int ncand = st->ncand;
    if (ncand > w.pair_cap) {  // capacity overflow: keep the old pair set and raise the status; the pair set stays dirty,
                               // so every step raises it again until the world fits (no silently stale physics)
        if (ctx.gtid == 0) RB_RAISE(w, -4);
        ctx.grid_sync();
        return;
    }
    // order the candidates by (collider1, collider2): LSD over the low word's used bits, then the high word's
    unsigned long long* ck = grid_radix_sort(ctx, w.cand_key, w.cand_key2, ncand, 0, cbits, w.radix_hist);
    unsigned long long* other = ck == w.cand_key ? w.cand_key2 : w.cand_key;
    grid_radix_zero(ctx, w.radix_hist, p_hi);
    ctx.grid_sync();
    ck = grid_radix_sort(ctx, ck, other, ncand, 32, 32 + cbits, w.radix_hist);
    // unchanged pair set (the usual case while AABBs merely move): nothing to merge, the schedule stays valid
    int cur = st->cur, nxt = 1 - cur, nold = st->npairs;
    const unsigned long long* okey = w.pb[cur].key;
    if (ctx.gtid == 0) st->bp_diff = ncand != nold ? 1 : 0;
    ctx.grid_sync();
    if (ncand == nold) {
        int diff = 0;
        for (int i = ctx.gtid; i < ncand; i += ctx.gsize) diff |= ck[i] != okey[i];
        if (diff) st->bp_diff = 1;
        ctx.grid_sync();
    }
    if (!st->bp_diff) {   // (bp_dirty / bp_ran are not read again during this step)
        if (ctx.gtid == 0) { st->bp_dirty = 0; st->bp_ran = 1; st->ncand = 0; }
        return;
    }
    // merge: carry persistent per-pair state from the old sorted table to the new one.
    for (int i = ctx.gtid; i < ncand; i += ctx.gsize) {
        unsigned long long k = ck[i];
        w.pb[nxt].key[i] = k;
        w.remap_src[i] = bsearch_u64(okey, nold, k);
    }
    ctx.grid_sync();
    for (long long e = ctx.gtid; e < (long long)ncand * PR_ROWS; e += ctx.gsize) {
        int r = (int)(e / ncand), i = (int)(e % ncand);
        int src = w.remap_src[i];
        float4 v;
        if (src >= 0) {
            v = prow(w, cur, r, src);
        } else {
            v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r == PR_INFO) v.w = as_float_i(COLOR_UNCOLORED);
            if (r == PR_BODIES) {
                unsigned long long k = ck[i];
                int c1 = (int)(k >> 32), c2 = (int)(k & 0xffffffffu);
                v = make_float4(as_float_i(-1), as_float_i(-1), as_float_i(w.c_parent[c1]), as_float_i(w.c_parent[c2]));
            }
        }
        prow(w, nxt, r, i) = v;
    }
    // removed pairs: end-touch frees the colour (contacts.rs:333-335).
    for (int j = ctx.gtid; j < nold; j += ctx.gsize) {
        if (bsearch_u64(ck, ncand, okey[j]) < 0) {
            float4 info = prow(w, cur, PR_INFO, j), bod = prow(w, cur, PR_BODIES, j);
            if (as_int(info.z) > 0 || (as_int(info.x) & 16)) emit_collision_event(w, (int)(okey[j] >> 32), (int)(okey[j] & 0xffffffffu), false);   // a touching (or intersecting sensor) pair that leaves the broad phase stops
            clear_color_bits(w, as_int(info.w), as_int(bod.x), as_int(bod.y));
        }
    }
    ctx.grid_sync();
    if (ctx.gtid == 0) {
        st->cur = nxt;
        st->npairs = ncand;
        st->bp_dirty = 0;
        st->bp_ran = 1;
        st->sched_dirty = 1;
        st->ncand = 0;   // (doubles as the colouring's pending counter)
    }
    ctx.grid_sync();
}

// ------------------------------------------------------------------------------------------------
// P2: narrow phase, one thread per pair (process_pair, pair_update.rs:67-680).
// ------------------------------------------------------------------------------------------------
RB_HD float combine_coeff(float c1, float c2, int r1, int r2) {  // coefficient_combine_rule.rs:51-84
    int rule = r1 > r2 ? r1 : r2;
    if (rule == 0) return (c1 + c2) / 2.0f;
    if (rule == 1) return fabsf(min2(c1, c2));
    if (rule == 2) return c1 * c2;
    if (rule == 3) return max2(c1, c2);
    if (rule == 4) return clampf(c1 + c2, 0.0f, 1.0f);
    return sqrtf(max2(c1, 0.0f) * max2(c2, 0.0f));
}

RB_HD float pose_drift(const pose& base, const pose& cur, float max_extent) {  // contact_pair.rs:299-323
    float trans = norm(cur.t - base.t);
    quat d = qmul(cur.q, qconj(base.q));
    float chord = 2.0f * norm(mk3(d.x, d.y, d.z)) * max_extent;
    return trans + chord;
}
RB_HD float rot_cos(quat base, quat cur) {  // contact_pair.rs:284-293
    float c = qdot(base, cur);
    return 2.0f * c * c - 1.0f;
}
RB_HD float origin_radius(const World& w, int shape, vec3 he) {
    if (shape == SHAPE_CONVEX) { const float4 i = w.hulls.info[(int)he.x]; return norm(mk3(i.x + he.y, i.y + he.y, i.z + he.y)); }
    if (shape == SHAPE_CAPSULE) return norm(mk3(he.y, he.x + he.y, he.y));   // corner of the local AABB (the axis only permutes it)
    return shape == SHAPE_BALL ? norm(mk3(he.x, he.x, he.x)) : norm(he);
}

// manifold_reduction.rs:4-84
RB_HD void reduce_manifold(const RawManifold& m, int* sel, int& nsel, float prediction) {
    if (m.n <= 4) return;
    sel[0] = sel[1] = sel[2] = sel[3] = -1;
    float deepest = FMAX32;
    for (int i = 0; i < m.n; ++i)
        if (m.pt[i].dist < deepest) { deepest = m.pt[i].dist; sel[0] = i; }
    if (sel[0] < 0) { nsel = 0; return; }
    vec3 a = m.pt[sel[0]].p1;
    float furthest = -FMAX32;
    for (int i = 0; i < m.n; ++i) {
        float d = norm2(m.pt[i].p1 - a);
        if (i != sel[0] && m.pt[i].dist <= prediction && d > furthest) { furthest = d; sel[1] = i; }
    }
    if (sel[1] < 0) { nsel = 1; return; }
    vec3 b = m.pt[sel[1]].p1;
    if (a.x == b.x && a.y == b.y && a.z == b.z) { nsel = 1; return; }
    vec3 tangent = cross3(b - a, m.n1);
    float mn = FMAX32, mx = -FMAX32;
    for (int i = 0; i < m.n; ++i) {
        if (i == sel[0] || i == sel[1] || m.pt[i].dist > prediction) continue;
        float d = dot3(m.pt[i].p1 - a, tangent);
        if (d < mn) { mn = d; sel[2] = i; }
        if (d > mx) { mx = d; sel[3] = i; }
    }
    if (sel[2] < 0) nsel = 2;
    else if (sel[2] == sel[3]) nsel = 3;
    else nsel = 4;
}

// Polyhedron manifolds (SHAPES = 1 only).  A separating-axis search over two polyhedra is hundreds of candidate axes: one
// thread per pair is a long chain of dependent local-memory traffic however few pairs there are.  So the pairs that will get
// a full manifold this step (same tests as the per-pair loop below: an awake owned body, not recycled) are listed first,
// then each is handed to a whole WARP (consecutive list entries to different CTAs), whose lanes share the candidate axes
// (rb_poly.cuh) with the polyhedra staged in shared memory; the raw manifold goes to a scratch table the per-pair pass reads.
template <class Ctx>
RB_PHASE void phase_convex_manifolds(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int buf = st->cur, np = st->npairs;
    const float prediction = w.prm.prediction;
    const float recycle = w.prm.contact_recycling ? w.prm.recycle_dist : 0.0f;
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        const unsigned long long key = w.pb[buf].key[i];
        const int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
        if (!pair_is_poly_poly(w.c_shape[c1], w.c_shape[c2])) continue;
        const float4 bod0 = prow(w, buf, PR_BODIES, i);
        const int flags = as_int(prow(w, buf, PR_INFO, i).x);
        if (!body_is_sim(w, as_int(bod0.z)) && !body_is_sim(w, as_int(bod0.w)) && !(w.has_filters && !(flags & 64))) continue;
        if (recycle > 0.0f && (flags & 1)) {
            const pose cp1 = collider_pose(w, c1), cp2 = collider_pose(w, c2);
            const pose p12 = pinv_mul(cp1, cp2);
            const float4 rt = prow(w, buf, PR_RT, i);
            const pose base = mkpose(mkq(prow(w, buf, PR_RQ, i)), xyz(rt));
            const float drift = pose_drift(base, p12, rt.w);
            const float rc = min2(rot_cos(mkq(prow(w, buf, PR_ROT1, i)), cp1.q), rot_cos(mkq(prow(w, buf, PR_ROT2, i)), cp2.q));
            if (drift <= prow(w, buf, PR_LN1, i).w && rc > 0.98f) continue;
        }
        w.convex_work[atomic_add(&st->nconvex, 1)] = i;
    }
    ctx.grid_sync();
    RB_SHARED float s_poly[RADIX_MAX_WARPS][3 * 3 * HULL_MAX_VERTS];   // per warp: va, vb, nb
    const int nwork = st->nconvex;
    const int warps_per_block = ctx.bsize / ctx.nlanes < RADIX_MAX_WARPS ? ctx.bsize / ctx.nlanes : RADIX_MAX_WARPS;
    const int warp = ctx.btid / ctx.nlanes;
    if (warp < warps_per_block) {
        vec3* va = reinterpret_cast<vec3*>(s_poly[warp]);
        vec3* vb = va + HULL_MAX_VERTS;
        vec3* nb = vb + HULL_MAX_VERTS;
        for (int k = warp * ctx.nblocks + ctx.bid; k < nwork; k += warps_per_block * ctx.nblocks) {
            const int i = w.convex_work[k];
            const unsigned long long key = w.pb[buf].key[i];
            const int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
            const pose p12 = pinv_mul(collider_pose(w, c1), collider_pose(w, c2));
            PolyLocal l1, l2;
            float r1, r2;
            const Poly A = poly_of_shape(w.hulls, w.c_shape[c1], xyz(w.c_he[c1]), l1, r1);
            const Poly B = poly_of_shape(w.hulls, w.c_shape[c2], xyz(w.c_he[c2]), l2, r2);
            RawManifold raw;
            manifold_poly_poly(ctx.lane, ctx.nlanes, A, r1, B, r2, p12, prediction + (w.c_mat[c1].z + w.c_mat[c2].z), va, vb, nb, raw);
            if (ctx.lane == 0) poly_raw_store(w.convex_raw + (size_t)i * POLY_RAW_STRIDE, raw);
        }
    }
    ctx.grid_sync();
    if (ctx.gtid == 0) st->nconvex = 0;
}

template <int SHAPES = 0, class Ctx>
RB_PHASE void phase_narrow_phase(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int buf = st->cur, np = st->npairs;
    const float prediction = w.prm.prediction, dt = w.prm.dt;
    const float recycle = w.prm.contact_recycling ? w.prm.recycle_dist : 0.0f;
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        unsigned long long key = w.pb[buf].key[i];
        int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
        {   // pairs without an AWAKE body simulated by this rank are not updated: they belong to another rank
            // (multi-GPU sharding) or to a sleeping island, whose bodies do not move
            // (with collider filters, a pair the narrow phase has never updated is updated once whatever its bodies: a pair of two
            // static colliders, or a pair that a filter change brought back under a sleeping body)
            float4 bod0 = prow(w, buf, PR_BODIES, i);
            if (!body_is_sim(w, as_int(bod0.z)) && !body_is_sim(w, as_int(bod0.w)) &&
                !(w.has_filters && !(as_int(prow(w, buf, PR_INFO, i).x) & 64)))
                continue;
        }
        pose cp1 = collider_pose(w, c1), cp2 = collider_pose(w, c2);
        float4 info = prow(w, buf, PR_INFO, i);
        int flags = as_int(info.x), npts_old = as_int(info.y), nsc_old = as_int(info.z), color = as_int(info.w);
        pose p12 = pinv_mul(cp1, cp2);
        bool forceless = false;
        if (w.has_filters) {   // (a kernel parameter: uniform)
            const float4 bodf = prow(w, buf, PR_BODIES, i);
            forceless = pair_forceless(w, c1, c2, as_int(bodf.z), as_int(bodf.w));
        }
        // contact recycling (pair_update.rs:111-171); a pair whose solver outcome changed is recomputed (:116-121)
        if (recycle > 0.0f && (flags & 1) && forceless == ((flags & 32) != 0)) {
            float4 rt = prow(w, buf, PR_RT, i);
            pose base = mkpose(mkq(prow(w, buf, PR_RQ, i)), xyz(rt));
            float drift = pose_drift(base, p12, rt.w);
            float rc = min2(rot_cos(mkq(prow(w, buf, PR_ROT1, i)), cp1.q), rot_cos(mkq(prow(w, buf, PR_ROT2, i)), cp2.q));
            if (drift <= prow(w, buf, PR_LN1, i).w && rc > 0.98f) continue;
        }
        float4 bod = prow(w, buf, PR_BODIES, i);
        int b1 = as_int(bod.z), b2 = as_int(bod.w);
        bool dyn1 = body_is_dyn(w, b1), dyn2 = body_is_dyn(w, b2);
        int sh1 = w.c_shape[c1], sh2 = w.c_shape[c2];
        vec3 he1 = xyz(w.c_he[c1]), he2 = xyz(w.c_he[c2]);
        float4 m1 = w.c_mat[c1], m2 = w.c_mat[c2];
        float skin1 = m1.z, skin2 = m2.z;
        RawManifold raw;
        if (SHAPES && pair_is_poly_poly(sh1, sh2)) poly_raw_load(w.convex_raw + (size_t)i * POLY_RAW_STRIDE, raw);   // (phase_convex_manifolds)
        else contact_manifold<SHAPES>(w.hulls, sh1, he1, sh2, he2, p12, prediction + (skin1 + skin2), raw);

        if (w.has_sensors && ((w.c_events[c1] | w.c_events[c2]) & 4)) {   // (a kernel parameter guards the loads)
            // a pair with a sensor (narrow_phase/intersections.rs:17-221): no contacts, no colour, no island edge -- only whether
            // the shapes intersect (the deepest manifold point is not positive), with a CollisionEvent when that changes
            bool inter = false;
            for (int k = 0; k < raw.n; ++k) inter = inter || raw.pt[k].dist <= 0.0f;
            if (inter != ((flags & 16) != 0)) emit_collision_event(w, c1, c2, inter);
            prow(w, buf, PR_INFO, i) = make_float4(as_float_i((inter ? 16 : 0) | (w.has_filters ? 64 : 0)), as_float_i(0), as_float_i(0), as_float_i(color));
            continue;
        }

        // match_contacts: carry ContactData by feature ids (ball manifolds keep their single point).
        float4 o_pb[MAX_PTS], o_pd[MAX_PTS], o_tw[MAX_PTS], o_d1[MAX_PTS], o_d2[MAX_PTS];
        for (int k = 0; k < MAX_PTS; ++k) {
            if (k < npts_old) {
                o_pb[k] = prow(w, buf, PR_PB + k, i); o_pd[k] = prow(w, buf, PR_PD + k, i);
                o_tw[k] = prow(w, buf, PR_TW + k, i); o_d1[k] = prow(w, buf, PR_DP1 + k, i);
                o_d2[k] = prow(w, buf, PR_DP2 + k, i);
            }
        }
        bool ball = sh1 == SHAPE_BALL || sh2 == SHAPE_BALL;

        int2 rules1 = w.c_rules[c1], rules2 = w.c_rules[c2];
        float friction = combine_coeff(m1.x, m2.x, rules1.x, rules2.x);
        float restitution = combine_coeff(m1.y, m2.y, rules1.y, rules2.y);
        vec3 normal = rotate(cp1.q, raw.n1);

        int sel[4] = {0, 1, 2, 3};
        int nsel = raw.n < MAX_PTS ? raw.n : MAX_PTS;
        reduce_manifold(raw, sel, nsel, prediction);
        if (nsel > 1) {  // planar lexicographic sort (pair_update.rs:433-457)
            vec3 e0, e1;
            ortho_basis(raw.n1, e0, e1);
            float k0[4], k1[4];
            int ks[4];
            for (int q = 0; q < nsel; ++q) {
                vec3 p = raw.pt[sel[q]].p1;
                k0[q] = dot3(p, e0); k1[q] = dot3(p, e1); ks[q] = sel[q];
            }
            for (int q = 1; q < nsel; ++q) {
                float a0 = k0[q], a1 = k1[q];
                int as = ks[q];
                int j = q;
                while (j > 0 && (k0[j - 1] > a0 || (k0[j - 1] == a0 && k1[j - 1] > a1))) {
                    k0[j] = k0[j - 1]; k1[j] = k1[j - 1]; ks[j] = ks[j - 1];
                    --j;
                }
                k0[j] = a0; k1[j] = a1; ks[j] = as;
            }
            for (int q = 0; q < nsel; ++q) sel[q] = ks[q];
        }

        pose com1 = pident(), com2 = pident();
        vec3 lv1 = zero3(), av1 = zero3(), wc1 = zero3(), lv2 = zero3(), av2 = zero3(), wc2 = zero3();
        if (b1 >= 0) { lv1 = xyz(w.b_linvel[b1]); av1 = xyz(w.b_angvel[b1]); wc1 = xyz(w.b_wcom[b1]); }
        if (b2 >= 0) { lv2 = xyz(w.b_linvel[b2]); av2 = xyz(w.b_angvel[b2]); wc2 = xyz(w.b_wcom[b2]); }
        const int rel_dom = relative_dominance(w, b1, b2);
        const bool loc1 = dyn1 && rel_dom <= 0, loc2 = dyn2 && rel_dom >= 0;   // dominance-superior sides keep world anchors (pair_update.rs:538-545)
        if (loc1) com1 = prepend_translation(body_pose(w, b1), xyz(w.b_lcom_im[b1]));
        if (loc2) com2 = prepend_translation(body_pose(w, b2), xyz(w.b_lcom_im[b2]));

        int nsc = 0;
        for (int k = 0; k < nsel; ++k) {
            const RawPt& rp = raw.pt[sel[k]];
            float4 pd = make_float4(0.f, 0.f, 0.f, 0.f), tw = pd, d1 = pd, d2 = pd;
            for (int o = 0; o < npts_old; ++o) {
                if (ball || (as_uint(o_pb[o].w) == rp.fid1 && as_uint(o_pd[o].w) == rp.fid2)) {
                    pd = o_pd[o]; tw = o_tw[o]; d1 = o_d1[o]; d2 = o_d2[o];
                }
            }
            if (forceless) { pd = make_float4(0.f, 0.f, 0.f, 0.f); tw = pd; }   // (no impulse, nothing to warm-start)
            pd.w = as_float(rp.fid2);
            float eff = rp.dist - skin1 - skin2;
            vec3 wp1 = xform(cp1, rp.p1), wp2 = xform(cp2, rp.p2);
            bool keep = eff < prediction;
            if (!keep) {
                vec3 v1 = b1 >= 0 ? lv1 + cross3(av1, wp1 - wc1) : zero3();
                vec3 v2 = b2 >= 0 ? lv2 + cross3(av2, wp2 - wc2) : zero3();
                keep = eff + dot3(v2 - v1, normal) * dt < prediction;
            }
            if (keep) {  // localise + freeze lever arms (pair_update.rs:536-577)
                float shift = dot3(wp2 - wp1, normal) - eff;
                vec3 p1 = wp1 + normal * shift;
                vec3 point = (p1 + wp2) * 0.5f;
                d1 = f4(loc1 ? point - com1.t : point, 0.0f);
                d2 = f4(loc2 ? point - com2.t : point, 0.0f);
                vec3 a1 = loc1 ? xform_inv(com1, p1) : p1;
                vec3 a2 = loc2 ? xform_inv(com2, wp2) : wp2;
                prow(w, buf, PR_A1 + nsc, i) = f4(a1, as_float_i(k));
                prow(w, buf, PR_A2 + nsc, i) = f4(a2, 0.0f);
                ++nsc;
            }
            prow(w, buf, PR_PA + k, i) = f4(rp.p1, rp.dist);
            prow(w, buf, PR_PB + k, i) = f4(rp.p2, as_float(rp.fid1));
            prow(w, buf, PR_PD + k, i) = pd;
            prow(w, buf, PR_TW + k, i) = tw;
            prow(w, buf, PR_DP1 + k, i) = d1;
            prow(w, buf, PR_DP2 + k, i) = d2;
        }
        float max_drift = 0.0f;
        if (recycle > 0.0f) {  // pair_update.rs:582-613
            float max_extent = (flags & 1) ? prow(w, buf, PR_RT, i).w : max2(origin_radius(w, sh1, he1), origin_radius(w, sh2, he2));
            max_drift = nsc > 0 ? recycle : min2(recycle, prediction);
            flags |= 1;
            prow(w, buf, PR_RT, i) = f4(p12.t, max_extent);
            prow(w, buf, PR_RQ, i) = f4(p12.q);
            prow(w, buf, PR_ROT1, i) = f4(cp1.q);
            prow(w, buf, PR_ROT2, i) = f4(cp2.q);
        }
        prow(w, buf, PR_LN1, i) = f4(raw.n1, max_drift);
        prow(w, buf, PR_LN2, i) = f4(raw.n2, restitution);
        prow(w, buf, PR_NORMAL, i) = f4(normal, friction);
        // transitions (pair_update.rs:622-629; contacts.rs:300-385)
        bool had = nsc_old > 0, has = nsc > 0;
        if (has && dyn1 != dyn2) {   // sharding: a contact with a body simulated by ANOTHER rank means two shards' islands merged
            const int bo = dyn1 ? b2 : b1;
            if (bo >= 0 && w.b_type[bo] == BODY_DYNAMIC && w.b_owned[bo] != 1) RB_RAISE(w, -6);
        }
        if (had != has) {
            st->sched_dirty = 1;
            emit_collision_event(w, c1, c2, has);
            if (!has) flags &= ~8;   // the force-event status resets when the colliders separate (geometry/mod.rs:208-217)
            if (has) {
                if (!forceless) {
                    flags |= 2;  // pending colour (deferred greedy pass)
                    st->ntodo = 1;
                }
                // a contact that begins wakes the sleeping side's whole island (narrow_phase/mod.rs:53-67)
                if (dyn1 && w.b_sleeping[b1]) { w.wake_req[w.isl_label[b1]] = 1; st->wake_any = 1; }
                if (dyn2 && w.b_sleeping[b2]) { w.wake_req[w.isl_label[b2]] = 1; st->wake_any = 1; }
            } else {
                clear_color_bits(w, color, as_int(bod.x), as_int(bod.y));
                color = COLOR_UNCOLORED;
                prow(w, buf, PR_BODIES, i) = make_float4(as_float_i(-1), as_float_i(-1), bod.z, bod.w);
            }
        }
        if (w.has_filters) {
            if (had && has && forceless != ((flags & 32) != 0)) {   // a touching pair gains or loses its forces: recolour, reschedule
                st->sched_dirty = 1;
                if (forceless) {
                    clear_color_bits(w, color, as_int(bod.x), as_int(bod.y));
                    color = COLOR_UNCOLORED;
                    flags &= ~8;
                    prow(w, buf, PR_BODIES, i) = make_float4(as_float_i(-1), as_float_i(-1), bod.z, bod.w);
                } else {
                    flags |= 2;
                    st->ntodo = 1;
                }
            }
            flags = (forceless ? (flags | 32) : (flags & ~32)) | 64;
        }
        prow(w, buf, PR_INFO, i) = make_float4(as_float_i(flags), as_float_i(nsel), as_float_i(nsc), as_float_i(color));
    }
}

// ------------------------------------------------------------------------------------------------
// P3a: deferred greedy colouring of the pairs that began touching, in the reference's canonical order
// (min body, max body, edge) (contacts.rs:366-385; narrow_phase/mod.rs:87-152) -- body = arena index of the
// collider's parent (fixed bodies included), u32::MAX for a parentless collider; the edge index, which only
// orders pairs between the SAME two bodies, is replaced by the pair-table index (ascending collider pair).
// Parallel formulation of the sequential greedy: a pending pair is coloured in the round where it is the
// first pending pair, in that order, on each of its dynamic bodies -- which reproduces the sequential result
// exactly.  Two-level minimum per body: the smallest order key, then the smallest pair index with that key.
// ------------------------------------------------------------------------------------------------
RB_HD int first_free_low(const unsigned* m) {   // lowest clear bit in 0..119, else 128
    for (int wd = 0; wd < 4; ++wd) {
        unsigned inv = ~m[wd];
        if (wd == 3) inv &= 0x00ffffffu;  // colours 96..119 only
        if (inv) {
            int b = 0;
            while (!((inv >> b) & 1u)) ++b;
            return wd * 32 + b;
        }
    }
    return 128;
}
RB_HD int first_free_high(const unsigned* m) {  // highest clear bit <= 127, else 128
    for (int wd = 3; wd >= 0; --wd) {
        unsigned inv = ~m[wd];
        if (inv) {
            int b = 31;
            while (!((inv >> b) & 1u)) --b;
            return wd * 32 + b;
        }
    }
    return 128;
}
RB_HD unsigned long long color_order_key(int b1, int b2) {
    const unsigned a = b1 < 0 ? 0xffffffffu : (unsigned)b1, b = b2 < 0 ? 0xffffffffu : (unsigned)b2;
    return ((unsigned long long)(a < b ? a : b) << 32) | (a < b ? b : a);
}

template <class Ctx>
RB_PHASE void section_coloring(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int buf = st->cur, np = st->npairs;
    // the pairs awaiting a colour, listed once (cons_pair_tmp is free until the schedule): the bidding rounds below walk
    // this list, not the whole pair table (a settling pile runs dozens of rounds over a few thousand pending pairs)
    int* list = w.cons_pair_tmp;
    for (int i = ctx.gtid; i < np; i += ctx.gsize)
        if (as_int(prow(w, buf, PR_INFO, i).x) & 2) list[atomic_add(&st->ncand, 1)] = i;   // (ncand: 0 outside the broad phase)
    ctx.grid_sync();
    const int nlist = st->ncand < w.cons_cap ? st->ncand : w.cons_cap;
    ctx.grid_sync();
    if (ctx.gtid == 0) st->ncand = 0;
    ctx.grid_sync();
    for (;;) {
        // A1: every pending pair bids its order key for its dynamic bodies
        for (int k = ctx.gtid; k < nlist; k += ctx.gsize) {
            const int i = list[k];
            int flags = as_int(prow(w, buf, PR_INFO, i).x);
            if (!(flags & 2)) continue;
            float4 bod = prow(w, buf, PR_BODIES, i);
            int b1 = as_int(bod.z), b2 = as_int(bod.w);
            const unsigned long long key = color_order_key(b1, b2);
            if (body_is_dyn(w, b1)) atomic_min64(&w.body_minkey[b1], key);
            if (body_is_dyn(w, b2)) atomic_min64(&w.body_minkey[b2], key);
            st->ncand = 1;   // some pair is still pending (a flag: every writer stores the same value)
        }
        ctx.grid_sync();
        int pending = st->ncand;
        if (pending == 0) break;
        // A2: among the pairs holding a body's smallest key, the lowest pair index
        for (int k = ctx.gtid; k < nlist; k += ctx.gsize) {
            const int i = list[k];
            int flags = as_int(prow(w, buf, PR_INFO, i).x);
            if (!(flags & 2)) continue;
            float4 bod = prow(w, buf, PR_BODIES, i);
            int b1 = as_int(bod.z), b2 = as_int(bod.w);
            const unsigned long long key = color_order_key(b1, b2);
            if (body_is_dyn(w, b1) && w.body_minkey[b1] == key) atomic_min(&w.body_min[b1], i);
            if (body_is_dyn(w, b2) && w.body_minkey[b2] == key) atomic_min(&w.body_min[b2], i);
        }
        ctx.grid_sync();
        // B: winners take the first colour free on both bodies
        for (int k = ctx.gtid; k < nlist; k += ctx.gsize) {
            const int i = list[k];
            float4 info = prow(w, buf, PR_INFO, i);
            int flags = as_int(info.x);
            if (!(flags & 2)) continue;
            float4 bod = prow(w, buf, PR_BODIES, i);
            int b1 = as_int(bod.z), b2 = as_int(bod.w);
            bool d1 = body_is_dyn(w, b1), d2 = body_is_dyn(w, b2);
            if ((d1 && w.body_min[b1] != i) || (d2 && w.body_min[b2] != i)) continue;
            int color = COLOR_OVERFLOW, cb0 = -1, cb1 = -1;
            if (d1 && d2) {
                unsigned m[4];
                for (int k2 = 0; k2 < 4; ++k2) m[k2] = w.color_mask[b1 * 4 + k2] | w.color_mask[b2 * 4 + k2];
                int c = first_free_low(m);
                if (c < 128) { color = c; cb0 = b1; cb1 = b2; }
            } else if (d1 || d2) {
                int b = d1 ? b1 : b2;
                int c = first_free_high(&w.color_mask[b * 4]);
                if (c < 128) { color = c; cb0 = b; }
            }
            if (color < 128) {
                if (cb0 >= 0) w.color_mask[cb0 * 4 + (color >> 5)] |= 1u << (color & 31);
                if (cb1 >= 0) w.color_mask[cb1 * 4 + (color >> 5)] |= 1u << (color & 31);
            }
            prow(w, buf, PR_BODIES, i) = make_float4(as_float_i(cb0), as_float_i(cb1), bod.z, bod.w);
            info.x = as_float_i((flags & ~2) | 4);  // bit2: coloured this round (scratch reset below)
            info.w = as_float_i(color);
            prow(w, buf, PR_INFO, i) = info;
        }
        ctx.grid_sync();
        // C: reset the bidding scratch
        for (int k = ctx.gtid; k < nlist; k += ctx.gsize) {
            const int i = list[k];
            float4 info = prow(w, buf, PR_INFO, i);
            int flags = as_int(info.x);
            if (!(flags & 6)) continue;
            float4 bod = prow(w, buf, PR_BODIES, i);
            int b1 = as_int(bod.z), b2 = as_int(bod.w);
            if (body_is_dyn(w, b1)) { w.body_min[b1] = 0x7fffffff; w.body_minkey[b1] = ~0ull; }
            if (body_is_dyn(w, b2)) { w.body_min[b2] = 0x7fffffff; w.body_minkey[b2] = ~0ull; }
            if (flags & 4) { info.x = as_float_i(flags & ~4); prow(w, buf, PR_INFO, i) = info; }
        }
        if (ctx.gtid == 0) st->ncand = 0;
        ctx.grid_sync();
    }
    if (ctx.gtid == 0) st->ntodo = 0;
    ctx.grid_sync();
}

// ------------------------------------------------------------------------------------------------
// Grid-wide exclusive scan of ints: per-thread chunks, a shared-memory scan of the partial sums inside every CTA, then
// every CTA adds up the totals of the CTAs before it (no serial pass of one CTA over all the partials: that
// serialises the scan).  `tmp` needs gsize + 1 entries.  Returns the total in tmp[gsize].
// ------------------------------------------------------------------------------------------------
template <class Ctx>
RB_PHASE void grid_exclusive_scan(const Ctx& ctx, const int* in, int* out, int n, int* tmp) {
    RB_SHARED int s_part[1024];
    RB_SHARED int s_base;
    int chunk = (n + ctx.gsize - 1) / ctx.gsize;
    int b = ctx.gtid * chunk, e = b + chunk < n ? b + chunk : n;
    int s = 0;
    for (int i = b; i < e; ++i) s += in[i];
    // inclusive scan of the per-thread sums within the CTA (Hillis-Steele)
    s_part[ctx.btid] = s;
    ctx.block_sync();
    for (int off = 1; off < ctx.bsize; off <<= 1) {
        const int v = ctx.btid >= off ? s_part[ctx.btid - off] : 0;
        ctx.block_sync();
        s_part[ctx.btid] += v;
        ctx.block_sync();
    }
    const int excl = s_part[ctx.btid] - s;
    if (ctx.btid == ctx.bsize - 1) tmp[ctx.bid] = s_part[ctx.btid];   // the CTA's total
    ctx.grid_sync();
    // what the CTAs before this one hold (and, by the last CTA, the grand total)
    int before = 0;
    for (int k = ctx.btid; k < ctx.bid; k += ctx.bsize) before += tmp[k];
    ctx.block_sync();   // (s_part is reused)
    s_part[ctx.btid] = before;
    ctx.block_sync();
    for (int off = ctx.bsize >> 1; off > 0; off >>= 1) {
        if (ctx.btid < off) s_part[ctx.btid] += s_part[ctx.btid + off];
        ctx.block_sync();
    }
    if (ctx.btid == 0) {
        s_base = s_part[0];
        if (ctx.bid == ctx.nblocks - 1) tmp[ctx.gsize] = s_part[0] + tmp[ctx.bid];
    }
    ctx.block_sync();
    int run = s_base + excl;
    for (int i = b; i < e; ++i) { int v = in[i]; out[i] = run; run += v; }
    ctx.grid_sync();
}

// Concurrent union-find (hook the larger root under the smaller one; find with path HALVING).
// Invariant: parent[y] <= y for every y, so no cycle can form; every value a racing thread may
// store into parent[cur] is an ancestor of cur that is smaller than cur.
RB_HD int uf_find(int* parent, int x) {
    int cur = x;
    for (;;) {
        int next = parent[cur];
        if (next == cur) return cur;
        int gp = parent[next];
        if (gp != next) parent[cur] = gp;   // gp < next < cur
        cur = next;
    }
}
// Read-only find (no path halving): used by the flatten pass, whose in-place root writes must not be
// overwritten by another thread's stale halving store.
RB_HD int uf_find_ro(const int* parent, int x) {
    int cur = x;
    for (;;) {
        int next = parent[cur];
        if (next == cur) return cur;
        cur = next;
    }
}
RB_HD void uf_union(int* parent, int a, int b) {  // hook the larger root under the smaller one
    for (;;) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        int lo = a < b ? a : b, hi = a < b ? b : a;
        int old = atomic_cas(&parent[hi], hi, lo);
        if (old == hi) return;
    }
}

// P3b: connected components (persistent islands, island_manager/persistent.rs:1-3), work items,
// colour stage order (init.rs:163-254) and the per-item constraint schedule.
// Connected components over ALL dynamic bodies of this rank, awake or asleep (a sleeping island keeps its label, so
// that a contact with any of its bodies can wake all of them).
template <class Ctx>
RB_PHASE void section_components(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int buf = st->cur, np = st->npairs, nb = w.nb, nj = w.nj;
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) w.isl_label[b] = b;
    ctx.grid_sync();
    // union over touching dynamic-dynamic pairs and joints
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        if (as_int(prow(w, buf, PR_INFO, i).z) <= 0) continue;
        float4 bod = prow(w, buf, PR_BODIES, i);
        int b1 = as_int(bod.z), b2 = as_int(bod.w);
        // Two touching kinematic bodies are no island edge.  A touching pair whose solver groups fail still is one, as the
        // reference links islands over every pair with an active contact whatever its solver flags (substep_groups.rs:73-87).
        if (body_is_dyn(w, b1) && body_is_dyn(w, b2) && !(w.has_filters && w.b_type[b1] != BODY_DYNAMIC && w.b_type[b2] != BODY_DYNAMIC))
            uf_union(w.isl_label, b1, b2);
    }
    for (int j = ctx.gtid; j < nj; j += ctx.gsize) {
        int4 ji = w.j_info[j];
        if (body_is_dyn(w, ji.x) && body_is_dyn(w, ji.y)) uf_union(w.isl_label, ji.x, ji.y);
    }
    ctx.grid_sync();
    // flatten
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) w.isl_label[b] = uf_find_ro(w.isl_label, b);
    ctx.grid_sync();
}

// ------------------------------------------------------------------------------------------------
// Sleeping (island_manager/sleep.rs, manager.rs:320-392; RigidBodyActivation::update_energy,
// rigid_body_components.rs:1417-1470).  Whole islands only: an island falls asleep when EVERY body in it has been
// below the motion threshold for time_until_sleep, and a contact that begins with one of its bodies wakes all of them.
// ------------------------------------------------------------------------------------------------
constexpr float SLEEP_LINEAR_THRESHOLD = 0.05f, SLEEP_ANGULAR_THRESHOLD = 0.5f, SLEEP_TIME_UNTIL = 0.5f;

template <class Ctx>
RB_PHASE void section_wake(const Ctx& ctx, const World& w) {
    State* st = w.st;
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize)
        if (body_is_dyn(w, b) && w.b_sleeping[b] && w.wake_req[w.isl_label[b]]) {
            w.b_sleeping[b] = 0;
            w.b_sleep_time[b] = 0.0f;   // "strong" wake-up: the timer restarts
            st->sched_dirty = 1;
        }
    ctx.grid_sync();
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize) w.wake_req[b] = 0;
    if (ctx.gtid == 0) st->wake_any = 0;
    ctx.grid_sync();
}

template <class Ctx>
RB_PHASE void section_sleep(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int stamp = st->sleep_stamp;
    const float dt = w.prm.dt, linear_threshold = SLEEP_LINEAR_THRESHOLD * w.prm.length_unit;
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize) {
        if (!body_is_sim(w, b)) continue;
        const bool may = !(w.b_flags[b] & FLAG_NO_SLEEP);
        const pose cur = body_pose(w, b);
        const pose prev = mkpose(mkq(w.b_sleep_prev_q[b]), xyz(w.b_sleep_prev_t[b]));
        w.b_sleep_prev_t[b] = f4(cur.t, 0.0f);
        w.b_sleep_prev_q[b] = f4(cur.q);
        const vec3 av = xyz(w.b_angvel[b]);
        const float sq_angvel = dot3(av, av), ext = w.b_max_extent[b];
        const bool angular_ok = ext > 0.0f ? (may && sq_angvel < 1.5707963267948966f * 1.5707963267948966f)
                                           : (may && sq_angvel < SLEEP_ANGULAR_THRESHOLD * SLEEP_ANGULAR_THRESHOLD);
        const float drift = pose_drift(prev, cur, ext);
        bool can = may && angular_ok && drift * 0.5f < linear_threshold * dt;
        if (w.b_type[b] != BODY_DYNAMIC) {   // platforms only sleep while both velocities are exactly zero (:1457-1461)
            const vec3 lv = xyz(w.b_linvel[b]);
            can = may && dot3(lv, lv) == 0.0f && sq_angvel == 0.0f;
        }
        const float t = can ? w.b_sleep_time[b] + dt : 0.0f;
        w.b_sleep_time[b] = t;
        if (!(t >= SLEEP_TIME_UNTIL)) w.isl_block[w.isl_label[b]] = stamp;   // one restless body keeps its island awake
    }
    ctx.grid_sync();
    for (int b = ctx.gtid; b < w.nb; b += ctx.gsize) {
        if (!body_is_sim(w, b) || w.isl_block[w.isl_label[b]] == stamp) continue;
        w.b_sleeping[b] = 1;                  // RigidBody::sleep (rigid_body.rs:804-807)
        w.b_sleep_time[b] = SLEEP_TIME_UNTIL;
        w.b_linvel[b] = make_float4(0.f, 0.f, 0.f, 0.f);
        w.b_angvel[b] = make_float4(0.f, 0.f, 0.f, 0.f);
        float* s13 = w.state13 + (size_t)b * 13;
        for (int k = 7; k < 13; ++k) s13[k] = 0.0f;
        st->sched_dirty = 1;
    }
    ctx.grid_sync();
}

// P3b: work items, colour stage order (init.rs:163-254) and the per-item constraint schedule of the AWAKE islands.
template <class Ctx>
RB_PHASE void section_schedule(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int buf = st->cur, np = st->npairs, nb = w.nb, nj = w.nj;
    // S1 reset
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) { w.isl_nb[b] = 0; w.isl_ncons[b] = 0; w.isl_item[b] = -1; }
    if (w.any_extra)
        for (int b = ctx.gtid; b < nb; b += ctx.gsize) w.isl_key[b] = 0u;
    for (int c = ctx.gtid; c < NUM_COLORS; c += ctx.gsize) w.color_count[c] = 0;
    for (int i = ctx.gtid; i < 3 * (w.item_cap + 1); i += ctx.gsize) w.item_cursor[i] = 0;
    for (int i = ctx.gtid; i <= w.item_cap; i += ctx.gsize) { w.item_body_start[i] = 0; w.item_cons_start[i] = 0; w.item_joint_start[i] = 0; }
    ctx.grid_sync();
    RB_CSTAMP(7);
    // S4 per-root counts + global colour histogram
    for (int b = ctx.gtid; b < nb; b += ctx.gsize)
        if (body_is_sim(w, b)) atomic_add(&w.isl_nb[w.isl_label[b]], 1);
    // substep solve-groups (island_manager/substep_groups.rs:107-123): an island's key = the largest
    // additional_solver_iterations among its members (bits 24..31 of the body flags)
    if (w.any_extra)
        for (int b = ctx.gtid; b < nb; b += ctx.gsize) {
            const unsigned extra = w.b_flags[b] >> 24;
            if (extra != 0u && body_is_sim(w, b)) atomic_max_u(&w.isl_key[w.isl_label[b]], extra);
        }
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        float4 info = prow(w, buf, PR_INFO, i);
        if (as_int(info.z) <= 0 || (w.has_filters && (as_int(info.x) & 32))) continue;   // (forceless pairs are no constraint)
        float4 bod = prow(w, buf, PR_BODIES, i);
        int b1 = as_int(bod.z), b2 = as_int(bod.w);
        int b = body_is_sim(w, b1) ? b1 : (body_is_sim(w, b2) ? b2 : -1);
        if (b < 0) continue;
        atomic_add(&w.isl_ncons[w.isl_label[b]], 1);
        int color = as_int(info.w);
        atomic_add(&w.color_count[color > COLOR_OVERFLOW ? COLOR_OVERFLOW : color], 1);
    }
    for (int j = ctx.gtid; j < nj; j += ctx.gsize) {
        int4 ji = w.j_info[j];
        int b = body_is_sim(w, ji.x) ? ji.x : (body_is_sim(w, ji.y) ? ji.y : -1);
        if (b >= 0) atomic_add(&w.isl_ncons[w.isl_label[b]], 1);
    }
    ctx.grid_sync();
    RB_CSTAMP(8);
    // S5 colour stage order: big colours ascending, then small colours ascending, then overflow.  One CTA, a thread per
    // colour ranking itself against a shared copy of the counts (a single thread walking global memory is far slower).
    if (ctx.bid == 0) {
        RB_SHARED int s_cnt[NUM_COLORS];
        for (int c = ctx.btid; c < NUM_COLORS; c += ctx.bsize) s_cnt[c] = w.color_count[c];
        ctx.block_sync();
        for (int c = ctx.btid; c < NUM_COLORS; c += ctx.bsize) {
            const int n = s_cnt[c];
            int nbig = 0, nsmall = 0, before = 0;
            const bool big = n >= BIG_COLOR_MIN;
            for (int k = 0; k < 128; ++k) {
                const int nk = s_cnt[k];
                if (nk == 0) continue;
                const bool kb = nk >= BIG_COLOR_MIN;
                if (kb) ++nbig; else ++nsmall;
                if (k < c && kb == big) ++before;
            }
            int p = -1;
            if (c < 128) { if (n > 0) p = big ? before : nbig + before; }
            else {
                if (n > 0) p = nbig + nsmall;
                st->nused_colors = nbig + nsmall + (n > 0 ? 1 : 0);
            }
            w.color_pos[c] = p;
        }
    }
    RB_CSTAMP(9);
    // S6 work items: exclusive prefix of the cost of the small islands in root order.
    int* cost = w.isl_item;  // reuse as input, overwritten by the item id below
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) {
        int c = 0;
        if (body_is_sim(w, b) && w.isl_label[b] == b) {
            int nbod = w.isl_nb[b], ncon = w.isl_ncons[b];
            bool large = nbod > ITEM_BODY_CAP || ncon > ITEM_CONS_CAP;
            c = large ? 0 : (nbod > ncon ? nbod : ncon);
        }
        cost[b] = c;
    }
    ctx.grid_sync();
    grid_exclusive_scan(ctx, cost, w.body_item, nb, w.scan_tmp);  // body_item temporarily holds the prefix
    int total_cost = w.scan_tmp[ctx.gsize];
    int nitems = 1 + (total_cost + ITEM_TARGET - 1) / ITEM_TARGET;
    if (nitems > w.item_cap) {
        if (ctx.gtid == 0) RB_RAISE(w, -4);
        nitems = w.item_cap;
    }
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) {
        int it = -1;
        if (body_is_sim(w, b) && w.isl_label[b] == b) {
            int nbod = w.isl_nb[b], ncon = w.isl_ncons[b];
            bool large = nbod > ITEM_BODY_CAP || ncon > ITEM_CONS_CAP;
            it = large ? 0 : 1 + w.body_item[b] / ITEM_TARGET;
            if (it >= nitems) it = nitems - 1;
        }
        w.isl_item[b] = it;
    }
    ctx.grid_sync();
    RB_CSTAMP(10);
    // S7 per-item counts
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) {
        int it = body_is_sim(w, b) ? w.isl_item[w.isl_label[b]] : -1;
        w.body_item[b] = it;
        if (it >= 0) atomic_add(&w.item_body_start[it], 1);
        if (w.any_extra) w.b_key[b] = (unsigned char)(it >= 0 ? w.isl_key[w.isl_label[b]] : 0u);
    }
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        const float4 info = prow(w, buf, PR_INFO, i);
        if (as_int(info.z) <= 0 || (w.has_filters && (as_int(info.x) & 32))) continue;
        float4 bod = prow(w, buf, PR_BODIES, i);
        int b1 = as_int(bod.z), b2 = as_int(bod.w);
        int b = body_is_sim(w, b1) ? b1 : (body_is_sim(w, b2) ? b2 : -1);
        if (b >= 0) atomic_add(&w.item_cons_start[w.isl_item[w.isl_label[b]]], 1);
    }
    for (int j = ctx.gtid; j < nj; j += ctx.gsize) {
        int4 ji = w.j_info[j];
        int b = body_is_sim(w, ji.x) ? ji.x : (body_is_sim(w, ji.y) ? ji.y : -1);
        if (b >= 0) atomic_add(&w.item_joint_start[w.isl_item[w.isl_label[b]]], 1);
    }
    ctx.grid_sync();
    RB_CSTAMP(11);
    // S8 scans (counts -> starts); entry [nitems] becomes the total.
    grid_exclusive_scan(ctx, w.item_body_start, w.item_body_start, nitems + 1, w.scan_tmp);
    grid_exclusive_scan(ctx, w.item_cons_start, w.item_cons_start, nitems + 1, w.scan_tmp);
    grid_exclusive_scan(ctx, w.item_joint_start, w.item_joint_start, nitems + 1, w.scan_tmp);
    int ncons = w.item_cons_start[nitems];
    if (ncons > w.cons_cap) {
        if (ctx.gtid == 0) RB_RAISE(w, -4);
    }
    RB_CSTAMP(12);
    // S9 scatter bodies / manifolds / joints into their item segments
    int* cur_b = w.item_cursor;
    int* cur_c = w.item_cursor + (w.item_cap + 1);
    int* cur_j = w.item_cursor + 2 * (w.item_cap + 1);
    for (int b = ctx.gtid; b < nb; b += ctx.gsize) {
        int it = w.body_item[b];
        if (it < 0) { w.body_local[b] = -1; continue; }
        int l = atomic_add(&cur_b[it], 1);
        w.item_bodies[w.item_body_start[it] + l] = b;
        w.body_local[b] = l;
    }
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        const float4 info = prow(w, buf, PR_INFO, i);
        if (as_int(info.z) <= 0 || (w.has_filters && (as_int(info.x) & 32))) continue;
        float4 bod = prow(w, buf, PR_BODIES, i);
        int b1 = as_int(bod.z), b2 = as_int(bod.w);
        int b = body_is_sim(w, b1) ? b1 : (body_is_sim(w, b2) ? b2 : -1);
        if (b < 0) continue;
        int it = w.body_item[b];
        int l = atomic_add(&cur_c[it], 1);
        int pos = w.item_cons_start[it] + l;
        if (pos < w.cons_cap) w.cons_pair_tmp[pos] = i;
    }
    for (int j = ctx.gtid; j < nj; j += ctx.gsize) {
        int4 ji = w.j_info[j];
        int b = body_is_sim(w, ji.x) ? ji.x : (body_is_sim(w, ji.y) ? ji.y : -1);
        if (b < 0) continue;
        int it = w.body_item[b];
        int l = atomic_add(&cur_j[it], 1);
        w.joint_tmp[w.item_joint_start[it] + l] = j;
    }
    ctx.grid_sync();
    RB_CSTAMP(13);
    // S10a item 0 (the grid-wide islands: up to every constraint of the world) is sorted by colour stage by the WHOLE grid:
    // per-CTA histograms of contiguous chunks, totals and per-CTA bases through global atomics, scatter.  The order inside
    // a colour is arbitrary here as in S10 (constraints of one colour share no body); the overflow colour is put in index
    // order afterwards.  One CTA alone is too slow for the 30 000 - 70 000 constraints of keva / pyramid3.
    for (int pass = 0; pass < 2; ++pass) {   // 0: contacts, 1: joints
        RB_SHARED int hist0[NUM_COLORS + 1];
        RB_SHARED int offs0[NUM_COLORS + 1];
        RB_SHARED int base0[NUM_COLORS + 1];
        RB_SHARED int curs0[NUM_COLORS + 1];
        const int* starts = pass == 0 ? w.item_cons_start : w.item_joint_start;
        const int s0 = starts[0];
        int s1 = starts[1];
        if (pass == 0 && s1 > w.cons_cap) s1 = s0 > w.cons_cap ? s0 : w.cons_cap;
        const int* src = pass == 0 ? w.cons_pair_tmp : w.joint_tmp;
        int* dst = pass == 0 ? w.cons_pair : w.joint_sched;
        int* offs = pass == 0 ? w.item_color_off : w.item_jcolor_off;   // (item 0's row)
        const int* cpos = pass == 0 ? w.color_pos : w.jcolor_pos;
        int* ghist = w.order_hist;                       // [NUM_COLORS + 1] totals   (order_hist is free until S11)
        int* gcurs = w.order_hist + (NUM_COLORS + 1);    // [NUM_COLORS + 1] running bases of the CTAs
        if (s1 <= s0) {   // (uniform) nothing in item 0: an empty colour table
            for (int c = ctx.gtid; c <= NUM_COLORS; c += ctx.gsize) offs[c] = 0;
            continue;
        }
        for (int c = ctx.gtid; c < 2 * (NUM_COLORS + 1); c += ctx.gsize) ghist[c] = 0;
        for (int c = ctx.btid; c <= NUM_COLORS; c += ctx.bsize) { hist0[c] = 0; curs0[c] = 0; }
        ctx.grid_sync();
        const int n0 = s1 - s0;
        const int chunk = (n0 + ctx.nblocks - 1) / ctx.nblocks;
        const int q0 = s0 + ctx.bid * chunk, q1 = q0 + chunk < s1 ? q0 + chunk : s1;
        for (int q = q0 + ctx.btid; q < q1; q += ctx.bsize) {
            const int id = src[q];
            int color = pass == 0 ? as_int(prow(w, buf, PR_INFO, id).w) : w.j_info[id].w;
            if (color > COLOR_OVERFLOW) color = COLOR_OVERFLOW;
            atomic_add(&hist0[cpos[color]], 1);
        }
        ctx.block_sync();
        for (int c = ctx.btid; c < NUM_COLORS; c += ctx.bsize)
            if (hist0[c] > 0) atomic_add(&ghist[c], hist0[c]);
        ctx.grid_sync();
        for (int c = ctx.btid; c < NUM_COLORS; c += ctx.bsize) {
            offs0[c] = ghist[c];                                              // totals (prefix below)
            base0[c] = hist0[c] > 0 ? atomic_add(&gcurs[c], hist0[c]) : 0;    // where this CTA's share of the colour starts
        }
        ctx.block_sync();
        if (ctx.btid == 0) {
            int run = 0;
            for (int c = 0; c <= NUM_COLORS; ++c) { const int v = c < NUM_COLORS ? offs0[c] : 0; offs0[c] = run; run += v; }
        }
        ctx.block_sync();
        if (ctx.bid == 0)
            for (int c = ctx.btid; c <= NUM_COLORS; c += ctx.bsize) offs[c] = offs0[c];
        for (int q = q0 + ctx.btid; q < q1; q += ctx.bsize) {
            const int id = src[q];
            int color = pass == 0 ? as_int(prow(w, buf, PR_INFO, id).w) : w.j_info[id].w;
            if (color > COLOR_OVERFLOW) color = COLOR_OVERFLOW;
            const int p = cpos[color];
            dst[s0 + offs0[p] + base0[p] + atomic_add(&curs0[p], 1)] = id;
        }
        ctx.grid_sync();
        if (ctx.gtid == 0 && cpos[COLOR_OVERFLOW] >= 0) {   // the overflow colour is solved sequentially: order it by index
            const int p = cpos[COLOR_OVERFLOW];
            const int a = s0 + offs0[p], e = s0 + offs0[p + 1];
            for (int x = a + 1; x < e; ++x) {
                int v = dst[x], y = x;
                while (y > a && dst[y - 1] > v) { dst[y] = dst[y - 1]; --y; }
                dst[y] = v;
            }
        }
        ctx.grid_sync();
        for (int q = s0 + ctx.gtid; q < s1; q += ctx.gsize) {   // headers (item 0: global body ids)
            const int id = dst[q];
            int b1, b2;
            if (pass == 0) {
                const float4 bod = prow(w, buf, PR_BODIES, id);
                b1 = as_int(bod.z); b2 = as_int(bod.w);
            } else {
                const int4 ji = w.j_info[id];
                b1 = ji.x; b2 = ji.y;
            }
            int id1 = body_is_sim(w, b1) ? b1 : NO_BODY;
            int id2 = body_is_sim(w, b2) ? b2 : NO_BODY;
            if (w.any_extra) (pass == 0 ? w.cons_key : w.j_key)[q] = w.b_key[id1 != NO_BODY ? b1 : b2];   // (both ends share the island)
            if (pass == 0) {   // contact_with_twist_friction.rs:71-84
                const int rel_dom = relative_dominance(w, b1, b2);
                if (rel_dom > 0) id1 = NO_BODY;
                if (rel_dom < 0) id2 = NO_BODY;
                w.cons_hdr[q] = make_int4(id, id1, id2, 0);
            } else {
                w.j_sched_ids[q] = make_int4(id, id1, id2, 0);
            }
        }
        ctx.grid_sync();
    }
    // S10 per-item counting sort by colour stage (one CTA per item), headers for the solver.
    for (int it = 1 + ctx.bid; it < nitems; it += ctx.nblocks) {
        RB_SHARED int hist[NUM_COLORS + 1];
        RB_SHARED int curs[NUM_COLORS + 1];
        for (int pass = 0; pass < 2; ++pass) {  // 0: contacts, 1: joints
            const int* starts = pass == 0 ? w.item_cons_start : w.item_joint_start;
            int s0 = starts[it], s1 = starts[it + 1];
            if (pass == 0 && s1 > w.cons_cap) s1 = s0 > w.cons_cap ? s0 : w.cons_cap;
            const int* src = pass == 0 ? w.cons_pair_tmp : w.joint_tmp;
            int* dst = pass == 0 ? w.cons_pair : w.joint_sched;
            int* offs = (pass == 0 ? w.item_color_off : w.item_jcolor_off) + (size_t)it * (NUM_COLORS + 1);
            const int* cpos = pass == 0 ? w.color_pos : w.jcolor_pos;
            for (int c = ctx.btid; c <= NUM_COLORS; c += ctx.bsize) { hist[c] = 0; curs[c] = 0; }
            ctx.block_sync();
            for (int q = s0 + ctx.btid; q < s1; q += ctx.bsize) {
                int id = src[q];
                int color = pass == 0 ? as_int(prow(w, buf, PR_INFO, id).w) : w.j_info[id].w;
                if (color > COLOR_OVERFLOW) color = COLOR_OVERFLOW;
                atomic_add(&hist[cpos[color]], 1);
            }
            ctx.block_sync();
            if (ctx.btid == 0) {
                int run = 0;
                for (int c = 0; c <= NUM_COLORS; ++c) { int v = c < NUM_COLORS ? hist[c] : 0; hist[c] = run; offs[c] = run; run += v; }
            }
            ctx.block_sync();
            for (int q = s0 + ctx.btid; q < s1; q += ctx.bsize) {
                int id = src[q];
                int color = pass == 0 ? as_int(prow(w, buf, PR_INFO, id).w) : w.j_info[id].w;
                if (color > COLOR_OVERFLOW) color = COLOR_OVERFLOW;
                int p = cpos[color];
                int l = atomic_add(&curs[p], 1);
                dst[s0 + hist[p] + l] = id;
            }
            ctx.block_sync();
            // the overflow colour is solved sequentially: order it by index
            if (ctx.btid == 0 && cpos[COLOR_OVERFLOW] >= 0) {
                int p = cpos[COLOR_OVERFLOW];
                int a = s0 + offs[p], e = s0 + offs[p + 1];
                for (int x = a + 1; x < e; ++x) {
                    int v = dst[x], y = x;
                    while (y > a && dst[y - 1] > v) { dst[y] = dst[y - 1]; --y; }
                    dst[y] = v;
                }
            }
            ctx.block_sync();
            // headers
            for (int q = s0 + ctx.btid; q < s1; q += ctx.bsize) {
                int id = dst[q];
                int b1, b2;
                if (pass == 0) {
                    float4 bod = prow(w, buf, PR_BODIES, id);
                    b1 = as_int(bod.z); b2 = as_int(bod.w);
                } else {
                    int4 ji = w.j_info[id];
                    b1 = ji.x; b2 = ji.y;
                }
                int id1 = body_is_sim(w, b1) ? (it == 0 ? b1 : w.body_local[b1]) : NO_BODY;
                int id2 = body_is_sim(w, b2) ? (it == 0 ? b2 : w.body_local[b2]) : NO_BODY;
                if (w.any_extra) (pass == 0 ? w.cons_key : w.j_key)[q] = w.b_key[id1 != NO_BODY ? b1 : b2];
                if (pass == 0) {   // contact_with_twist_friction.rs:71-84
                    const int rel_dom = relative_dominance(w, b1, b2);
                    if (rel_dom > 0) id1 = NO_BODY;
                    if (rel_dom < 0) id2 = NO_BODY;
                }
                if (pass == 0) w.cons_hdr[q] = make_int4(id, id1, id2, 0);
                else w.j_sched_ids[q] = make_int4(id, id1, id2, 0);
            }
            ctx.block_sync();
            // per-body adjacency of the contact constraints, in stage (= slot) order: entry = slot * 2 + side.
            // The body-centric warm start of the shared-memory items walks it (rb_solver.cuh).
            if (pass == 0 && it > 0) {
                const int lb0 = w.item_body_start[it], lb1 = w.item_body_start[it + 1];
                for (int l = lb0 + ctx.btid; l < lb1; l += ctx.bsize) w.adj_cnt[l] = 0;
                ctx.block_sync();
                for (int q = s0 + ctx.btid; q < s1; q += ctx.bsize) {
                    int4 h = w.cons_hdr[q];
                    if (h.y >= 0) atomic_add(&w.adj_cnt[lb0 + h.y], 1);
                    if (h.z >= 0) atomic_add(&w.adj_cnt[lb0 + h.z], 1);
                }
                ctx.block_sync();
                if (ctx.btid == 0) {
                    int run = 2 * s0;
                    for (int l = lb0; l < lb1; ++l) { w.adj_off[l] = run; run += w.adj_cnt[l]; w.adj_cnt[l] = 0; }
                }
                ctx.block_sync();
                for (int q = s0 + ctx.btid; q < s1; q += ctx.bsize) {
                    int4 h = w.cons_hdr[q];
                    if (h.y >= 0) w.adj_list[w.adj_off[lb0 + h.y] + atomic_add(&w.adj_cnt[lb0 + h.y], 1)] = (q - s0) * 2;
                    if (h.z >= 0) w.adj_list[w.adj_off[lb0 + h.z] + atomic_add(&w.adj_cnt[lb0 + h.z], 1)] = (q - s0) * 2 + 1;
                }
                ctx.block_sync();
                for (int l = lb0 + ctx.btid; l < lb1; l += ctx.bsize) {   // order every short list by slot
                    int* a = w.adj_list + w.adj_off[l];
                    const int n = w.adj_cnt[l];
                    for (int x = 1; x < n; ++x) {
                        int v = a[x], y = x;
                        while (y > 0 && a[y - 1] > v) { a[y] = a[y - 1]; --y; }
                        a[y] = v;
                    }
                }
                ctx.block_sync();
            }
        }
    }
    ctx.grid_sync();
    RB_CSTAMP(14);
    // S11 launch order of the items: non-empty items 1.., most expensive first (counting sort by cost class),
    // consumed through per-kernel atomic cursors so that the long items start first and CTAs stay balanced.
    {
        int* hist = w.order_hist;
        int* curs = w.order_hist + ORDER_BUCKETS + 1;
        for (int c = ctx.gtid; c <= ORDER_BUCKETS; c += ctx.gsize) { hist[c] = 0; if (c < ORDER_BUCKETS) curs[c] = 0; }
        ctx.grid_sync();
        for (int it = 1 + ctx.gtid; it < nitems; it += ctx.gsize) {
            int nbod = w.item_body_start[it + 1] - w.item_body_start[it];
            int work = (w.item_cons_start[it + 1] - w.item_cons_start[it]) + (w.item_joint_start[it + 1] - w.item_joint_start[it]);
            if (nbod == 0 && work == 0) continue;
            int cost = nbod > work ? nbod : work;
            atomic_add(&hist[ORDER_BUCKETS - 1 - (cost < ORDER_BUCKETS ? cost : ORDER_BUCKETS - 1)], 1);
        }
        ctx.grid_sync();
        grid_exclusive_scan(ctx, hist, hist, ORDER_BUCKETS + 1, w.scan_tmp);
        for (int it = 1 + ctx.gtid; it < nitems; it += ctx.gsize) {
            int nbod = w.item_body_start[it + 1] - w.item_body_start[it];
            int work = (w.item_cons_start[it + 1] - w.item_cons_start[it]) + (w.item_joint_start[it + 1] - w.item_joint_start[it]);
            if (nbod == 0 && work == 0) continue;
            int cost = nbod > work ? nbod : work;
            int k = ORDER_BUCKETS - 1 - (cost < ORDER_BUCKETS ? cost : ORDER_BUCKETS - 1);
            w.item_order[hist[k] + atomic_add(&curs[k], 1)] = it;
        }
        ctx.grid_sync();
    }
    if (ctx.gtid == 0) {
        st->norder = w.order_hist[ORDER_BUCKETS];
        st->nitems = nitems;
        st->ncons = ncons < w.cons_cap ? ncons : w.cons_cap;
        st->nlarge_bodies = w.item_body_start[1] - w.item_body_start[0];
        st->nlarge_cons = w.item_cons_start[1] - w.item_cons_start[0];
        st->nlarge_joints = w.item_joint_start[1] - w.item_joint_start[0];
        int nisl = 0;
        (void)nisl;
        st->sched_dirty = 0;
        st->sched_ran = 1;
    }
    ctx.grid_sync();
}

// The whole pre-solve pipeline of one step.
// atan(z) for z in [0, 1]: odd minimax polynomial evaluated with explicit fused multiply-adds, so the kernels and the
// oracle agree bit for bit (libm's atan2f differs between the host and the device in the last place).
RB_HD float ccd_atan01(float z) {
    const float s = z * z;
    float p = -0.0117212f;
    p = fma_(p, s, 0.05265332f);
    p = fma_(p, s, -0.11643287f);
    p = fma_(p, s, 0.19354346f);
    p = fma_(p, s, -0.33262347f);
    p = fma_(p, s, 0.99997726f);
    return p * z;
}
// Rotation angle (0..pi) of a unit quaternion with vector-part length `vlen` and scalar part `w`: 2 atan2(vlen, |w|).
RB_HD float ccd_quat_angle(float vlen, float w) {
    const float aw = w < 0.0f ? -w : w;
    if (vlen == 0.0f) return 0.0f;
    const float half = vlen <= aw ? ccd_atan01(vlen / aw) : 1.5707964f - ccd_atan01(aw / vlen);
    return half * 2.0f;
}

// interpolate_kinematic_velocities (substep.rs:242-265; RigidBodyPosition::interpolate_velocity, rigid_body_components.rs:
// 147-196): a position-based kinematic body gets the velocity that reaches its next_position in one step (the
// rotation's scaled axis through ccd_quat_angle).  After collision detection, before the solve, like the reference.
template <class Ctx>
RB_PHASE void phase_kinematic_velocities(const Ctx& ctx, const World& w) {
    for (int k = ctx.gtid; k < w.nkinpos; k += ctx.gsize) {
        const int b = w.kinpos_list[k];
        if (w.b_type[b] != BODY_KIN_POS) continue;
        const vec3 lc = xyz(w.b_lcom_im[b]);
        const pose cur = body_pose(w, b), nxt = mkpose(mkq(w.b_next_q[b]), xyz(w.b_next_t[b]));
        const vec3 dl = xform(nxt, lc) - xform(cur, lc);
        const quat dq = qmul(nxt.q, qconj(cur.q));
        const vec3 dv = mk3(dq.x, dq.y, dq.z);
        const float len = norm(dv);
        vec3 sa = zero3();
        if (len > 1.0e-12f) {
            float angle = ccd_quat_angle(len, dq.w);
            if (dq.w < 0.0f) angle = 6.2831855f - angle;   // 2 atan2(len, w) for w < 0
            sa = dv * (angle / len);
        }
        w.b_linvel[b] = f4(dl * w.prm.inv_dt_full, 0.0f);
        w.b_angvel[b] = f4(sa * w.prm.inv_dt_full, 0.0f);
    }
}

template <int SHAPES = 0, class Ctx>
RB_PHASE void collide_pipeline(const Ctx& ctx, const World& w) {
    State* st = w.st;
    if (ctx.gtid == 0) { st->bp_ran = 0; st->sched_ran = 0; st->sleep_stamp += 1; }
    RB_CSTAMP(0);
    phase_refresh_colliders<SHAPES>(ctx, w);
    ctx.grid_sync();
    RB_CSTAMP(1);
    if (st->bp_dirty || st->lists_dirty) section_broad_phase(ctx, w);
    RB_CSTAMP(2);
    if constexpr (SHAPES != 0) { if (w.convex_work) phase_convex_manifolds(ctx, w); }   // (a kernel parameter: uniform)
    phase_narrow_phase<SHAPES>(ctx, w);
    ctx.grid_sync();
    RB_CSTAMP(3);
    if (w.nkinpos > 0) { phase_kinematic_velocities(ctx, w); ctx.grid_sync(); }   // (a kernel parameter: uniform)
    if (st->wake_any) section_wake(ctx, w);
    if (st->ntodo) section_coloring(ctx, w);
    RB_CSTAMP(4);
    if (st->sched_dirty) section_components(ctx, w);
    if (w.sleep_enabled) section_sleep(ctx, w);
    RB_CSTAMP(5);
    if (st->sched_dirty) section_schedule(ctx, w);
    RB_CSTAMP(6);
}

}  // namespace rb
