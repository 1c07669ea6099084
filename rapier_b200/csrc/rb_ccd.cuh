// rb_ccd.cuh -- continuous collision detection: motion clamping of fast bodies (SURVEY 8 f2).
//
// Reference: src/dynamics/ccd/ccd_solver.rs (update_ccd_active_flags :49-92, solve_continuous :162-321,
// apply_clamps :325-340), src/dynamics/ccd/sweeps.rs (sweep_fast_body :503-626, cast_collider_pair :282-352,
// cast_sub_shape :354-447), the fast-body criterion rigid_body_components.rs:1101-1156, and the call site
// src/pipeline/physics_pipeline/substep.rs:492-520: after the velocity solve, every awake dynamic body whose solved
// motion exceeds half its thinnest extent sweeps its colliders from `position` to `next_position` against the FIXED
// colliders, and `next_position` is clamped to the earliest impact; velocities are untouched, the residual approach
// is resolved by the next step's speculative contacts.
//
// The time of impact itself lives in the reference's parry fork (parry::query::sweep_toi: Sweep, ToiProxy,
// sweep_time_of_impact -- a Box2D-v3-style b2TimeOfImpact over point-cloud proxies), which is NOT under
// /root/reference.  It is restated here from the published algorithm's contract: cores (a ball's centre, a
// cuboid's hull) are advanced along the sweep until their distance drops to `target = max(slop, r1 + r2 - slop)`
// within `0.25 * slop`; a pair that starts within that distance reports fraction 0 and is ignored (3-D: "advances",
// sweeps.rs:287-289).  The advance is conservative advancement on a separating-axis lower bound of the distance
// (exact for face / edge / edge-edge features), so the clamp is never later than the true impact: parity with the
// fork is within the tolerance band, not bit-level (DESIGN.md, "parity unpinned").  The multi-substep splitter
// (max_ccd_substeps > 1) and sensor-crossing events are not implemented.
#pragma once
#include "rb_collide.cuh"

namespace rb {

// The advancement closes the gap by a factor (1 - closing speed / bound) per iteration.  When the rotation bound dominates
// (a long box turning by radians in one step) or the sweep grazes an obstacle, that factor stays near 0.9 -- 0.97 and a 1 m
// gap needs a hundred iterations or more to reach the 0.25 slop band; with a cap of 32 such sweeps stopped millimetres to
// centimetres short of the band, or clamped a body that only passed near an obstacle (tests/test_ccd_reference.py).
// Sweeps that converge quickly are not affected.
constexpr int CCD_MAX_ITERS = 256;

// (ccd_atan01 / ccd_quat_angle: rb_collide.cuh, shared with the kinematic velocity interpolation)

// Sweep::from_poses / Sweep::transform_at (Box2D b2Sweep): the centre of mass moves on a straight line, the rotation is
// the normalised linear interpolation of the two quaternions, the frame origin follows from the local centre.
struct CcdSweep { vec3 c1, c2; quat q1, q2; vec3 lc; };
RB_HD CcdSweep ccd_sweep(const pose& a, const pose& b, vec3 lc) {
    CcdSweep s;
    s.c1 = xform(a, lc); s.c2 = xform(b, lc); s.q1 = a.q; s.q2 = b.q; s.lc = lc;
    if (qdot(a.q, b.q) < 0.0f) { s.q2.x = -b.q.x; s.q2.y = -b.q.y; s.q2.z = -b.q.z; s.q2.w = -b.q.w; }
    return s;
}
RB_HD pose ccd_sweep_at(const CcdSweep& s, float beta) {
    const float om = 1.0f - beta;
    quat q;
    q.x = fma_(s.q2.x, beta, s.q1.x * om); q.y = fma_(s.q2.y, beta, s.q1.y * om);
    q.z = fma_(s.q2.z, beta, s.q1.z * om); q.w = fma_(s.q2.w, beta, s.q1.w * om);
    q = qnormalize(q);
    const vec3 c = madd3(s.c1 * om, s.c2, beta);
    return mkpose(q, c - rotate(q, s.lc));
}

RB_HD float ccd_abs(float x) { return x < 0.0f ? -x : x; }

// Distance between the CORES of a fixed shape A and a moving shape B (ball = its centre, cuboid = the box) and the
// unit direction n from A towards B.  For two cuboids the distance is the largest separation over the 15 candidate
// axes (a lower bound of the true distance, equal to it unless the closest features are two vertices or a vertex
// and an edge).  Returns false when the cores touch or overlap.
RB_HD bool ccd_core_distance(int shA, vec3 heA, const pose& pA, int shB, vec3 heB, const pose& pB, float& d, vec3& n) {
    if (shA == SHAPE_BALL && shB == SHAPE_BALL) {
        const vec3 dl = pB.t - pA.t;
        d = norm(dl);
        if (!(d > 0.0f)) return false;
        n = dl * (1.0f / d);
        return true;
    }
    if (shA == SHAPE_BALL || shB == SHAPE_BALL) {   // point against box, in the box's frame
        const bool box_is_a = shB == SHAPE_BALL;
        const pose& pbox = box_is_a ? pA : pB;
        const vec3 he = box_is_a ? heA : heB;
        const vec3 p = xform_inv(pbox, box_is_a ? pB.t : pA.t);
        const vec3 q = mk3(clampf(p.x, -he.x, he.x), clampf(p.y, -he.y, he.y), clampf(p.z, -he.z, he.z));
        const vec3 dl = p - q;
        d = norm(dl);
        if (!(d > 0.0f)) return false;
        const vec3 nw = rotate(pbox.q, dl * (1.0f / d));   // from the box towards the point
        n = box_is_a ? nw : -nw;
        return true;
    }
    const mat3 ra = rotmat(pA.q), rb_ = rotmat(pB.q);
    const vec3 ax[3] = {ra.c0, ra.c1, ra.c2}, bx[3] = {rb_.c0, rb_.c1, rb_.c2};
    const vec3 dc = pB.t - pA.t;
    float best = -3.4028235e38f;
    vec3 bn = mk3(0.0f, 1.0f, 0.0f);
    auto test = [&](vec3 a) {
        float s = dot3(a, dc);
        if (s < 0.0f) { a = -a; s = -s; }
        const float ea = fma_(heA.z, ccd_abs(dot3(a, ax[2])), fma_(heA.y, ccd_abs(dot3(a, ax[1])), heA.x * ccd_abs(dot3(a, ax[0]))));
        const float eb = fma_(heB.z, ccd_abs(dot3(a, bx[2])), fma_(heB.y, ccd_abs(dot3(a, bx[1])), heB.x * ccd_abs(dot3(a, bx[0]))));
        const float sep = s - ea - eb;
        if (sep > best) { best = sep; bn = a; }
    };
#pragma unroll
    for (int i = 0; i < 3; ++i) test(ax[i]);
#pragma unroll
    for (int i = 0; i < 3; ++i) test(bx[i]);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const vec3 c = cross3(ax[i], bx[j]);
            const float l2 = norm2(c);
            if (l2 > 1.0e-6f) test(c * (1.0f / sqrtf(l2)));
        }
    d = best;
    n = bn;
    return best > 0.0f;
}

// sweep_time_of_impact (restated, see the header): the fraction of the sweep at which the moving shape B comes within
// the target distance of the fixed shape A, -1 when it does not before the end of the sweep.  0 = within it from the start.
RB_HD float ccd_toi(int shA, vec3 heA, const pose& pA, int shB, vec3 heB, const CcdSweep& sw, float slop) {
    const float total = (shA == SHAPE_BALL ? heA.x : 0.0f) + (shB == SHAPE_BALL ? heB.x : 0.0f);
    const float target = max2(slop, total - slop), tol = 0.25f * slop;
    // bounds of the motion per unit of sweep fraction: the centre's velocity, and the rotation rate of the normalised
    // linear interpolation (at most 4 tan(phi / 2), phi = half the total angle, sin(phi) = |vector part of q2 q1^-1|)
    const vec3 vc = sw.c2 - sw.c1;
    const quat dq = qmul(sw.q2, qconj(sw.q1));
    float x = norm(mk3(dq.x, dq.y, dq.z));
    if (x > 1.0f) x = 1.0f;
    const float wrate = 4.0f * x / (1.0f + sqrtf(max2(1.0f - x * x, 0.0f)));
    const vec3 al = mk3(ccd_abs(sw.lc.x), ccd_abs(sw.lc.y), ccd_abs(sw.lc.z));
    const float rmax = shB == SHAPE_BALL ? norm(al) : norm(heB + al);   // farthest core point from the centre of rotation
    float t = 0.0f;
    for (int it = 0; it < CCD_MAX_ITERS; ++it) {
        const pose pB = ccd_sweep_at(sw, t);
        float d;
        vec3 n;
        if (!ccd_core_distance(shA, heA, pA, shB, heB, pB, d, n)) return t == 0.0f ? 0.0f : t;   // cores in contact
        if (d < target + tol) return t;
        const float bound = max2(-dot3(vc, n), 0.0f) + wrate * rmax;
        if (!(bound > 0.0f)) return -1.0f;
        t = t + (d - target) / bound;
        if (!(t < 1.0f)) return -1.0f;
    }
    return t;   // iteration cap: t is still a safe (early) stop
}

// rigid_body_components.rs:1125-1156 is_moving_fast_with_next_position on the solved motion of body b (`op` = position,
// `np` = next_position): the larger of the pose delta and the interpolated-velocity estimate (pose_errors, :178-196;
// the scaled-axis angle through ccd_quat_angle) against half the thinnest extent.
RB_HD bool ccd_is_moving_fast(const Params& P, vec3 lcom, const pose& op, const pose& np, float ext, float thickness) {
    const vec3 dcom = xform(np, lcom) - xform(op, lcom);
    const quat dq = qmul(np.q, qconj(op.q));
    const float x = norm(mk3(dq.x, dq.y, dq.z));
    const float max_delta_position = norm(dcom) + 2.0f * x * ext;
    const float max_velocity = norm(dcom * P.inv_dt_full) + (ccd_quat_angle(x, dq.w) * P.inv_dt_full) * ext;
    return max2(max_delta_position, max_velocity * P.dt) > 0.5f * thickness;
}

// Whether collider c's sweep may stop at collider cj: their collision groups pass and, in a world with collider filters, in
// their test modes, and so do their solver groups -- a pair without forces is a pseudo-hit the sweep ignores (sweeps.rs:563-568).
RB_HD bool ccd_groups_allow(const World& w, int c, int cj, uint2 g1) {
    const uint2 g2 = w.c_groups[cj];
    if (!w.has_filters) return (g1.x & g2.y) != 0 && (g2.x & g1.y) != 0;
    const uint4 f1 = w.c_filter[c], f2 = w.c_filter[cj];
    return groups_test(g1.x, g1.y, f1.w & 1u, g2.x, g2.y, f2.w & 1u) && groups_test(f1.x, f1.y, f1.w >> 1, f2.x, f2.y, f2.w >> 1);
}

// sweep_fast_body + apply_clamps for one fast, non-bullet body: the earliest impact of any of its colliders against
// the fixed colliders, and the pose at that fraction of the body's own sweep.  One thread; fast bodies are rare.
// (Always inlined: as an out-of-line call inside k_collide -- ABI call, 900 B more stack -- it costs time on every step of the
//  headline workload even when it is never executed.)
RB_HD pose ccd_clamp_body(const World& w, int b, pose op, pose np, bool bullet = false) {
    const State* st = w.st;
    const vec3 lcom = xyz(w.b_lcom_im[b]);
    const float slop = w.prm.linear_slop;
    const unsigned long long* skey = w.stat_key[st->stat_sorted];
    const int ns = st->nstat, nwide = st->nwide < WIDE_CAP ? st->nwide : WIDE_CAP;
    const float wn = as_float(st->stat_wn_bits) * 1.0001f + 1.0e-6f;
    float frac = 1.0f;
    for (int c = w.b_col_head[b]; c >= 0; c = w.c_next[c]) {
        const int sh = w.c_shape[c];
        if (sh == SHAPE_REMOVED || sh >= SHAPE_CAPSULE) continue;   // (capsules and convex polyhedra are not swept: speculative contacts only)
        if (w.has_sensors && (w.c_events[c] & EV_SENSOR)) continue;   // sensors neither sweep nor stop a sweep (ccd_solver.rs:92-93)
        const vec3 he = xyz(w.c_he[c]);
        const pose rel = mkpose(mkq(w.c_rel_q[c]), xyz(w.c_rel_t[c]));
        const pose cs = pmul(op, rel), ce = pmul(np, rel);
        const CcdSweep sw = ccd_sweep(cs, ce, xform_inv(rel, lcom));
        vec3 lo1, hi1, lo2, hi2;
        shape_aabb(sh, he, cs, lo1, hi1);
        shape_aabb(sh, he, ce, lo2, hi2);
        const float4 amin = make_float4(min2(lo1.x, lo2.x), min2(lo1.y, lo2.y), min2(lo1.z, lo2.z), 0.0f);
        const float4 amax = make_float4(max2(hi1.x, hi2.x), max2(hi1.y, hi2.y), max2(hi1.z, hi2.z), 0.0f);
        const uint2 g1 = w.c_groups[c];
        auto cast = [&](int cj) {
            if (!fat_overlap(amin, amax, w.c_fat_min[cj], w.c_fat_max[cj])) return;
            const int pj = w.c_parent[cj];
            if (pj >= 0 && w.b_type[pj] != BODY_FIXED) return;   // tier_allows (sweeps.rs:36-42): non-bullets only hit fixed targets
            if (w.c_shape[cj] >= SHAPE_CAPSULE) return;
            if (w.has_sensors && (w.c_events[cj] & EV_SENSOR)) return;
            if (!ccd_groups_allow(w, c, cj, g1)) return;
            const float f = ccd_toi(w.c_shape[cj], xyz(w.c_he[cj]), collider_pose(w, cj), sh, he, sw, slop);
            if (f > 0.0f && f < frac) frac = f;
        };
        if (bullet) {
            // a bullet also sweeps the colliders of kinematic / dynamic bodies -- never of other bullets -- standing still at their
            // end-of-step pose (already clamped by the first pass): sweeps.rs:36-42, :101-109; candidates by their broad-phase
            // (fat) AABBs of this step, like the reference's BVH query (:111-127)
            const int nd = st->ndyn;
            for (int i = 0; i < nd; ++i) {
                const int cj = w.dyn_list[i];
                const int pj = w.c_parent[cj], shj = w.c_shape[cj];
                if (pj == b || pj < 0 || shj == SHAPE_REMOVED || shj >= SHAPE_CAPSULE) continue;
                if (!type_is_solver(w.b_type[pj])) continue;
                if (w.has_sensors && (w.c_events[cj] & EV_SENSOR)) continue;
                if (w.b_type[pj] == BODY_DYNAMIC && (w.b_flags[pj] & FLAG_CCD)) continue;
                if (!fat_overlap(amin, amax, w.c_fat_min[cj], w.c_fat_max[cj])) continue;
                if (!ccd_groups_allow(w, c, cj, g1)) continue;
                const pose tp = pmul(body_pose(w, pj), mkpose(mkq(w.c_rel_q[cj]), xyz(w.c_rel_t[cj])));
                const float f = ccd_toi(shj, xyz(w.c_he[cj]), tp, sh, he, sw, slop);
                if (f > 0.0f && f < frac) frac = f;
            }
        }
        const unsigned amax_key = sortable_float(amax.x);
        for (int j = lower_bound_u64(skey, ns, (unsigned long long)sortable_float(amin.x - wn) << 32); j < ns; ++j) {
            const unsigned long long kj = skey[j];
            if ((unsigned)(kj >> 32) > amax_key) break;
            cast((int)(kj & 0xffffffffu));
        }
        for (int k = 0; k < nwide; ++k) cast(w.wide_list[k]);
    }
    if (frac < 1.0f) return ccd_sweep_at(ccd_sweep(op, np, lcom), frac);
    return np;
}

}  // namespace rb
