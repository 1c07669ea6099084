// rb_solver.cuh -- the velocity solver + integrator, fused per work item.
//
// One work item = a group of whole connected components ("islands").  An item is solved start to
// finish by ONE CTA with its bodies' velocities / poses / inverse inertias staged in shared memory, or
// -- for islands too large for a CTA (item 0) -- by the whole grid with bodies in HBM and grid-wide
// barriers.  Two step functions do it:
//   solve_item<R>     the streaming / grid-wide solve, one skeleton over an executor (BlockExec / GridExec /
//                     GridSpreadExec), a body store (SmemBodies / GlobalBodies) and a constraint-row policy R:
//                     HbmRows<FM, JM> (Cons tables in HBM/L2: every item of the general path, and the items
//                     k_collide takes) or PoolRows<L> (lane-cooperative rows in the L2 pool: the grid-wide item 0
//                     outside the general path)
//   solve_item_coop   the shared-memory items: bodies, impulses and (when they fit) constraint rows in shared memory
// Either way the stage order is the reference's:
//   S1 solver-body init   staged_island_solver/worker.rs:46-104, solver_body.rs:82-121
//   S2 generate           contact_with_twist_friction.rs:58-424
//   per substep: S3 increments+gyro (worker.rs:235-284), S4 joint rows (joint_constraint_builder.rs:77-152),
//                S5 update+warmstart per colour (contact_with_twist_friction.rs:426-522, :633-678),
//                S6 biased solve: joints then contacts per colour (staged_island_solver/solve.rs:12-209),
//                S7 integrate (worker.rs:568-631), S8 relax solve (contact_with_twist_friction.rs:529-554, :680-781)
//   S9 restitution (worker.rs:657-734)  S10 impulse writeback (:742-802)  S11 body writeback (:809-897)
//   + advance_to_final_positions for the item's bodies (substep.rs:84-224; rigid_body_components.rs:528-572).
// Constraint rows hold only what cannot be recomputed cheaply: lever arms, effective masses,
// builder anchors and the accumulated impulses; jacobians, rhs and cfm are recomputed from the
// staged body state in every sweep (same expressions, hence the same bits, as storing them).
#pragma once
#include "rb_collide.cuh"
#include "rb_ccd.cuh"

namespace rb {

constexpr int SB_VEC = 7;              // float4 per staged body
constexpr int SB_STRIDE = SB_VEC * 4;  // floats per staged body
// staged body layout (float4 rows, LDS.128-friendly):
//   0 (lin, incr_lin.x)  1 (ang, incr_lin.y)  2 q  3 (t, incr_lin.z)  4 (im, incr_ang.x)  5 (ii xx xy xz yy)  6 (ii yz zz, incr_ang.y, incr_ang.z)

struct BodyState { vec3 lin, ang; pose p; sym3 ii; vec3 im; };

struct SmemBodies {
    float* s;
    RB_HD float4* row(int i, int r) const { return reinterpret_cast<float4*>(s) + i * SB_VEC + r; }
    RB_HD vec3 lin(int i) const { return xyz(*row(i, 0)); }
    RB_HD vec3 ang(int i) const { return xyz(*row(i, 1)); }
    RB_HD void set_vel(int i, vec3 l, vec3 a) const {
        float4* r0 = row(i, 0); float4* r1 = row(i, 1);
        *r0 = make_float4(l.x, l.y, l.z, r0->w);
        *r1 = make_float4(a.x, a.y, a.z, r1->w);
    }
    RB_HD pose xf(int i) const { return mkpose(mkq(*row(i, 2)), xyz(*row(i, 3))); }
    RB_HD void set_xf(int i, const pose& p) const {
        *row(i, 2) = f4(p.q);
        float4* r3 = row(i, 3);
        *r3 = make_float4(p.t.x, p.t.y, p.t.z, r3->w);
    }
    RB_HD sym3 ii(int i) const {
        float4 a = *row(i, 5), b = *row(i, 6);
        sym3 m; m.xx = a.x; m.xy = a.y; m.xz = a.z; m.yy = a.w; m.yz = b.x; m.zz = b.y;
        return m;
    }
    RB_HD vec3 im(int i) const { return xyz(*row(i, 4)); }
    RB_HD void set_mass(int i, const sym3& m, vec3 im_) const {
        float4* r4 = row(i, 4); float4* r6 = row(i, 6);
        *r4 = make_float4(im_.x, im_.y, im_.z, r4->w);
        *row(i, 5) = make_float4(m.xx, m.xy, m.xz, m.yy);
        *r6 = make_float4(m.yz, m.zz, r6->z, r6->w);
    }
    RB_HD vec3 incr_lin(int i) const { return mk3(row(i, 0)->w, row(i, 1)->w, row(i, 3)->w); }
    RB_HD vec3 incr_ang(int i) const { return mk3(row(i, 4)->w, row(i, 6)->z, row(i, 6)->w); }
    RB_HD void set_incr(int i, vec3 l, vec3 a) const {
        row(i, 0)->w = l.x; row(i, 1)->w = l.y; row(i, 3)->w = l.z;
        row(i, 4)->w = a.x; row(i, 6)->z = a.y; row(i, 6)->w = a.z;
    }
};

struct GlobalBodies {  // ids are global body indices; inverse masses are read from the body tables
    const World* w;
    RB_HD vec3 lin(int i) const { return xyz(w->s_lin[i]); }
    RB_HD vec3 ang(int i) const { return xyz(w->s_ang[i]); }
    RB_HD void set_vel(int i, vec3 l, vec3 a) const { w->s_lin[i] = f4(l, 0.f); w->s_ang[i] = f4(a, 0.f); }
    RB_HD pose xf(int i) const { return mkpose(mkq(w->s_q[i]), xyz(w->s_t[i])); }
    RB_HD void set_xf(int i, const pose& p) const { w->s_q[i] = f4(p.q); w->s_t[i] = f4(p.t, 0.f); }
    RB_HD sym3 ii(int i) const { return load_ii(*w, i); }
    RB_HD vec3 im(int i) const { return xyz(w->b_eim[i]); }
    RB_HD void set_mass(int, const sym3&, vec3) const {}
    RB_HD vec3 incr_lin(int i) const { return xyz(w->s_incr_lin[i]); }
    RB_HD vec3 incr_ang(int i) const { return xyz(w->s_incr_ang[i]); }
    RB_HD void set_incr(int i, vec3 l, vec3 a) const { w->s_incr_lin[i] = f4(l, 0.f); w->s_incr_ang[i] = f4(a, 0.f); }
};

template <class B>
RB_HD BodyState gather_body(const B& bd, int id) {  // world-attached side: identity / zero (solver_body.rs:11-33)
    BodyState g;
    if (id == NO_BODY) {
        g.lin = zero3(); g.ang = zero3(); g.p = pident(); g.ii = sym_zero(); g.im = zero3();
    } else {
        g.lin = bd.lin(id); g.ang = bd.ang(id); g.p = bd.xf(id); g.ii = bd.ii(id); g.im = bd.im(id);
    }
    return g;
}
template <class B>
RB_HD void scatter_vel(const B& bd, int id, vec3 l, vec3 a) {
    if (id != NO_BODY) bd.set_vel(id, l, a);
}

RB_HD float bouncy(float restitution, bool is_new) {  // contact_pair.rs:773-779
    return is_new ? (restitution > 0.0f ? 1.0f : 0.0f) : (restitution >= 1.0f ? 1.0f : 0.0f);
}

// One contact constraint (manifold) as the sweeps see it.  In the register-resident path a thread keeps
// its constraint in this struct for the whole step; the streaming path loads / stores it per sweep.
struct Cons {
    int id1, id2, nc;
    int pair, cid[MAX_PTS];       // pair-table row and per-point contact slot (writeback targets)
    vec3 dir; float fric;         // dir1, friction limit
    vec3 t1; float wr;            // tangent1, twist effective mass
    vec3 dp1[MAX_PTS]; float r[MAX_PTS];       // lever arms body 1, projected masses
    vec3 dp2[MAX_PTS]; float dist0[MAX_PTS];   // lever arms body 2, rebased separations
    vec3 lp1[MAX_PTS], lp2[MAX_PTS];           // builder anchors (body-local)
    vec3 tdp1, tdp2; float tr0, tr1, tr2;      // friction-centre arms, tangent K matrix
    float twd[MAX_PTS];
    float imp[MAX_PTS], acc[MAX_PTS];          // normal impulses + accumulators
    float ti0, ti1, ta0, ta1, wi, wa;          // tangent / twist impulses + accumulators
    // FrictionModel::Coulomb: per-point tangent impulses + accumulators and tangent K (the jacobians are
    // recomputed from dp1 / dp2 in every sweep, like the twist model's friction-centre jacobians)
    float pti0[MAX_PTS], pti1[MAX_PTS], pta0[MAX_PTS], pta1[MAX_PTS], pk0[MAX_PTS], pk1[MAX_PTS], pk2[MAX_PTS];
};

template <int FM = 0>
RB_HD void cons_store_static(const World& w, int q, const Cons& c) {
    crow(w, CR_DIR, q) = f4(c.dir, c.fric);
    crow(w, CR_T1, q) = f4(c.t1, c.wr);
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        if (k < c.nc) {
            crow(w, CR_DP1 + k, q) = f4(c.dp1[k], c.r[k]);
            crow(w, CR_DP2 + k, q) = f4(c.dp2[k], c.dist0[k]);
            float4 a = crow(w, CR_LP1 + k, q), b = crow(w, CR_LP2 + k, q);   // keep w: seed / cid
            crow(w, CR_LP1 + k, q) = f4(c.lp1[k], a.w);
            crow(w, CR_LP2 + k, q) = f4(c.lp2[k], b.w);
            if (FM) crow(w, CR_PTK + k, q) = make_float4(c.pk0[k], c.pk1[k], c.pk2[k], 0.0f);
        }
    }
    crow(w, CR_TDP1, q) = f4(c.tdp1, c.tr0);
    crow(w, CR_TDP2, q) = f4(c.tdp2, c.tr1);
    float4 l1 = crow(w, CR_LFC1, q);
    l1.w = c.tr2;
    crow(w, CR_LFC1, q) = l1;
    crow(w, CR_TWD, q) = make_float4(c.twd[0], c.twd[1], c.twd[2], c.twd[3]);
}
template <int FM = 0>
RB_HD void cons_store_dyn(const World& w, int q, const Cons& c) {
    crow(w, CR_IMP, q) = make_float4(c.imp[0], c.imp[1], c.imp[2], c.imp[3]);
    crow(w, CR_ACC, q) = make_float4(c.acc[0], c.acc[1], c.acc[2], c.acc[3]);
    crow(w, CR_TI, q) = make_float4(c.ti0, c.ti1, c.ta0, c.ta1);
    crow(w, CR_WI, q) = make_float4(c.wi, c.wa, 0.0f, 0.0f);
    if (FM) {
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k)
            if (k < c.nc) crow(w, CR_PTI + k, q) = make_float4(c.pti0[k], c.pti1[k], c.pta0[k], c.pta1[k]);
    }
}
template <int FM = 0>
RB_HD void cons_load(const World& w, int q, Cons& c) {
    int4 h = w.cons_hdr[q];
    c.id1 = h.y; c.id2 = h.z; c.nc = h.w;
    float4 a = crow(w, CR_DIR, q), b = crow(w, CR_T1, q);
    c.dir = xyz(a); c.fric = a.w; c.t1 = xyz(b); c.wr = b.w;
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        if (k < c.nc) {
            float4 d1 = crow(w, CR_DP1 + k, q), d2 = crow(w, CR_DP2 + k, q);
            c.dp1[k] = xyz(d1); c.r[k] = d1.w; c.dp2[k] = xyz(d2); c.dist0[k] = d2.w;
            c.lp1[k] = xyz(crow(w, CR_LP1 + k, q)); c.lp2[k] = xyz(crow(w, CR_LP2 + k, q));
        }
    }
    float4 t1r = crow(w, CR_TDP1, q), t2r = crow(w, CR_TDP2, q), tw = crow(w, CR_TWD, q);
    c.tdp1 = xyz(t1r); c.tr0 = t1r.w; c.tdp2 = xyz(t2r); c.tr1 = t2r.w; c.tr2 = crow(w, CR_LFC1, q).w;
    c.twd[0] = tw.x; c.twd[1] = tw.y; c.twd[2] = tw.z; c.twd[3] = tw.w;
    float4 im = crow(w, CR_IMP, q), ac = crow(w, CR_ACC, q), ti = crow(w, CR_TI, q), wi = crow(w, CR_WI, q);
    c.imp[0] = im.x; c.imp[1] = im.y; c.imp[2] = im.z; c.imp[3] = im.w;
    c.acc[0] = ac.x; c.acc[1] = ac.y; c.acc[2] = ac.z; c.acc[3] = ac.w;
    c.ti0 = ti.x; c.ti1 = ti.y; c.ta0 = ti.z; c.ta1 = ti.w; c.wi = wi.x; c.wa = wi.y;
    if (FM) {
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k)
            if (k < c.nc) {
                float4 pi = crow(w, CR_PTI + k, q), pk = crow(w, CR_PTK + k, q);
                c.pti0[k] = pi.x; c.pti1[k] = pi.y; c.pta0[k] = pi.z; c.pta1[k] = pi.w;
                c.pk0[k] = pk.x; c.pk1[k] = pk.y; c.pk2[k] = pk.z;
            }
    }
}

// S2: contact_with_twist_friction.rs:58-424 for the manifold scheduled at slot q.  Fills `c`; the
// rarely used fields (restitution seeds, friction-centre anchors, contact ids) go to the HBM rows.
// FM: friction model (compile time, so the twist kernels carry none of the Coulomb code): 0 = Simplified (twist), 1 = Coulomb.
template <int FM = 0, class B>
RB_HD void cons_generate(const World& w, const B& bd, int q, int buf, int item, Cons& c) {
    int4 h = w.cons_hdr[q];
    const int p = h.x, id1 = h.y, id2 = h.z;
    BodyState g1 = gather_body(bd, id1), g2 = gather_body(bd, id2);
    vec3 com1 = g1.p.t, com2 = g2.p.t;
    float4 nrm = prow(w, buf, PR_NORMAL, p);
    float restitution = prow(w, buf, PR_LN2, p).w;
    int count = as_int(prow(w, buf, PR_INFO, p).z);
    if (count > MAX_PTS) count = MAX_PTS;
    vec3 dir = -xyz(nrm);
    vec3 t1 = ortho_vector(dir);
    vec3 t2 = cross3(dir, t1);
    float inv_n = 1.0f / (float)count;
    vec3 fc1 = zero3(), fc2 = zero3();
    float tws = 0.0f, tgs0 = 0.0f, tgs1 = 0.0f;
    vec3 pts[MAX_PTS];
    bool any_seed = false;
    c.id1 = id1; c.id2 = id2; c.nc = count; c.pair = p;
    c.dir = dir; c.fric = nrm.w; c.t1 = t1;
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        c.imp[k] = 0.0f; c.acc[k] = 0.0f; c.twd[k] = 0.0f; c.cid[k] = 0;
        if (k < count) {
            float4 a1 = prow(w, buf, PR_A1 + k, p), a2 = prow(w, buf, PR_A2 + k, p);
            int cid = as_int(a1.w);
            c.cid[k] = cid;
            float4 pd = prow(w, buf, PR_PD + cid, p);
            vec3 wt = xyz(prow(w, buf, PR_TW + cid, p));
            vec3 dp1 = xyz(prow(w, buf, PR_DP1 + cid, p)), dp2 = xyz(prow(w, buf, PR_DP2 + cid, p));
            float ws_imp = pd.y, ws_twist = pd.z;
            float w0 = dot3(wt, t1), w1 = dot3(wt, t2);
            float bz = bouncy(restitution, pd.x == 0.0f);
            vec3 p1 = xform(g1.p, xyz(a1));
            vec3 p2 = xform(g2.p, xyz(a2));
            float dist = dot3(p1 - p2, dir);
            vec3 point = com1 + dp1;
            pts[k] = point;
            fc1 = madd3(fc1, point, inv_n);
            fc2 = madd3(fc2, com2 + dp2, inv_n);
            vec3 v1 = g1.lin + cross3(g1.ang, dp1);
            vec3 v2 = g2.lin + cross3(g2.ang, dp2);
            tws = fma_(ws_twist, inv_n, tws);
            tgs0 = fma_(w0, inv_n, tgs0);
            tgs1 = fma_(w1, inv_n, tgs1);
            vec3 td1 = cross3(dp1, dir), td2 = cross3(dp2, -dir);
            vec3 itd1 = smul(g1.ii, td1), itd2 = smul(g2.ii, td2);
            vec3 imsum = g1.im + g2.im;
            float r = safe_inv(dot3(dir, had(imsum, dir)) + dot3(itd1, td1) + dot3(itd2, td2));
            float pv = dot3(v1 - v2, dir);
            float seed = bz * restitution * pv;
            any_seed = any_seed || seed < 0.0f;
            c.imp[k] = ws_imp;
            c.acc[k] = -ws_imp;
            c.dp1[k] = dp1; c.r[k] = r;
            c.dp2[k] = dp2; c.dist0[k] = dist - dot3(point - (com2 + dp2), dir);
            c.lp1[k] = xform_inv(g1.p, point);
            c.lp2[k] = xform_inv(g2.p, com2 + dp2);
            crow(w, CR_LP1 + k, q).w = seed;
            crow(w, CR_LP2 + k, q).w = as_float_i(cid);
            if (FM) {   // contact_with_coulomb_friction.rs:255-302: one tangent part per point, arms = the point's own
                const vec3 a10 = cross3(dp1, t1), a20 = cross3(dp2, -t1), a11 = cross3(dp1, t2), a21 = cross3(dp2, -t2);
                const vec3 i10 = smul(g1.ii, a10), i20 = smul(g2.ii, a20), i11 = smul(g1.ii, a11), i21 = smul(g2.ii, a21);
                c.pti0[k] = w0; c.pti1[k] = w1; c.pta0[k] = -w0; c.pta1[k] = -w1;
                c.pk0[k] = dot3(t1, had(imsum, t1)) + dot3(i10, a10) + dot3(i20, a20);
                c.pk1[k] = dot3(t2, had(imsum, t2)) + dot3(i11, a11) + dot3(i21, a21);
                c.pk2[k] = 2.0f * (dot3(i10, a11) + dot3(i20, a21));
            }
        }
    }
    float wimp = count > 1 ? tws : 0.0f;
    vec3 tdp1 = fc1 - com1, tdp2 = fc2 - com2;
    float wr = 0.0f;
    if (count > 1) {
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k)
            if (k < count) c.twd[k] = norm(fc1 - pts[k]);
        vec3 i1 = smul(g1.ii, dir), i2 = smul(g2.ii, -dir);
        wr = safe_inv(dot3(i1, dir) + dot3(i2, -dir));
    }
    vec3 td10 = cross3(tdp1, t1), td20 = cross3(tdp2, -t1), td11 = cross3(tdp1, t2), td21 = cross3(tdp2, -t2);
    vec3 itd10 = smul(g1.ii, td10), itd20 = smul(g2.ii, td20), itd11 = smul(g1.ii, td11), itd21 = smul(g2.ii, td21);
    vec3 imsum = g1.im + g2.im;
    c.tr0 = dot3(t1, had(imsum, t1)) + dot3(itd10, td10) + dot3(itd20, td20);
    c.tr1 = dot3(t2, had(imsum, t2)) + dot3(itd11, td11) + dot3(itd21, td21);
    c.tr2 = 2.0f * (dot3(itd10, td11) + dot3(itd20, td21));
    c.wr = wr;
    c.tdp1 = tdp1; c.tdp2 = tdp2;
    c.ti0 = tgs0; c.ti1 = tgs1; c.ta0 = -tgs0; c.ta1 = -tgs1;
    c.wi = wimp; c.wa = -wimp;
    crow(w, CR_LFC1, q) = f4(xform_inv(g1.p, fc1), c.tr2);
    crow(w, CR_LFC2, q) = f4(xform_inv(g2.p, fc2), 0.0f);
    h.w = count;
    w.cons_hdr[q] = h;
    if (any_seed) w.item_flags[item] = 1;
}

// Sweep modes
constexpr int MODE_WARMSTART = 0, MODE_BIASED = 1, MODE_RELAX = 2, MODE_RESTITUTION = 3;

// ---- per-row primitives shared by the serial sweep and the lane-cooperative sweep -----------------
struct PointPre { vec3 td1, td2, itd1, itd2; float rhs, cfm; };

// rhs and cfm of one normal row from the CURRENT poses
// (contact_with_twist_friction.rs:473-503 update, :543-550 refresh_rhs_wo_bias).
RB_HD void point_rhs(const Params& P, const BodyState& g1, const BodyState& g2, vec3 dir, vec3 lp1, vec3 lp2, float dist0, int mode,
                     float cfm_soft, float erp, float& rhs_out, float& cfm_out) {
    rhs_out = 0.0f;
    cfm_out = 1.0f;
    if (mode == MODE_BIASED || mode == MODE_RELAX) {
        vec3 p1 = xform(g1.p, lp1);
        vec3 p2 = xform(g2.p, lp2);
        float dist = dist0 + dot3(p1 - p2, dir);
        float rhs = max2(dist, 0.0f) * P.sub_inv_dt;
        if (mode == MODE_BIASED) {
            rhs = rhs + clampf(dist * erp, -P.max_corrective_velocity, 0.0f);
            cfm_out = dist <= 0.0f ? cfm_soft : 1.0f;
        }
        rhs_out = rhs;
    }
}
// Angular jacobians of one normal row (contact_with_twist_friction.rs:261-264); constant during a step.
RB_HD void point_jac(const BodyState& g1, const BodyState& g2, vec3 dir, vec3 dp1, vec3 dp2, PointPre& o) {
    o.td1 = cross3(dp1, dir);
    o.td2 = cross3(dp2, -dir);
    o.itd1 = smul(g1.ii, o.td1);
    o.itd2 = smul(g2.ii, o.td2);
}
RB_HD PointPre point_pre(const Params& P, const BodyState& g1, const BodyState& g2, vec3 dir, vec3 dp1, vec3 dp2,
                         vec3 lp1, vec3 lp2, float dist0, int mode, float cfm_soft, float erp) {
    PointPre o;
    point_rhs(P, g1, g2, dir, lp1, lp2, dist0, mode, cfm_soft, erp, o.rhs, o.cfm);
    point_jac(g1, g2, dir, dp1, dp2, o);
    return o;
}
// One projected Gauss-Seidel normal row (contact_constraint_element.rs:481-504): returns dlambda.
RB_HD float point_solve(const PointPre& pp, float r, float imp, vec3 dir, vec3 v1, vec3 w1, vec3 v2, vec3 w2, float& new_imp) {
    float dvel = dot3(dir, v1) + dot3(pp.td1, w1) - dot3(dir, v2) + dot3(pp.td2, w2) + pp.rhs;
    float nl = pp.cfm * max2(fma_(-r, dvel, imp), 0.0f);
    new_imp = nl;
    return nl - imp;
}
// End-of-step restitution row (contact_constraint_element.rs:508-534).
RB_HD float point_restitution(const PointPre& pp, float r, float imp, float acc, float seed, vec3 dir, vec3 v1, vec3 w1, vec3 v2,
                              vec3 w2, float& new_imp) {
    float dvel = dot3(dir, v1) + dot3(pp.td1, w1) - dot3(dir, v2) + dot3(pp.td2, w2) + seed;
    bool gate = seed < 0.0f && (acc + imp) > 0.0f;
    float nl = max2(fma_(-r, dvel, imp), 0.0f);
    if (!gate) nl = imp;
    new_imp = nl;
    return nl - imp;
}
RB_HD void apply_normal(vec3 lin1, vec3 lin2, vec3 itd1, vec3 itd2, float dl, vec3& v1, vec3& w1, vec3& v2, vec3& w2) {
    v1 = madd3(v1, lin1, dl);
    w1 = madd3(w1, itd1, dl);
    v2 = madd3(v2, lin2, -dl);
    w2 = madd3(w2, itd2, dl);
}

struct FrictionState { float ti0, ti1, wi; };
// Jacobians of the friction rows (constant during a step): tangent torque directions and their
// inverse-inertia images, twist directions (contact_with_twist_friction.rs:330-379).
struct FrictionJac { vec3 td10, td11, td20, td21, i10, i11, i20, i21, tw1, tw2; };
RB_HD FrictionJac friction_jac(const BodyState& g1, const BodyState& g2, vec3 dir, vec3 t1, vec3 t2, vec3 tdp1, vec3 tdp2) {
    FrictionJac j;
    j.td10 = cross3(tdp1, t1); j.td11 = cross3(tdp1, t2);
    j.td20 = cross3(tdp2, -t1); j.td21 = cross3(tdp2, -t2);
    j.i10 = smul(g1.ii, j.td10); j.i11 = smul(g1.ii, j.td11); j.i20 = smul(g2.ii, j.td20); j.i21 = smul(g2.ii, j.td21);
    j.tw1 = smul(g1.ii, dir); j.tw2 = smul(g2.ii, dir);
    return j;
}
// Twist then tangent (contact_with_twist_friction.rs:737-777; contact_constraint_element.rs:650-705, :735-756).
RB_HD void friction_solve_jac(const Params& P, const BodyState& g1, const BodyState& g2, vec3 dir, vec3 t1, vec3 t2, int nc,
                              float tlimit, float wlimit, float wr, const FrictionJac& j, float tr0, float tr1, float tr2, bool relax,
                              vec3 lfc1, vec3 lfc2, FrictionState& f, vec3& v1, vec3& w1, vec3& v2, vec3& w2) {
    if (nc > 1) {
        float dvel = dot3(dir, w1 - w2) + 0.0f;
        float nl = clampf(fma_(-wr, dvel, f.wi), -wlimit, wlimit);
        float dl = nl - f.wi;
        f.wi = nl;
        w1 = madd3(w1, j.tw1, dl);
        w2 = madd3(w2, j.tw2, -dl);
    }
    float rhs0 = 0.0f, rhs1 = 0.0f;  // tangent rhs_wo_bias = tangent_velocity . t = 0 (no hooks)
    if (!relax) {  // update(): bias from the friction-centre drift (contact_with_twist_friction.rs:506-514)
        vec3 p1 = xform(g1.p, lfc1);
        vec3 p2 = xform(g2.p, lfc2);
        rhs0 = 0.0f + dot3(p1 - p2, t1) * P.sub_inv_dt;
        rhs1 = 0.0f + dot3(p1 - p2, t2) * P.sub_inv_dt;
    }
    float dv0 = dot3(t1, v1) + dot3(j.td10, w1) - dot3(t1, v2) + dot3(j.td20, w2) + rhs0;
    float dv1 = dot3(t2, v1) + dot3(j.td11, w1) - dot3(t2, v2) + dot3(j.td21, w2) + rhs1;
    float k11 = tr0, k22 = tr1, k12 = tr2 * 0.5f;
    float inv_det = safe_inv(fma_(k11, k22, -(k12 * k12)));
    float d0 = fma_(k22, dv0, -(k12 * dv1)) * inv_det;
    float d1 = fma_(k11, dv1, -(k12 * dv0)) * inv_det;
    float n0 = f.ti0 - d0, n1 = f.ti1 - d1;
    float len = sqrtf(fma_(n1, n1, n0 * n0));
    if (len > tlimit) {
        float sc = tlimit / len;
        n0 = n0 * sc;
        n1 = n1 * sc;
    }
    float dl0 = n0 - f.ti0, dl1 = n1 - f.ti1;
    f.ti0 = n0;
    f.ti1 = n1;
    v1 = madd3v(v1, madd3(t1 * dl0, t2, dl1), g1.im);
    w1 = madd3(madd3(w1, j.i10, dl0), j.i11, dl1);
    v2 = madd3v(v2, madd3(t1 * (-dl0), t2, -dl1), g2.im);
    w2 = madd3(madd3(w2, j.i20, dl0), j.i21, dl1);
}
RB_HD void friction_solve(const Params& P, const BodyState& g1, const BodyState& g2, vec3 dir, vec3 t1, vec3 t2, int nc,
                          float tlimit, float wlimit, float wr, vec3 tdp1, vec3 tdp2, float tr0, float tr1, float tr2,
                          bool relax, vec3 lfc1, vec3 lfc2, FrictionState& f, vec3& v1, vec3& w1, vec3& v2, vec3& w2) {
    FrictionJac j = friction_jac(g1, g2, dir, t1, t2, tdp1, tdp2);
    friction_solve_jac(P, g1, g2, dir, t1, t2, nc, tlimit, wlimit, wr, j, tr0, tr1, tr2, relax, lfc1, lfc2, f, v1, w1, v2, w2);
}
// Friction + twist warm start (contact_constraint_element.rs:627-647, :720-732).
RB_HD void friction_warmstart_jac(const BodyState& g1, const BodyState& g2, vec3 t1, vec3 t2, int nc, const FrictionJac& j,
                                  float ti0, float ti1, float wi, vec3& v1, vec3& w1, vec3& v2, vec3& w2) {
    v1 = madd3v(v1, madd3(t1 * ti0, t2, ti1), g1.im);
    w1 = madd3(madd3(w1, j.i10, ti0), j.i11, ti1);
    v2 = madd3v(v2, madd3(t1 * (-ti0), t2, -ti1), g2.im);
    w2 = madd3(madd3(w2, j.i20, ti0), j.i21, ti1);
    if (nc > 1) {
        w1 = madd3(w1, j.tw1, wi);
        w2 = madd3(w2, j.tw2, -wi);
    }
}
RB_HD void friction_warmstart(const BodyState& g1, const BodyState& g2, vec3 dir, vec3 t1, vec3 t2, int nc, vec3 tdp1, vec3 tdp2,
                              float ti0, float ti1, float wi, vec3& v1, vec3& w1, vec3& v2, vec3& w2) {
    FrictionJac j = friction_jac(g1, g2, dir, t1, t2, tdp1, tdp2);
    friction_warmstart_jac(g1, g2, t1, t2, nc, j, ti0, ti1, wi, v1, w1, v2, w2);
}

// One constraint, one sweep, one thread (streaming path; constraint in registers for the call).
// MODE_WARMSTART = builder.update + constraint.warmstart (fused, worker.rs:438-539);
// MODE_BIASED / MODE_RELAX = (refresh_rhs_wo_bias +) solve; MODE_RESTITUTION = apply_restitution.
template <int FM = 0, class B>
RB_HD void cons_sweep(const World& w, const B& bd, int q, Cons& c, int mode, bool solve_friction) {
    const Params& P = w.prm;
    const int id1 = c.id1, id2 = c.id2, nc = c.nc;
    BodyState g1 = gather_body(bd, id1), g2 = gather_body(bd, id2);
    vec3 v1 = g1.lin, w1 = g1.ang, v2 = g2.lin, w2 = g2.ang;
    const vec3 dir = c.dir, t1 = c.t1;
    const vec3 t2 = cross3(dir, t1);
    const bool is_static = id1 == NO_BODY || id2 == NO_BODY;
    const float stf = is_static ? 1.0f : 0.0f;
    const float cfm_soft = P.dyn_cfm + stf * (P.static_cfm - P.dyn_cfm);
    const float erp = P.dyn_erp + stf * (P.static_erp - P.dyn_erp);
    const vec3 lin1 = had(dir, g1.im), lin2 = had(dir, g2.im);

    if (mode == MODE_RESTITUTION) {
        bool any = false;
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k)
            if (k < nc) any = any || crow(w, CR_LP1 + k, q).w < 0.0f;
        if (!any) return;
    }
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        if (k < nc) {
            PointPre pp = point_pre(P, g1, g2, dir, c.dp1[k], c.dp2[k], c.lp1[k], c.lp2[k], c.dist0[k], mode, cfm_soft, erp);
            float dl;
            if (mode == MODE_WARMSTART) {
                float l = c.imp[k];
                c.acc[k] = c.acc[k] + l;
                l = l * P.warmstart_coeff;
                c.imp[k] = l;
                dl = l;
            } else if (mode == MODE_RESTITUTION) {
                float nl;
                dl = point_restitution(pp, c.r[k], c.imp[k], c.acc[k], crow(w, CR_LP1 + k, q).w, dir, v1, w1, v2, w2, nl);
                c.imp[k] = nl;
            } else {
                float nl;
                dl = point_solve(pp, c.r[k], c.imp[k], dir, v1, w1, v2, w2, nl);
                c.imp[k] = nl;
            }
            apply_normal(lin1, lin2, pp.itd1, pp.itd2, dl, v1, w1, v2, w2);
        }
    }
    if (FM && mode == MODE_WARMSTART) {   // contact_with_coulomb_friction.rs:438-447, :584-592
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k) {
            if (k < nc) {
                c.pta0[k] = c.pta0[k] + c.pti0[k]; c.pta1[k] = c.pta1[k] + c.pti1[k];
                c.pti0[k] = c.pti0[k] * P.warmstart_coeff; c.pti1[k] = c.pti1[k] * P.warmstart_coeff;
                friction_warmstart(g1, g2, dir, t1, t2, 1, c.dp1[k], c.dp2[k], c.pti0[k], c.pti1[k], 0.0f, v1, w1, v2, w2);
            }
        }
    } else if (FM && mode != MODE_RESTITUTION && solve_friction) {   // :659-676, limit = mu * lambda_k per point
        const bool relax = mode == MODE_RELAX;
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k) {
            if (k < nc) {
                const float tlimit = (0.0f + c.imp[k]) * c.fric;
                FrictionState f;
                f.ti0 = c.pti0[k]; f.ti1 = c.pti1[k]; f.wi = 0.0f;
                friction_solve(P, g1, g2, dir, t1, t2, 1, tlimit, 0.0f, 0.0f, c.dp1[k], c.dp2[k], c.pk0[k], c.pk1[k], c.pk2[k], relax,
                               c.lp1[k], c.lp2[k], f, v1, w1, v2, w2);
                c.pti0[k] = f.ti0; c.pti1[k] = f.ti1;
            }
        }
    } else if (mode == MODE_WARMSTART) {
        c.ta0 = c.ta0 + c.ti0; c.ta1 = c.ta1 + c.ti1;
        c.ti0 = c.ti0 * P.warmstart_coeff; c.ti1 = c.ti1 * P.warmstart_coeff;
        c.wa = c.wa + c.wi;
        c.wi = c.wi * P.warmstart_coeff;
        friction_warmstart(g1, g2, dir, t1, t2, nc, c.tdp1, c.tdp2, c.ti0, c.ti1, c.wi, v1, w1, v2, w2);
    } else if (mode != MODE_RESTITUTION && solve_friction) {
        float tlimit = 0.0f, wlimit = 0.0f;
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k) {
            if (k < nc) {
                tlimit = tlimit + c.imp[k];
                wlimit = fma_(c.imp[k], c.twd[k], wlimit);
            }
        }
        tlimit = tlimit * c.fric;
        wlimit = wlimit * c.fric;
        const bool relax = mode == MODE_RELAX;
        vec3 lfc1 = zero3(), lfc2 = zero3();
        if (!relax) { lfc1 = xyz(crow(w, CR_LFC1, q)); lfc2 = xyz(crow(w, CR_LFC2, q)); }
        FrictionState f;
        f.ti0 = c.ti0; f.ti1 = c.ti1; f.wi = c.wi;
        friction_solve(P, g1, g2, dir, t1, t2, nc, tlimit, wlimit, c.wr, c.tdp1, c.tdp2, c.tr0, c.tr1, c.tr2, relax, lfc1, lfc2, f,
                       v1, w1, v2, w2);
        c.ti0 = f.ti0; c.ti1 = f.ti1; c.wi = f.wi;
    }
    scatter_vel(bd, id1, v1, w1);
    scatter_vel(bd, id2, v2, w2);
}

RB_HD float canon0(float x) { return x == 0.0f ? 0.0f : x; }

// S10: contact_with_twist_friction.rs:783-829
// `ids_in_c`: c.pair / c.cid are valid (shared-memory path); otherwise they are fetched from the schedule rows.
template <int FM = 0>
RB_HD void cons_writeback(const World& w, int q, int buf, const Cons& c, bool ids_in_c = false) {
    const int p = ids_in_c ? c.pair : w.cons_hdr[q].x;
    vec3 t2 = cross3(c.dir, c.t1);
    if (FM) {   // contact_with_coulomb_friction.rs:683-740: per-point world tangent impulse; the twist slot is left alone
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k) {
            if (k < c.nc) {
                const int cid = ids_in_c ? c.cid[k] : as_int(crow(w, CR_LP2 + k, q).w);
                const float b0 = canon0(c.pti0[k]), b1 = canon0(c.pti1[k]);
                vec3 twk = c.t1 * b0 + t2 * b1;
                float* pd = &prow(w, buf, PR_PD + cid, p).x;
                pd[0] = canon0(c.acc[k] + c.imp[k]);
                pd[1] = canon0(c.imp[k]);
                prow(w, buf, PR_TW + cid, p) = f4(mk3(canon0(twk.x), canon0(twk.y), canon0(twk.z)), 0.0f);
            }
        }
        return;
    }
    float a0 = canon0(c.ti0), a1 = canon0(c.ti1);
    vec3 tw = c.t1 * a0 + t2 * a1;
    tw = mk3(canon0(tw.x), canon0(tw.y), canon0(tw.z));
    float twist = canon0(c.wi);
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        if (k < c.nc) {
            int cid = ids_in_c ? c.cid[k] : as_int(crow(w, CR_LP2 + k, q).w);
            float* pd = &prow(w, buf, PR_PD + cid, p).x;   // .w (feature id) stays as it is: no read needed
            pd[0] = canon0(c.acc[k] + c.imp[k]);
            pd[1] = canon0(c.imp[k]);
            pd[2] = twist;
            prow(w, buf, PR_TW + cid, p) = f4(tw, 0.0f);
        }
    }
}

// rigid_body.rs:2023-2046
RB_HD vec3 gyro_corrected(vec3 angvel, quat axes, vec3 pin, vec3 ipin, float dt) {
    vec3 wl = rotate_inv(axes, angvel);
    vec3 cur = had(pin, wl);
    vec3 eg = (-cross3(wl, cur)) * dt;
    vec3 tot = cur + eg;
    float ts = norm2(tot);
    if (ts != 0.0f) {
        vec3 capped = tot * sqrtf(norm2(cur) / ts);
        return rotate(axes, had(ipin, capped));
    }
    return angvel;
}

// ------------------------------------------------------------------------------------------------
// Joints (locked axes): per-substep rows (joint_constraint_helper.rs:95-164, :411-461, :628-722).
// ------------------------------------------------------------------------------------------------
// MASK: the joint's locked axes when known at compile time (0 = read them from the joint): the unrolled row loops
// then only keep the locked slots, which is what keeps a spherical joint's three rows in registers.
template <unsigned MASK, class B>
RB_HD void joint_update_t(const World& w, const B& bd, int q) {
    int4 h = w.j_sched_ids[q];
    const int j = h.x, id1 = h.y, id2 = h.z;
    int4 ji = w.j_info[j];
    const unsigned locked = MASK ? MASK : (unsigned)ji.z;
    BodyState g1 = gather_body(bd, id1), g2 = gather_body(bd, id2);
    // transform_to_solver_body_space (generic_joint.rs:624-636)
    pose lf1 = mkpose(mkq(w.j_f1_q[j]), xyz(w.j_f1_t[j]));
    pose lf2 = mkpose(mkq(w.j_f2_q[j]), xyz(w.j_f2_t[j]));
    if (id1 == NO_BODY) lf1 = pmul(body_pose(w, ji.x), lf1); else lf1.t = lf1.t - xyz(w.b_lcom_im[ji.x]);
    if (id2 == NO_BODY) lf2 = pmul(body_pose(w, ji.y), lf2); else lf2.t = lf2.t - xyz(w.b_lcom_im[ji.y]);
    pose f1 = pmul(g1.p, lf1), f2 = pmul(g2.p, lf2);
    float2 soft = w.j_soft[j];
    float omega = soft.x * 6.283185307179586f;
    float sdt = w.prm.sub_dt;
    float erp_inv_dt = omega / (sdt * omega + 2.0f * soft.y);
    float erpv = sdt * erp_inv_dt;
    float cfm_coeff = 0.0f;
    if (erpv != 0.0f) {
        float e1 = 1.0f / erpv - 1.0f;
        cfm_coeff = e1 * e1 / ((1.0f + e1) * 4.0f * soft.y * soft.y);
    }
    mat3 basis = rotmat(f1.q);
    vec3 bc[3] = {basis.c0, basis.c1, basis.c2};
    vec3 lin_err = f2.t - f1.t;
    vec3 nc1 = f2.t;
#pragma unroll
    for (int i = 0; i < 3; ++i)
        if (locked & (1u << i)) nc1 = nc1 - bc[i] * dot3(lin_err, bc[i]);
    f1.t = nc1;
    vec3 r1 = f1.t - g1.p.t, r2 = f2.t - g2.p.t;
    float sgn = copysign1(qdot(f1.q, f2.q));
    quat ae = qmul(qconj(f1.q), f2.q);
    vec3 aerr = mk3(ae.x * sgn, ae.y * sgn, ae.z * sgn);
    vec3 a = mk3(f1.q.x, f1.q.y, f1.q.z), b = mk3(f2.q.x, f2.q.y, f2.q.z);
    float wa = f1.q.w, wb = f2.q.w;
    vec3 cv = a * wb + b * wa;
    float ab = dot3(a, b);
    vec3 imsum = g1.im + g2.im;
    // Row slots are FIXED (0..2 = locked angular x y z, 3..5 = locked linear x y z: the reference's row order,
    // joint_constraint_helper.rs) and every loop below is fully unrolled with the slot's lock bit as a predicate, so
    // the rows stay in registers (a compacted, dynamically indexed array would live in local memory).  Unlocked
    // slots are skipped, so the locked rows see exactly the operations of the compacted form.
    vec3 lin[6], aj1[6], aj2[6], ia1[6], ia2[6];
    float rhs[6], rwb[6], cg[6], il[6];
    bool on[6];
#pragma unroll
    for (int sl = 0; sl < 6; ++sl) {
        const int dofi = sl < 3 ? sl + 3 : sl - 3;   // slot -> degree of freedom (3..5 angular, 0..2 linear)
        on[sl] = (locked & (1u << dofi)) != 0;
        lin[sl] = aj1[sl] = aj2[sl] = ia1[sl] = ia2[sl] = zero3();
        rhs[sl] = rwb[sl] = cg[sl] = il[sl] = 0.0f;
        if (!on[sl]) continue;
        if (sl < 3) {
            const int ax = sl;
            // row `ax` of D = 0.5 (a b^T + (wa wb - a.b) I - [cv]x + b a^T)  (rotation_ops.rs:121-137), times sgn
            float av = comp(a, ax), bv = comp(b, ax);
            float dg = wa * wb - ab;
            vec3 cx = ax == 0 ? mk3(0.0f, -cv.z, cv.y) : (ax == 1 ? mk3(cv.z, 0.0f, -cv.x) : mk3(-cv.y, cv.x, 0.0f));
            vec3 row = mk3((av * b.x + (ax == 0 ? dg : 0.0f) - cx.x + bv * a.x) * 0.5f,
                           (av * b.y + (ax == 1 ? dg : 0.0f) - cx.y + bv * a.y) * 0.5f,
                           (av * b.z + (ax == 2 ? dg : 0.0f) - cx.z + bv * a.z) * 0.5f);
            vec3 aj = row * sgn;
            aj1[sl] = aj; aj2[sl] = aj;
            ia1[sl] = smul(g1.ii, aj); ia2[sl] = smul(g2.ii, aj);
            rhs[sl] = 0.0f + comp(aerr, ax) * erp_inv_dt;
        } else {
            const int i = sl - 3;
            lin[sl] = bc[i]; aj1[sl] = cross3(r1, bc[i]); aj2[sl] = cross3(r2, bc[i]);
            ia1[sl] = smul(g1.ii, aj1[sl]); ia2[sl] = smul(g2.ii, aj2[sl]);
            rhs[sl] = 0.0f + dot3(bc[i], lin_err) * erp_inv_dt;
        }
    }
#pragma unroll
    for (int jx = 0; jx < 6; ++jx) {  // finalize_constraints: Gram-Schmidt in the mass metric
        if (!on[jx]) continue;
        float djj = dot3(lin[jx], had(imsum, lin[jx])) + dot3(ia1[jx], aj1[jx]) + dot3(ia2[jx], aj2[jx]);
        float gain = djj * cfm_coeff + cg[jx];
        float inv_djj = safe_inv(djj);
        il[jx] = safe_inv(djj + gain);
        cg[jx] = gain;
#pragma unroll
        for (int ix = jx + 1; ix < 6; ++ix) {
            if (!on[ix]) continue;
            float dij = dot3(lin[ix], had(imsum, lin[jx])) + dot3(ia1[ix], aj1[jx]) + dot3(ia2[ix], aj2[jx]);
            float coeff = dij * inv_djj;
            lin[ix] = lin[ix] - lin[jx] * coeff;
            aj1[ix] = aj1[ix] - aj1[jx] * coeff;
            aj2[ix] = aj2[ix] - aj2[jx] * coeff;
            ia1[ix] = ia1[ix] - ia1[jx] * coeff;
            ia2[ix] = ia2[ix] - ia2[jx] * coeff;
            rwb[ix] = rwb[ix] - rwb[jx] * coeff;
            rhs[ix] = rhs[ix] - rhs[jx] * coeff;
        }
    }
    int len = 0, packed = 0;
#pragma unroll
    for (int sl = 0; sl < 6; ++sl) {
        if (!on[sl]) continue;
        const int dofi = sl < 3 ? sl + 3 : sl - 3;
        const int s = 6 * q + len;
        jrow(w, JR_LIN, s) = f4(lin[sl], 0.0f);   // impulse restarts from 0 (warmstart_joints = false)
        jrow(w, JR_A1, s) = f4(aj1[sl], il[sl]);
        jrow(w, JR_A2, s) = f4(aj2[sl], rhs[sl]);
        jrow(w, JR_IA1, s) = f4(ia1[sl], rwb[sl]);
        jrow(w, JR_IA2, s) = f4(ia2[sl], cg[sl]);
        packed |= dofi << (8 + 4 * len);
        ++len;
    }
    h.w = len | packed;
    w.j_sched_ids[q] = h;
}
template <class B>
RB_HD void joint_update(const World& w, const B& bd, int q) {
    const unsigned locked = (unsigned)w.j_info[w.j_sched_ids[q].x].z;
    if (locked == 7u) joint_update_t<7u>(w, bd, q);          // spherical: linear x y z
    else if (locked == 63u) joint_update_t<63u>(w, bd, q);   // fixed
    else joint_update_t<0u>(w, bd, q);
}

// joint_velocity_constraint.rs:97-124.  The rows are loaded three at a time before the first of them is solved
// (their addresses do not depend on the sweep, and the stores of one row must not delay the loads of the next);
// three rows = a spherical joint, the common case, in one batch.
template <class B>
RB_HD void joint_solve(const World& w, const B& bd, int q, bool wo_bias) {
    int4 h = w.j_sched_ids[q];
    const int id1 = h.y, id2 = h.z, len = h.w & 0xff;
    BodyState g1 = gather_body(bd, id1), g2 = gather_body(bd, id2);
    vec3 v1 = g1.lin, w1 = g1.ang, v2 = g2.lin, w2 = g2.ang;
    for (int r0 = 0; r0 < len; r0 += 3) {
        float4 L[3], A1[3], A2[3], I1[3], I2[3];
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (r0 + k < len) {
                const int s = 6 * q + r0 + k;
                L[k] = jrow(w, JR_LIN, s); A1[k] = jrow(w, JR_A1, s); A2[k] = jrow(w, JR_A2, s); I1[k] = jrow(w, JR_IA1, s);
                I2[k] = jrow(w, JR_IA2, s);
            }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (r0 + k < len) {
                const int s = 6 * q + r0 + k;
                float rhs_c = wo_bias ? I1[k].w : A2[k].w;
                float dlin = dot3(xyz(L[k]), v2 - v1);
                float dang = dot3(xyz(A2[k]), w2) - dot3(xyz(A1[k]), w1);
                float rhs = dlin + dang + rhs_c;
                float total = L[k].w + A1[k].w * (rhs - I2[k].w * L[k].w);
                float delta = total - L[k].w;
                L[k].w = total;
                vec3 li = xyz(L[k]) * delta;
                v1 = madd3v(v1, li, g1.im);
                w1 = madd3(w1, xyz(I1[k]), delta);
                v2 = madd3v(v2, -li, g2.im);
                w2 = madd3(w2, xyz(I2[k]), -delta);
                jrow(w, JR_LIN, s) = L[k];
                if (wo_bias) { A2[k].w = I1[k].w; jrow(w, JR_A2, s) = A2[k]; }
            }
        }
    }
    scatter_vel(bd, id1, v1, w1);
    scatter_vel(bd, id2, v2, w2);
}

RB_HD void joint_writeback(const World& w, int q) {
    int4 h = w.j_sched_ids[q];
    int len = h.w & 0xff;
    for (int r = 0; r < len; ++r) {
        int dof = (h.w >> (8 + 4 * r)) & 0xf;
        w.j_impulses[h.x * 6 + dof] = jrow(w, JR_LIN, 6 * q + r).w;
    }
}

// ------------------------------------------------------------------------------------------------
// Generic joint path (JM = 1): locked axes + limits + motors, rows in the reference's order
// (JointConstraint::update, joint_velocity_constraint.rs:145-357): motors (angular, linear) orthogonalised among
// themselves, then locked axes and limits orthogonalised together; rows with bounded impulses are never pivots
// (finalize_constraints, joint_constraint_helper.rs:676-722).  12 row slots per joint; one thread builds a joint's rows
// in local memory (these joints are rare next to contacts; the locked-only path above keeps its register-resident form).
// ------------------------------------------------------------------------------------------------
constexpr int JROWS_GENERIC = 12;
struct GRow { vec3 lin, a1, a2, ia1, ia2; float inv_lhs, rhs, rwb, cg, cc, lo, hi; int dof, kind; };

RB_HD float atan2_poly(float y, float x) {   // atan2 in (-pi, pi] from ccd_atan01 (explicit arithmetic, equal to the oracle's bit for bit)
    const float ax = x < 0.0f ? -x : x, ay = y < 0.0f ? -y : y;
    if (ax == 0.0f && ay == 0.0f) return 0.0f;
    float a = ay <= ax ? ccd_atan01(ay / ax) : 1.5707964f - ccd_atan01(ax / ay);
    if (x < 0.0f) a = 3.1415927f - a;
    return y < 0.0f ? -a : a;
}
RB_HD float fabs1(float x) { return x < 0.0f ? -x : x; }
RB_HD void grows_finalize(GRow* r, int a, int b, vec3 imsum) {
    for (int jx = a; jx < b; ++jx) {
        GRow& cj = r[jx];
        const float djj = dot3(cj.lin, had(imsum, cj.lin)) + dot3(cj.ia1, cj.a1) + dot3(cj.ia2, cj.a2);
        const float gain = djj * cj.cc + cj.cg;
        const float inv_djj = safe_inv(djj);
        cj.inv_lhs = safe_inv(djj + gain);
        cj.cg = gain;
        if (!(cj.lo == -FMAX32 && cj.hi == FMAX32)) continue;
        for (int ix = jx + 1; ix < b; ++ix) {
            GRow& ci = r[ix];
            const float dij = dot3(ci.lin, had(imsum, cj.lin)) + dot3(ci.ia1, cj.a1) + dot3(ci.ia2, cj.a2);
            const float coeff = dij * inv_djj;
            ci.lin = ci.lin - cj.lin * coeff;
            ci.a1 = ci.a1 - cj.a1 * coeff;
            ci.a2 = ci.a2 - cj.a2 * coeff;
            ci.ia1 = ci.ia1 - cj.ia1 * coeff;
            ci.ia2 = ci.ia2 - cj.ia2 * coeff;
            ci.rwb = ci.rwb - cj.rwb * coeff;
            ci.rhs = ci.rhs - cj.rhs * coeff;
        }
    }
}
template <class B>
RB_HD void joint_update_generic(const World& w, const B& bd, int q, int sub) {
    int4 h = w.j_sched_ids[q];
    const int j = h.x, id1 = h.y, id2 = h.z;
    const int4 ji = w.j_info[j];
    const unsigned locked = (unsigned)ji.z;
    BodyState g1 = gather_body(bd, id1), g2 = gather_body(bd, id2);
    pose lf1 = mkpose(mkq(w.j_f1_q[j]), xyz(w.j_f1_t[j]));
    pose lf2 = mkpose(mkq(w.j_f2_q[j]), xyz(w.j_f2_t[j]));
    if (id1 == NO_BODY) lf1 = pmul(body_pose(w, ji.x), lf1); else lf1.t = lf1.t - xyz(w.b_lcom_im[ji.x]);
    if (id2 == NO_BODY) lf2 = pmul(body_pose(w, ji.y), lf2); else lf2.t = lf2.t - xyz(w.b_lcom_im[ji.y]);
    pose f1 = pmul(g1.p, lf1), f2 = pmul(g2.p, lf2);
    const float2 soft = w.j_soft[j];
    const float omega = soft.x * 6.283185307179586f;
    const float sdt = w.prm.sub_dt;
    const float erp_inv_dt = omega / (sdt * omega + 2.0f * soft.y);
    const float erpv = sdt * erp_inv_dt;
    float cfm_coeff = 0.0f;
    if (erpv != 0.0f) {
        const float e1 = 1.0f / erpv - 1.0f;
        cfm_coeff = e1 * e1 / ((1.0f + e1) * 4.0f * soft.y * soft.y);
    }
    const mat3 basis = rotmat(f1.q);
    const vec3 bc[3] = {basis.c0, basis.c1, basis.c2};
    const vec3 lin_err = f2.t - f1.t;
    vec3 nc1 = f2.t;
    for (int i = 0; i < 3; ++i)
        if (locked & (1u << i)) nc1 = nc1 - bc[i] * dot3(lin_err, bc[i]);
    f1.t = nc1;
    const vec3 r1 = f1.t - g1.p.t, r2 = f2.t - g2.p.t;
    const float sgn = copysign1(qdot(f1.q, f2.q));
    const quat ae = qmul(qconj(f1.q), f2.q);
    const float aerr[3] = {ae.x * sgn, ae.y * sgn, ae.z * sgn};
    const float aew = ae.w * sgn;
    const vec3 a = mk3(f1.q.x, f1.q.y, f1.q.z), b = mk3(f2.q.x, f2.q.y, f2.q.z);
    const float wa = f1.q.w, wb = f2.q.w;
    const vec3 cv = a * wb + b * wa;
    const float ab = dot3(a, b);
    const vec3 imsum = g1.im + g2.im;
    const unsigned free_axes = ~locked & 63u;
    const uint2 axes = w.j_axes[j];
    const unsigned limit_axes = axes.x & free_axes, motor_axes = axes.y & free_axes;
    const unsigned coupled = (axes.x >> 8) & 63u;   // coupled_axes (joint_velocity_constraint.rs:163-178)
    const bool has_lin_coupling = (coupled & 7u) != 0, has_ang_coupling = (coupled & 56u) != 0;
    const int first_lin = (coupled & 1u) ? 0 : ((coupled & 2u) ? 1 : 2);
    const int first_ang = (coupled & 8u) ? 3 : ((coupled & 16u) ? 4 : 5);
    const float inv_dt = w.prm.sub_inv_dt, max_bias = w.prm.max_corrective_velocity;
    GRow rows[JROWS_GENERIC];
    auto lock_linear_row = [&](int i, float erp, float cfm, int dof, int kind) {
        GRow r;
        r.lin = bc[i]; r.a1 = cross3(r1, bc[i]); r.a2 = cross3(r2, bc[i]);
        r.ia1 = smul(g1.ii, r.a1); r.ia2 = smul(g2.ii, r.a2);
        r.inv_lhs = 0.0f; r.cc = cfm; r.cg = 0.0f; r.rwb = 0.0f;
        r.rhs = 0.0f + dot3(bc[i], lin_err) * erp;
        r.lo = -FMAX32; r.hi = FMAX32; r.dof = dof; r.kind = kind;
        return r;
    };
    auto motor_coeffs = [&](int i, float4& ma, float& m_erp, float& m_cc, float& m_cg, float& max_imp) {
        ma = w.j_motor_a[j * 6 + i];
        const float2 mb = w.j_motor_b[j * 6 + i];
        m_erp = ma.z * safe_inv(sdt * ma.z + ma.w);
        const float c = safe_inv(sdt * sdt * ma.z + sdt * ma.w);
        const bool acc = as_int(mb.y) == 0;
        m_cc = acc ? c : 0.0f;
        m_cg = acc ? 0.0f : c;
        max_imp = mb.x * sdt;
    };
    int len = 0;
    for (int i = 3; i < 6; ++i) {   // motor_angular
        if (!((motor_axes & ~coupled) & (1u << i))) continue;
        float4 ma; float m_erp, m_cc, m_cg, max_imp;
        motor_coeffs(i, ma, m_erp, m_cc, m_cg, max_imp);
        GRow& r = rows[len++];
        const vec3 aj = bc[i - 3];
        float rwb = 0.0f;
        if (m_erp != 0.0f) {
            const float ce = clampf(aerr[i - 3], -1.0f, 1.0f);
            const float ang_dist = atan2_poly(ce, sqrtf(max2(1.0f - ce * ce, 0.0f))) * 2.0f;
            float s_err = ang_dist - ma.y;
            const float sg = s_err > 0.0f ? 1.0f : (s_err < 0.0f ? -1.0f : 0.0f);
            const float comp = s_err - sg * 6.2831855f;
            if (!(fabs1(s_err) < fabs1(comp))) s_err = comp;
            rwb = rwb + s_err * m_erp;
        }
        rwb = rwb + -ma.x;
        r.lin = zero3(); r.a1 = aj; r.a2 = aj; r.ia1 = smul(g1.ii, aj); r.ia2 = smul(g2.ii, aj);
        r.inv_lhs = 0.0f; r.cc = m_cc; r.cg = m_cg; r.rhs = rwb; r.rwb = rwb;
        r.lo = -max_imp; r.hi = max_imp; r.dof = i; r.kind = 2;
    }
    for (int i = 0; i < 3; ++i) {   // motor_linear
        if (!((motor_axes & ~coupled) & (1u << i))) continue;
        float4 ma; float m_erp, m_cc, m_cg, max_imp;
        motor_coeffs(i, ma, m_erp, m_cc, m_cg, max_imp);
        GRow r = lock_linear_row(i, 0.0f, 0.0f, i, 2);
        float rwb = 0.0f;
        if (m_erp != 0.0f) rwb = rwb + (dot3(lin_err, r.lin) - ma.y) * m_erp;
        float target_vel = ma.x;
        if (limit_axes & (1u << i)) {
            const float dist = dot3(lin_err, r.lin);
            const float2 lim = w.j_limits[j * 6 + i];
            target_vel = clampf(target_vel, (lim.x - dist) * inv_dt, (lim.y - dist) * inv_dt);
        }
        rwb = rwb + -target_vel;
        r.cc = m_cc; r.cg = m_cg; r.lo = -max_imp; r.hi = max_imp; r.rhs = rwb; r.rwb = rwb;
        rows[len++] = r;
    }
    // the distance row of the coupled linear axes (limit_linear_coupled / motor_linear_coupled, joint_constraint_helper.rs:210-283, :333-409)
    auto coupled_linear_row = [&](float& dist) {
        GRow r;
        vec3 lj = zero3(), a1 = zero3(), a2 = zero3();
        for (int i = 0; i < 3; ++i) {
            if (!(coupled & (1u << i))) continue;
            const float coeff = dot3(bc[i], lin_err);
            lj = lj + bc[i] * coeff;
            a1 = a1 + cross3(r1, bc[i]) * coeff;
            a2 = a2 + cross3(r2, bc[i]) * coeff;
        }
        dist = sqrtf(dot3(lj, lj));
        const float inv_dist = safe_inv(dist);
        r.lin = lj * inv_dist; r.a1 = a1 * inv_dist; r.a2 = a2 * inv_dist;
        r.ia1 = smul(g1.ii, r.a1); r.ia2 = smul(g2.ii, r.a2);
        r.inv_lhs = 0.0f;
        return r;
    };
    if ((motor_axes & coupled) & 7u) {   // motor_linear_coupled (:228-250); coupled angular motors build no row (:224-226)
        float4 ma; float m_erp, m_cc, m_cg, max_imp;
        motor_coeffs(first_lin, ma, m_erp, m_cc, m_cg, max_imp);
        float dist;
        GRow r = coupled_linear_row(dist);
        float rwb = 0.0f;
        if (m_erp != 0.0f) rwb = rwb + (dist - ma.y) * m_erp;
        float target_vel = ma.x;
        if (limit_axes & (1u << first_lin)) {
            const float2 lim = w.j_limits[j * 6 + first_lin];
            target_vel = clampf(target_vel, (lim.x - dist) * inv_dt, (lim.y - dist) * inv_dt);
        }
        rwb = rwb + -target_vel;
        r.cc = m_cc; r.cg = m_cg; r.lo = -max_imp; r.hi = max_imp; r.rhs = rwb; r.rwb = rwb;
        r.dof = first_lin; r.kind = 2;
        rows[len++] = r;
    }
    grows_finalize(rows, 0, len, imsum);
    const int start = len;
    for (int i = 3; i < 6; ++i) {   // lock_angular
        if (!(locked & (1u << i))) continue;
        const int ax = i - 3;
        const float av = comp(a, ax), bv = comp(b, ax);
        const float dg = wa * wb - ab;
        const vec3 cx = ax == 0 ? mk3(0.0f, -cv.z, cv.y) : (ax == 1 ? mk3(cv.z, 0.0f, -cv.x) : mk3(-cv.y, cv.x, 0.0f));
        const vec3 row = mk3((av * b.x + (ax == 0 ? dg : 0.0f) - cx.x + bv * a.x) * 0.5f,
                             (av * b.y + (ax == 1 ? dg : 0.0f) - cx.y + bv * a.y) * 0.5f,
                             (av * b.z + (ax == 2 ? dg : 0.0f) - cx.z + bv * a.z) * 0.5f);
        const vec3 aj = row * sgn;
        GRow& r = rows[len++];
        r.lin = zero3(); r.a1 = aj; r.a2 = aj; r.ia1 = smul(g1.ii, aj); r.ia2 = smul(g2.ii, aj);
        r.inv_lhs = 0.0f; r.cc = cfm_coeff; r.cg = 0.0f; r.rwb = 0.0f;
        r.rhs = 0.0f + aerr[ax] * erp_inv_dt;
        r.lo = -FMAX32; r.hi = FMAX32; r.dof = i; r.kind = 0;
    }
    for (int i = 0; i < 3; ++i)
        if (locked & (1u << i)) rows[len++] = lock_linear_row(i, erp_inv_dt, cfm_coeff, i, 0);
    for (int i = 3; i < 6; ++i) {   // limit_angular on the re-centred angle
        if (!((limit_axes & ~coupled) & (1u << i))) continue;
        const int ax = i - 3;
        const float4 al = w.j_anglim[j * 3 + ax];
        const float x = aerr[ax];
        const float sin_half = al.x * x - al.y * aew, cos_half = al.x * aew + al.y * x;
        float half = atan2_poly(sin_half, cos_half);
        if (fabs1(half) > 1.5707964f) half = half - copysignf(3.1415927f, half);
        const float ang = half * 2.0f;
        const bool min_enabled = ang <= -al.z, max_enabled = al.z <= ang;
        const vec3 aj = bc[ax];
        const float rhs_bias = clampf((max2(ang - al.z, 0.0f) - max2(-al.z - ang, 0.0f)) * erp_inv_dt, -max_bias, max_bias);
        GRow& r = rows[len++];
        r.lin = zero3(); r.a1 = aj; r.a2 = aj; r.ia1 = smul(g1.ii, aj); r.ia2 = smul(g2.ii, aj);
        r.inv_lhs = 0.0f; r.cc = cfm_coeff; r.cg = 0.0f; r.rwb = 0.0f;
        r.rhs = 0.0f + rhs_bias;
        r.lo = min_enabled ? -RB_INF : 0.0f; r.hi = max_enabled ? RB_INF : 0.0f; r.dof = i; r.kind = 1;
    }
    for (int i = 0; i < 3; ++i) {   // limit_linear
        if (!((limit_axes & ~coupled) & (1u << i))) continue;
        GRow r = lock_linear_row(i, erp_inv_dt, cfm_coeff, i, 1);
        const float dist = dot3(lin_err, r.lin);
        const float2 lim = w.j_limits[j * 6 + i];
        const bool min_enabled = dist <= lim.x, max_enabled = lim.y <= dist;
        const float rhs_bias = clampf((max2(dist - lim.y, 0.0f) - max2(lim.x - dist, 0.0f)) * erp_inv_dt, -max_bias, max_bias);
        r.rhs = r.rwb + rhs_bias;
        r.cc = cfm_coeff;
        r.lo = min_enabled ? -RB_INF : 0.0f; r.hi = max_enabled ? RB_INF : 0.0f;
        rows[len++] = r;
    }
    if (has_ang_coupling && (limit_axes & (1u << first_ang))) {   // limit_angular_coupled (joint_constraint_helper.rs:725-798): two coupled angular axes
        const unsigned ac = coupled >> 3;
        const int not_coupled = (ac & 1u) == 0 ? 0 : ((ac & 2u) == 0 ? 1 : ((ac & 4u) == 0 ? 2 : 3));
        if (not_coupled < 3) {
            const mat3 basis2 = rotmat(f2.q);
            const vec3 axis1 = bc[not_coupled], axis2 = not_coupled == 0 ? basis2.c0 : (not_coupled == 1 ? basis2.c1 : basis2.c2);
            // Rot3::from_rotation_arc(axis1, axis2).to_axis_angle() (glam, restated; atan2 by the shared polynomial)
            const float d = dot3(axis1, axis2);
            const float one_minus_eps = 1.0f - 2.0f * 1.1920929e-7f;
            float qx, qy, qz, qw;
            if (d > one_minus_eps) { qx = 0.0f; qy = 0.0f; qz = 0.0f; qw = 1.0f; }
            else if (d < -one_minus_eps) {
                const float sg = copysign1(axis1.z), aa = -1.0f / (sg + axis1.z), bb = axis1.x * axis1.y * aa;
                qx = bb; qy = sg + axis1.y * axis1.y * aa; qz = -axis1.y; qw = -4.371139e-8f;
            } else {
                const vec3 c = cross3(axis1, axis2);
                const float ww = 1.0f + d;
                const float inv = 1.0f / sqrtf(c.x * c.x + c.y * c.y + c.z * c.z + ww * ww);
                qx = c.x * inv; qy = c.y * inv; qz = c.z * inv; qw = ww * inv;
            }
            vec3 aj = mk3(1.0f, 0.0f, 0.0f);
            float angle = 0.0f;
            const vec3 v = mk3(qx, qy, qz);
            const float vl = sqrtf(dot3(v, v));
            if (vl >= 1.0e-8f) { angle = 2.0f * atan2_poly(vl, qw); aj = v * (1.0f / vl); }
            if (angle == 0.0f) {   // axis1.orthonormal_basis()[0]
                const float sg = copysign1(axis1.z), aa = -1.0f / (sg + axis1.z), bb = axis1.x * axis1.y * aa;
                aj = mk3(1.0f + sg * axis1.x * axis1.x * aa, sg * bb, -sg * axis1.x);
            }
            const float2 lim = w.j_limits[j * 6 + first_ang];
            const bool min_enabled = angle <= lim.x, max_enabled = lim.y <= angle;
            const float rhs_bias = clampf((max2(angle - lim.y, 0.0f) - max2(lim.x - angle, 0.0f)) * erp_inv_dt, -max_bias, max_bias);
            GRow& r = rows[len++];
            r.lin = zero3(); r.a1 = aj; r.a2 = aj; r.ia1 = smul(g1.ii, aj); r.ia2 = smul(g2.ii, aj);
            r.inv_lhs = 0.0f; r.cc = cfm_coeff; r.cg = 0.0f; r.rwb = 0.0f;
            r.rhs = 0.0f + rhs_bias;
            r.lo = min_enabled ? -RB_INF : 0.0f; r.hi = max_enabled ? RB_INF : 0.0f; r.dof = first_ang; r.kind = 1;
        }
    }
    if (has_lin_coupling && (limit_axes & (1u << first_lin))) {   // limit_linear_coupled (:210-283): the maximum distance only
        float dist;
        GRow r = coupled_linear_row(dist);
        const float hi = w.j_limits[j * 6 + first_lin].y;
        r.rwb = min2(dist - hi, 0.0f) * inv_dt;
        const float rhs_bias = clampf(max2(dist - hi, 0.0f) * erp_inv_dt, -max_bias, max_bias);
        r.rhs = r.rwb + rhs_bias;
        r.cc = cfm_coeff; r.cg = 0.0f;
        r.lo = 0.0f; r.hi = RB_INF; r.dof = first_lin; r.kind = 1;
        rows[len++] = r;
    }
    grows_finalize(rows, start, len, imsum);
    const size_t rs = (size_t)JROWS_GENERIC * w.joint_cap;   // row stride of the generic row tables
    for (int k = 0; k < len; ++k) {
        const size_t s = (size_t)JROWS_GENERIC * q + k;
        const GRow& r = rows[k];
        // the impulse restarts from 0, or with warmstart_joints from last step's written-back impulse (first substep) /
        // the same row of the previous substep, scaled by warmstart_coefficient (joint_constraint_builder.rs:116-150)
        float imp = 0.0f;
        if (w.prm.warmstart_joints) {
            const float* src = r.kind == 0 ? w.j_impulses : (r.kind == 1 ? w.j_limit_impulses : w.j_motor_impulses);
            const float seed = sub > 0 ? w.j_rows[JR_LIN * rs + s].w : src[j * 6 + r.dof];
            imp = seed * w.prm.warmstart_coeff;
        }
        w.j_rows[JR_LIN * rs + s] = f4(r.lin, imp);
        w.j_rows[JR_A1 * rs + s] = f4(r.a1, r.inv_lhs);
        w.j_rows[JR_A2 * rs + s] = f4(r.a2, r.rhs);
        w.j_rows[JR_IA1 * rs + s] = f4(r.ia1, r.rwb);
        w.j_rows[JR_IA2 * rs + s] = f4(r.ia2, r.cg);
        w.j_bnd[s] = make_float4(r.lo, r.hi, as_float_i(r.dof), as_float_i(r.kind));
    }
    h.w = len;
    w.j_sched_ids[q] = h;
}
template <class B>
RB_HD void joint_solve_generic(const World& w, const B& bd, int q, bool wo_bias, bool warm) {   // solve_generic with impulse_bounds (joint_velocity_constraint.rs:97-120)
    const int4 h = w.j_sched_ids[q];
    const int id1 = h.y, id2 = h.z, len = h.w;
    BodyState g1 = gather_body(bd, id1), g2 = gather_body(bd, id2);
    vec3 v1 = g1.lin, w1 = g1.ang, v2 = g2.lin, w2 = g2.ang;
    const size_t rs = (size_t)JROWS_GENERIC * w.joint_cap;
    for (int k = 0; k < len; ++k) {
        const size_t s = (size_t)JROWS_GENERIC * q + k;
        float4 L = w.j_rows[JR_LIN * rs + s], A1 = w.j_rows[JR_A1 * rs + s], A2 = w.j_rows[JR_A2 * rs + s];
        const float4 I1 = w.j_rows[JR_IA1 * rs + s], I2 = w.j_rows[JR_IA2 * rs + s], bnd = w.j_bnd[s];
        if (warm) {   // warmstart_generic (joint_velocity_constraint.rs:129-141): the carried impulse, right before the row's solve
            const vec3 wl = xyz(L) * L.w;
            v1 = madd3v(v1, wl, g1.im);
            w1 = madd3(w1, xyz(I1), L.w);
            v2 = madd3v(v2, -wl, g2.im);
            w2 = madd3(w2, xyz(I2), -L.w);
        }
        const float rhs_c = wo_bias ? I1.w : A2.w;
        const float dlin = dot3(xyz(L), v2 - v1);
        const float dang = dot3(xyz(A2), w2) - dot3(xyz(A1), w1);
        const float rhs = dlin + dang + rhs_c;
        const float total = clampf(L.w + A1.w * (rhs - I2.w * L.w), bnd.x, bnd.y);
        const float delta = total - L.w;
        L.w = total;
        const vec3 li = xyz(L) * delta;
        v1 = madd3v(v1, li, g1.im);
        w1 = madd3(w1, xyz(I1), delta);
        v2 = madd3v(v2, -li, g2.im);
        w2 = madd3(w2, xyz(I2), -delta);
        w.j_rows[JR_LIN * rs + s] = L;
        if (wo_bias) { A2.w = I1.w; w.j_rows[JR_A2 * rs + s] = A2; }
    }
    scatter_vel(bd, id1, v1, w1);
    scatter_vel(bd, id2, v2, w2);
}
RB_HD void joint_writeback_generic(const World& w, int q) {
    const int4 h = w.j_sched_ids[q];
    const size_t rs = (size_t)JROWS_GENERIC * w.joint_cap;
    for (int k = 0; k < h.w; ++k) {
        const size_t s = (size_t)JROWS_GENERIC * q + k;
        const float4 bnd = w.j_bnd[s];
        const int dof = as_int(bnd.z), kind = as_int(bnd.w);
        float* dst = kind == 0 ? w.j_impulses : (kind == 1 ? w.j_limit_impulses : w.j_motor_impulses);
        dst[h.x * 6 + dof] = w.j_rows[JR_LIN * rs + s].w;
    }
}

// rigid_body_components.rs:528-572 for body b at pose p; writes world_com / effective masses.
RB_HD void update_world_mass(const World& w, int b, const pose& p) {
    float4 lc = w.b_lcom_im[b];
    bool dyn = w.b_type[b] == BODY_DYNAMIC;
    unsigned fl = w.b_flags[b];
    w.b_wcom[b] = f4(xform(p, xyz(lc)), 0.0f);
    vec3 im = mk3(lc.w, lc.w, lc.w);
    vec3 d = xyz(w.b_ipi[b]);
    sym3 m = sym_zero();
    if (d.x != 0.0f || d.y != 0.0f || d.z != 0.0f) {
        mat3 r = rotmat(qmul(p.q, mkq(w.b_pframe[b])));
        m.xx = (r.c0.x * d.x) * r.c0.x + (r.c1.x * d.y) * r.c1.x + (r.c2.x * d.z) * r.c2.x;
        m.xy = (r.c0.x * d.x) * r.c0.y + (r.c1.x * d.y) * r.c1.y + (r.c2.x * d.z) * r.c2.y;
        m.xz = (r.c0.x * d.x) * r.c0.z + (r.c1.x * d.y) * r.c1.z + (r.c2.x * d.z) * r.c2.z;
        m.yy = (r.c0.y * d.x) * r.c0.y + (r.c1.y * d.y) * r.c1.y + (r.c2.y * d.z) * r.c2.y;
        m.yz = (r.c0.y * d.x) * r.c0.z + (r.c1.y * d.y) * r.c1.z + (r.c2.y * d.z) * r.c2.z;
        m.zz = (r.c0.z * d.x) * r.c0.z + (r.c1.z * d.y) * r.c1.z + (r.c2.z * d.z) * r.c2.z;
    }
    if (!dyn || (fl & FLAG_LTX)) im.x = 0.0f;
    if (!dyn || (fl & FLAG_LTY)) im.y = 0.0f;
    if (!dyn || (fl & FLAG_LTZ)) im.z = 0.0f;
    if (!dyn || (fl & FLAG_LRX)) { m.xx = 0.0f; m.xy = 0.0f; m.xz = 0.0f; }
    if (!dyn || (fl & FLAG_LRY)) { m.yy = 0.0f; m.xy = 0.0f; m.yz = 0.0f; }
    if (!dyn || (fl & FLAG_LRZ)) { m.zz = 0.0f; m.xz = 0.0f; m.yz = 0.0f; }
    w.b_eim[b] = f4(im, 0.0f);
    w.b_eii0[b] = make_float4(m.xx, m.xy, m.xz, m.yy);
    w.b_eii1[b] = make_float2(m.yz, m.zz);
}

// The queued CCD clamps (see body_writeback): sweep_fast_body + apply_clamps (ccd_solver.rs:162-238, :325-340), then
// advance_to_final_positions for the clamped bodies.  `n` = State::nccd read before the call; the caller resets it.
// `bullets`: false = the first pass (fast non-bullets against the fixed colliders), true = the second one (bullets against
// everything but bullets, at the poses the first pass left); the caller puts a barrier between the two.
template <class Ctx>
RB_PHASE void phase_ccd_pending(const Ctx& ctx, const World& w, int n, bool bullets) {
    for (int k = ctx.gtid; k < n; k += ctx.gsize) {
        const int b = w.ccd_list[k];
        if (w.b_type[b] != BODY_DYNAMIC) continue;
        if (((w.b_flags[b] & FLAG_CCD) != 0) != bullets) continue;
        const pose op = mkpose(mkq(w.ccd_start_q[b]), xyz(w.ccd_start_t[b])), np = body_pose(w, b);
        const pose cl = ccd_clamp_body(w, b, op, np, bullets);
        w.b_pos_t[b] = f4(cl.t, 0.0f);
        w.b_pos_q[b] = f4(cl.q);
        update_world_mass(w, b, cl);
        float* s = w.state13 + (size_t)b * 13;
        s[0] = cl.t.x; s[1] = cl.t.y; s[2] = cl.t.z; s[3] = cl.q.x; s[4] = cl.q.y; s[5] = cl.q.z; s[6] = cl.q.w;
    }
}

// NarrowPhase::emit_contact_force_events (solver_graph.rs:462-498) + ContactForceEvent::from_contact_pair (geometry/mod.rs:
// 223-258), after the impulse writeback: solver-active pairs whose colliders ask for force events and whose total
// normal impulse / dt exceeds the smaller threshold.  `started` = the pair was not above its threshold last step.
template <class Ctx>
RB_PHASE void phase_force_events(const Ctx& ctx, const World& w) {
    State* st = w.st;
    const int buf = st->cur, np = st->npairs;
    for (int i = ctx.gtid; i < np; i += ctx.gsize) {
        float4 info = prow(w, buf, PR_INFO, i);
        if (!pair_has_forces(w, info)) continue;
        const int nsc = as_int(info.z);
        const unsigned long long key = w.pb[buf].key[i];
        const int c1 = (int)(key >> 32), c2 = (int)(key & 0xffffffffu);
        const float t1 = (w.c_events[c1] & EV_CONTACT_FORCE) ? w.c_force_thr[c1] : FMAX32;
        const float t2 = (w.c_events[c2] & EV_CONTACT_FORCE) ? w.c_force_thr[c2] : FMAX32;
        const float threshold = min2(t1, t2);
        if (!(threshold < FMAX32)) continue;
        const float4 bod = prow(w, buf, PR_BODIES, i);
        if (!body_is_sim(w, as_int(bod.z)) && !body_is_sim(w, as_int(bod.w))) continue;
        float total = 0.0f, maxi = 0.0f;
        for (int k = 0; k < nsc && k < MAX_PTS; ++k) {
            const int cid = as_int(prow(w, buf, PR_A1 + k, i).w);
            const float imp = prow(w, buf, PR_PD + cid, i).x;
            total = total + imp;
            if (imp > maxi) maxi = imp;
        }
        const float magnitude = total * w.prm.inv_dt_full;
        int flags = as_int(info.x);
        if (magnitude > threshold) {
            const vec3 n = xyz(prow(w, buf, PR_NORMAL, i));
            const vec3 tf = (n * total) * w.prm.inv_dt_full;
            const int slot = atomic_add(&st->nev_force, 1);
            if (slot < w.ev_cap) {
                w.ev_force[slot] = make_float4(as_float_i(c1), as_float_i(c2), as_float_i((flags & PF_FORCE_EVENT) ? 0 : 1), as_float_i(w.step_index));
                w.ev_force[w.ev_cap + slot] = f4(tf, magnitude);
                w.ev_force[2 * w.ev_cap + slot] = f4(maxi > 0.0f ? n : zero3(), maxi * w.prm.inv_dt_full);
            } else RB_RAISE(w, STATUS_CAPACITY);
            flags |= PF_FORCE_EVENT;
        } else flags &= ~PF_FORCE_EVENT;
        if (flags != as_int(info.x)) { info.x = as_float_i(flags); prow(w, buf, PR_INFO, i) = info; }
    }
}

// Executors: how the threads of an item iterate and synchronise.
struct BlockExec {
    const BlockCtx* c;
    RB_HD int tid() const { return c->btid; }
    RB_HD int nth() const { return c->bsize; }
    RB_HD void sync() const { c->block_sync(); }
};
struct GridExec {
    const GridCtx* c;
    RB_HD int tid() const { return c->gtid; }
    RB_HD int nth() const { return c->gsize; }
    RB_HD void sync() const { c->grid_sync(); }
};

// Grid-wide executor that deals consecutive WARPS of work to different CTAs: a colour stage with a few hundred
// constraints then runs on a few warps of EVERY SM instead of filling the first SMs and leaving the rest idle.
struct GridSpreadExec {
    const GridCtx* c;
    RB_HD int tid() const { return ((c->btid / c->nlanes) * c->nblocks + c->bid) * c->nlanes + c->lane; }
    RB_HD int nth() const { return c->gsize; }
    RB_HD void sync() const { c->grid_sync(); }
};

// ---- body phases shared by every solve path -------------------------------------------------------
// a7 + S1: forces, solver bodies, per-substep increments (solve.rs:234-291; solver_body.rs:82-121; worker.rs:46-104)
template <class B>
RB_HD void body_init(const World& w, const B& bd, int b, int id, vec3 gravity) {
    const Params& P = w.prm;
    float4 lc = w.b_lcom_im[b];
    vec3 eim = xyz(w.b_eim[b]);
    sym3 eii = load_ii(w, b);
    float4 misc = w.b_misc[b];
    vec3 emass = mk3(inv_exact0(eim.x), inv_exact0(eim.y), inv_exact0(eim.z));
    vec3 force = xyz(w.b_uforce[b]) + had(gravity, emass) * misc.z;
    vec3 torque = xyz(w.b_utorque[b]);
    bd.set_vel(id, xyz(w.b_linvel[b]), xyz(w.b_angvel[b]));
    bd.set_xf(id, prepend_translation(body_pose(w, b), xyz(lc)));
    bd.set_mass(id, eii, eim);
    bd.set_incr(id, had(force, eim) * P.sub_dt, smul(eii, torque) * P.sub_dt);
}
// S3: velocity increment + gyroscopic correction (worker.rs:235-284)
template <class B>
RB_HD void body_increment(const World& w, const B& bd, int b, int id) {
    vec3 lin = bd.lin(id) + bd.incr_lin(id);
    vec3 ang = bd.ang(id) + bd.incr_ang(id);
    if (w.b_flags[b] & FLAG_GYRO) {
        quat axes = qmul(bd.xf(id).q, mkq(w.b_pframe[b]));
        ang = gyro_corrected(ang, axes, xyz(w.b_pi[b]), xyz(w.b_ipi[b]), w.prm.sub_dt);
    }
    bd.set_vel(id, lin, ang);
}
// S7: speed caps + linearised pose integration (worker.rs:568-631; rigid_body_components.rs:884-898)
template <class B>
RB_HD void body_integrate(const World& w, const B& bd, int b, int id) {
    const Params& P = w.prm;
    vec3 lin = bd.lin(id), ang = bd.ang(id);
    if (P.max_lin_vel != FMAX32) {
        float n = norm(lin);
        if (n > P.max_lin_vel) lin = lin * (P.max_lin_vel / n);
    }
    if (!(w.b_flags[b] & FLAG_FAST_ROT)) {
        float n = norm(ang);
        if (n > P.max_ang_vel) ang = ang * (P.max_ang_vel / n);
    }
    bd.set_vel(id, lin, ang);
    pose p = bd.xf(id);
    vec3 hang = ang * (P.sub_dt * 0.5f);
    quat dq; dq.x = hang.x; dq.y = hang.y; dq.z = hang.z; dq.w = 1.0f;
    p.q = qnormalize(qmul(dq, p.q));
    p.t = madd3(p.t, lin, P.sub_dt);
    bd.set_xf(id, p);
}
// S11 + advance_to_final_positions (worker.rs:809-897; substep.rs:84-224)
template <class B>
RB_HD void body_writeback(const World& w, const B& bd, int b, int id) {
    const Params& P = w.prm;
    float4 misc = w.b_misc[b];
    // (what the CCD test below reads is fetched here, with the other loads, so that it adds no round trip of its own)
    pose ccd_op = pident();
    float ccd_ext = 0.0f, ccd_thick = 0.0f;
    if (P.ccd) { ccd_op = body_pose(w, b); ccd_ext = w.b_ipi[b].w; ccd_thick = misc.w; }   // (copies of b_max_extent / b_ccd_thick in rows this function reads anyway)
    vec3 lin = bd.lin(id) * (1.0f / (1.0f + P.dt * misc.x));
    vec3 ang = bd.ang(id) * (1.0f / (1.0f + P.dt * misc.y));
    pose np = prepend_translation(bd.xf(id), -xyz(w.b_lcom_im[b]));
    // (a position-based kinematic body keeps exactly the pose its user asked for: worker.rs:836-842)
    if (w.b_type[b] == BODY_KIN_POS) np = mkpose(mkq(w.b_next_q[b]), xyz(w.b_next_t[b]));
    if (!(finite3(lin) && finite3(ang) && finite3(np.t) && isfinite(np.q.x) && isfinite(np.q.y) && isfinite(np.q.z) && isfinite(np.q.w))) {
        // Containment of non-finite state at the end-of-step chokepoint (physics_pipeline/quarantine.rs:14-47, :126-178):
        // the body keeps its last valid pose, loses its velocities and forces, is disabled (its colliders leave the
        // broad phase at the next step) and is reported through rb_world_get_quarantine; the step raises RB_ERR_NONFINITE.
        w.b_linvel[b] = make_float4(0.f, 0.f, 0.f, 0.f);
        w.b_angvel[b] = make_float4(0.f, 0.f, 0.f, 0.f);
        w.b_uforce[b] = make_float4(0.f, 0.f, 0.f, 0.f);
        w.b_utorque[b] = make_float4(0.f, 0.f, 0.f, 0.f);
        w.b_type[b] = BODY_REMOVED;
        float* s = w.state13 + (size_t)b * 13;
        for (int k = 7; k < 13; ++k) s[k] = 0.0f;
        const int slot = atomic_add(&w.st->nquarantine, 1);
        if (slot < w.nb) w.quarantine[slot] = b;
        w.st->lists_dirty = 3; w.st->bp_dirty = 1; w.st->sched_dirty = 1;
        RB_RAISE(w, STATUS_NONFINITE);
        return;
    }
    if (P.ccd && w.b_type[b] == BODY_DYNAMIC && ccd_is_moving_fast(P, xyz(w.b_lcom_im[b]), ccd_op, np, ccd_ext, ccd_thick)) {
        // CCD (substep.rs:492-520): a body whose solved motion exceeds half its thinnest extent is queued for motion clamping
        // with its start pose; the sweep itself (rb_ccd.cuh) runs at the start of the next step's
        // k_collide or at the next synchronising call (k_ccd_pending), so the solve kernels carry only this test.
        w.ccd_start_t[b] = f4(ccd_op.t, 0.0f);
        w.ccd_start_q[b] = f4(ccd_op.q);
        w.ccd_list[atomic_add(&w.st->nccd, 1)] = b;
        if (w.b_flags[b] & FLAG_CCD) atomic_add(&w.st->nccd_bullets, 1);
        atomic_add(&w.st->ccd_total, 1);
        w.host_hint[3] = 1;
    }
    w.b_linvel[b] = f4(lin, 0.0f);
    w.b_angvel[b] = f4(ang, 0.0f);
    w.b_pos_t[b] = f4(np.t, 0.0f);
    w.b_pos_q[b] = f4(np.q);
    update_world_mass(w, b, np);
    float* s = w.state13 + (size_t)b * 13;
    s[0] = np.t.x; s[1] = np.t.y; s[2] = np.t.z; s[3] = np.q.x; s[4] = np.q.y; s[5] = np.q.z; s[6] = np.q.w;
    s[7] = lin.x; s[8] = lin.y; s[9] = lin.z; s[10] = ang.x; s[11] = ang.y; s[12] = ang.z;
}

// =====================================================================================================
// Lane-cooperative shared-memory path: the island's bodies AND constraints live in shared memory for
// the whole step; each constraint is swept by L consecutive lanes (L = 4 on the GPU: one lane per
// manifold point), which compute the per-point jacobians / rhs in parallel and resolve the sequential
// Gauss-Seidel dependency between the points with __shfl_sync broadcasts.  Same primitives, same
// arithmetic, same results as the serial sweep.
// =====================================================================================================
// per-point float4 rows (one copy per manifold point)
enum CoopPointRow { PR4_TD1R = 0,   // torque_dir1 xyz, r (projected mass)
                    PR4_TD2D,       // torque_dir2 xyz, dist0
                    PR4_ITD1I,      // ii1*torque_dir1 xyz, id1 bits
                    PR4_ITD2A,      // ii2*torque_dir2 xyz, id2 bits
                    PR4_LP1,        // builder anchor on body 1 (body-local) xyz, contact slot (bits)
                    PR4_LP2,        // builder anchor on body 2 xyz, pair-table row (bits)
                    PR4_COUNT };
// per-constraint float4 rows
enum CoopConsRow { CR4_DIRF = 0,    // dir1 xyz, friction
                   CR4_T1W,         // tangent1 xyz, twist effective mass
                   CR4_TR,          // tangent K (r0 r1 r2), nc bits
                   CR4_TWD,         // twist_dists[4]
                   CR4_J0, CR4_J1, CR4_J2, CR4_J3, CR4_J4, CR4_J5, CR4_J6, CR4_J7,   // friction jacobians, packed (see put/get)
                   CR4_COUNT };
constexpr int COOP_ROWS = PR4_COUNT * MAX_PTS + CR4_COUNT;   // 36 float4 = 576 B per constraint, constant during a step
// mutable float4 rows (always resident in shared memory): the impulses
enum CoopMutRow { MR_IMP = 0,       // normal impulses of the 4 points
                  MR_ACC,           // their accumulators
                  MR_TI,            // tangent impulse xy, accumulators zw
                  MR_WI,            // twist impulse, accumulator
                  MR_DIST,          // separation of the 4 points at the poses of the last position integration
                  MR_COUNT };
constexpr int COOP_MIN_CHUNK = 8;      // smallest streaming chunk worth running (slots)
constexpr int COOP_MAX_CHUNKS = 640;   // chunk table of a streamed item (colour stages + splits of long stages)

// A window of constraint slots stored row-major (row r of slot s at p[r * stride + s]): the item's
// resident shared-memory copy, one staging buffer of the streaming pipeline, or the L2-resident pool.
// Odd strides keep the 4 point-lanes of a constraint on distinct 16-byte bank groups.
struct RowView {
    float4* p;
    int stride;
    RB_HD float4& pp(int row, int k, int s) const { return p[(row * MAX_PTS + k) * stride + s]; }
    RB_HD float4& pc(int row, int s) const { return p[(PR4_COUNT * MAX_PTS + row) * stride + s]; }
    RB_HD float4& mr(int row, int s) const { return p[row * stride + s]; }                                  // mutable rows
    RB_HD float& mf(int row, int k, int s) const { return reinterpret_cast<float*>(p + row * stride + s)[k]; }
};

// How one item maps onto the CTA's shared memory (a pure function of the item's sizes and the
// launch's shared-memory size, so both kernels agree on it).
struct CoopPlan {
    int body_slots;   // nb + 2: the item's bodies, the world pseudo body, the garbage slot
    int mstride;      // slot stride of the mutable rows
    int resident;     // 1: every constraint lives in shared memory for the whole step
    int stride;       // resident: slot stride of the constant rows; streaming: slots per staging buffer
    bool ok;
};
RB_HD CoopPlan coop_plan(int smem_floats, int nb, int n) {
    CoopPlan pl;
    pl.body_slots = nb + 2;
    pl.mstride = n | 1;
    const int avail = (smem_floats - pl.body_slots * SB_STRIDE) / 4 - MR_COUNT * pl.mstride;   // float4 left for constant rows
    const int R = avail > 0 ? avail / COOP_ROWS : 0;
    pl.resident = pl.mstride <= R ? 1 : 0;
    pl.stride = pl.resident ? pl.mstride : ((R / 2 - 1) | 1);
    pl.ok = pl.resident || ((R / 2 - 1) >= COOP_MIN_CHUNK && n / pl.stride + NUM_COLORS + 2 <= COOP_MAX_CHUNKS);
    return pl;
}

RB_HD void coop_put_jac(const RowView& cs, int s, const FrictionJac& j) {
    cs.pc(CR4_J0, s) = make_float4(j.td10.x, j.td10.y, j.td10.z, j.td11.x);
    cs.pc(CR4_J1, s) = make_float4(j.td11.y, j.td11.z, j.td20.x, j.td20.y);
    cs.pc(CR4_J2, s) = make_float4(j.td20.z, j.td21.x, j.td21.y, j.td21.z);
    cs.pc(CR4_J3, s) = make_float4(j.i10.x, j.i10.y, j.i10.z, j.i11.x);
    cs.pc(CR4_J4, s) = make_float4(j.i11.y, j.i11.z, j.i20.x, j.i20.y);
    cs.pc(CR4_J5, s) = make_float4(j.i20.z, j.i21.x, j.i21.y, j.i21.z);
    cs.pc(CR4_J6, s) = make_float4(j.tw1.x, j.tw1.y, j.tw1.z, j.tw2.x);
    cs.pc(CR4_J7, s) = make_float4(j.tw2.y, j.tw2.z, 0.0f, 0.0f);
}
RB_HD FrictionJac coop_get_jac(const RowView& cs, int s) {
    float4 a = cs.pc(CR4_J0, s), b = cs.pc(CR4_J1, s), c = cs.pc(CR4_J2, s), d = cs.pc(CR4_J3, s), e = cs.pc(CR4_J4, s),
           f = cs.pc(CR4_J5, s), g = cs.pc(CR4_J6, s), h = cs.pc(CR4_J7, s);
    FrictionJac j;
    j.td10 = mk3(a.x, a.y, a.z); j.td11 = mk3(a.w, b.x, b.y); j.td20 = mk3(b.z, b.w, c.x); j.td21 = mk3(c.y, c.z, c.w);
    j.i10 = mk3(d.x, d.y, d.z); j.i11 = mk3(d.w, e.x, e.y); j.i20 = mk3(e.z, e.w, f.x); j.i21 = mk3(f.y, f.z, f.w);
    j.tw1 = mk3(g.x, g.y, g.z); j.tw2 = mk3(g.w, h.x, h.y);
    return j;
}

// Store one generated constraint in its row window, with the jacobians that stay constant during
// the step precomputed (the serial path recomputes the same expressions in every sweep).
template <class B>
RB_HD void coop_put(const RowView& cs, const RowView& mu, const B& bd, int s, const Cons& c) {
    BodyState g1 = gather_body(bd, c.id1), g2 = gather_body(bd, c.id2);
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        PointPre pj;
        pj.td1 = pj.td2 = pj.itd1 = pj.itd2 = zero3();
        float r = 0.0f, d0 = 0.0f;
        vec3 l1 = zero3(), l2 = zero3();
        if (k < c.nc) {
            point_jac(g1, g2, c.dir, c.dp1[k], c.dp2[k], pj);
            r = c.r[k]; d0 = c.dist0[k]; l1 = c.lp1[k]; l2 = c.lp2[k];
        }
        cs.pp(PR4_TD1R, k, s) = f4(pj.td1, r);
        cs.pp(PR4_TD2D, k, s) = f4(pj.td2, d0);
        cs.pp(PR4_ITD1I, k, s) = f4(pj.itd1, as_float_i(c.id1));
        cs.pp(PR4_ITD2A, k, s) = f4(pj.itd2, as_float_i(c.id2));
        cs.pp(PR4_LP1, k, s) = f4(l1, as_float_i(c.cid[k]));
        cs.pp(PR4_LP2, k, s) = f4(l2, as_float_i(c.pair));
    }
    const vec3 t2 = cross3(c.dir, c.t1);
    coop_put_jac(cs, s, friction_jac(g1, g2, c.dir, c.t1, t2, c.tdp1, c.tdp2));
    cs.pc(CR4_DIRF, s) = f4(c.dir, c.fric);
    cs.pc(CR4_T1W, s) = f4(c.t1, c.wr);
    cs.pc(CR4_TR, s) = make_float4(c.tr0, c.tr1, c.tr2, as_float_i(c.nc));
    cs.pc(CR4_TWD, s) = make_float4(c.twd[0], c.twd[1], c.twd[2], c.twd[3]);
    mu.mr(MR_IMP, s) = make_float4(c.imp[0], c.imp[1], c.imp[2], c.imp[3]);
    mu.mr(MR_ACC, s) = make_float4(c.acc[0], c.acc[1], c.acc[2], c.acc[3]);
    mu.mr(MR_TI, s) = make_float4(c.ti0, c.ti1, c.ta0, c.ta1);
    mu.mr(MR_WI, s) = make_float4(c.wi, c.wa, 0.0f, 0.0f);
    // separation at the initial poses: what the first biased sweep needs (later ones reuse the relax sweep's)
    float ds[MAX_PTS];
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        ds[k] = 0.0f;
        if (k < c.nc) ds[k] = c.dist0[k] + dot3(xform(g1.p, c.lp1[k]) - xform(g2.p, c.lp2[k]), c.dir);
    }
    mu.mr(MR_DIST, s) = make_float4(ds[0], ds[1], ds[2], ds[3]);
}
RB_HD void coop_get_for_writeback(const RowView& cs, const RowView& mu, int s, Cons& c) {
    c.nc = as_int(cs.pc(CR4_TR, s).w);
    c.dir = xyz(cs.pc(CR4_DIRF, s)); c.t1 = xyz(cs.pc(CR4_T1W, s));
    c.pair = as_int(cs.pp(PR4_LP2, 0, s).w);
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) c.cid[k] = as_int(cs.pp(PR4_LP1, k, s).w);
    const float4 im = mu.mr(MR_IMP, s), ac = mu.mr(MR_ACC, s), ti = mu.mr(MR_TI, s);
    c.imp[0] = im.x; c.imp[1] = im.y; c.imp[2] = im.z; c.imp[3] = im.w;
    c.acc[0] = ac.x; c.acc[1] = ac.y; c.acc[2] = ac.z; c.acc[3] = ac.w;
    c.ti0 = ti.x; c.ti1 = ti.y; c.wi = mu.mr(MR_WI, s).x;
}

// Sub-warp broadcast from lane `src` of each L-lane group.
template <int L> RB_HD float lane_bcast(float v, int src) {
#if RB_DEVICE_BUILD
    if (L > 1) return __shfl_sync(0xffffffffu, v, src, L);
#endif
    (void)src;
    return v;
}
template <int L> RB_HD vec3 lane_bcast3(vec3 v, int src) {
    return mk3(lane_bcast<L>(v.x, src), lane_bcast<L>(v.y, src), lane_bcast<L>(v.z, src));
}
template <int L> RB_HD bool lane_any(bool p) {
#if RB_DEVICE_BUILD
    if (L > 1) {
        int v = p ? 1 : 0;
#pragma unroll
        for (int o = L / 2; o > 0; o >>= 1) v |= __shfl_xor_sync(0xffffffffu, v, o, L);
        return v != 0;
    }
#endif
    return p;
}

// Sweep the constraints in slots [a, e) of the item (part of one colour stage) with L lanes per constraint.
// `cs` is the shared-memory window the constant rows are read from (the resident copy or a staging
// buffer of the streaming pipeline), `mu` the resident window of the mutable impulses; both are
// indexed by item slot.  `wslot` is the staged world pseudo body (wslot + 1 = garbage slot).
// `q0` is the global schedule slot of the item's slot 0 (rare per-constraint rows stay in HBM).
// MODE is a compile-time constant so each sweep kind is straight-line code.
template <int L, int MODE, class B>
RB_HD void coop_stage(const World& w, const B& bd, const RowView& cs, const RowView& mu, int wslot, int q0, int a, int e,
                      int tid, int nth, bool solve_friction) {
    constexpr int PPL = MAX_PTS / L;   // points per lane
    const Params& P = w.prm;
    const int groups = nth / L, grp = tid / L, sub = tid % L;
    for (int base = a; base < e; base += groups) {
        const int s_raw = base + grp;
        const bool active = s_raw < e && grp < groups;
        const int s = active ? s_raw : a;   // inactive lanes shadow a valid slot (they must execute the shuffles)
        const float4 dirf = cs.pc(CR4_DIRF, s), t1w = cs.pc(CR4_T1W, s), trn = cs.pc(CR4_TR, s), wi4 = mu.mr(MR_WI, s);
        const int id1 = as_int(cs.pp(PR4_ITD1I, sub, s).w), id2 = as_int(cs.pp(PR4_ITD2A, sub, s).w), nc = as_int(trn.w);   // (replicated per point)
        // branch-free gathers: a world-attached side reads the staged identity/zero pseudo body.
        // Only what a sweep needs is loaded: velocities, inverse masses and (for the rhs) the poses.
        const int gi1 = id1 < 0 ? wslot : id1, gi2 = id2 < 0 ? wslot : id2;
        BodyState g1, g2;
        g1.lin = bd.lin(gi1); g1.ang = bd.ang(gi1); g1.im = bd.im(gi1);
        g2.lin = bd.lin(gi2); g2.ang = bd.ang(gi2); g2.im = bd.im(gi2);
        if (MODE == MODE_RELAX || (MODE == MODE_BIASED && solve_friction)) { g1.p = bd.xf(gi1); g2.p = bd.xf(gi2); }   // (friction in the bias pass reads the poses)
        vec3 v1 = g1.lin, w1 = g1.ang, v2 = g2.lin, w2 = g2.ang;
        const vec3 dir = xyz(dirf), t1 = xyz(t1w);
        const vec3 t2 = cross3(dir, t1);
        const bool is_static = id1 == NO_BODY || id2 == NO_BODY;
        const float stf = is_static ? 1.0f : 0.0f;
        const float cfm_soft = P.dyn_cfm + stf * (P.static_cfm - P.dyn_cfm);
        const float erp = P.dyn_erp + stf * (P.static_erp - P.dyn_erp);
        const vec3 lin1 = had(dir, g1.im), lin2 = had(dir, g2.im);

        // ---- parallel part: every lane prepares its own point(s) ----
        PointPre pre[PPL];
        float imp[PPL], acc[PPL], r[PPL], seed[PPL], dist_new[PPL];
        bool own_seed = false;
#pragma unroll
        for (int j = 0; j < PPL; ++j) {
            const int k = sub + j * L;
            const float4 a1 = cs.pp(PR4_TD1R, k, s), a2 = cs.pp(PR4_TD2D, k, s), b1 = cs.pp(PR4_ITD1I, k, s), b2 = cs.pp(PR4_ITD2A, k, s);
            pre[j].td1 = xyz(a1); pre[j].td2 = xyz(a2); pre[j].itd1 = xyz(b1); pre[j].itd2 = xyz(b2);
            r[j] = a1.w; imp[j] = mu.mf(MR_IMP, k, s); acc[j] = mu.mf(MR_ACC, k, s); seed[j] = 0.0f;
            pre[j].rhs = 0.0f; pre[j].cfm = 1.0f; dist_new[j] = 0.0f;
            if (k < nc) {
                // point_rhs.  Poses only change in the position integration, so the separation the relax sweep
                // evaluates is kept for the biased sweep of the next substep (the first one uses generate's).
                if (MODE == MODE_RELAX) {
                    vec3 p1 = xform(g1.p, xyz(cs.pp(PR4_LP1, k, s)));
                    vec3 p2 = xform(g2.p, xyz(cs.pp(PR4_LP2, k, s)));
                    const float dist = a2.w + dot3(p1 - p2, dir);
                    dist_new[j] = dist;
                    pre[j].rhs = max2(dist, 0.0f) * P.sub_inv_dt;
                }
                if (MODE == MODE_BIASED) {
                    float dist = mu.mf(MR_DIST, k, s);
                    if (P.num_relax == 0) {   // no relax sweep refreshes the cache: evaluate here
                        const pose x1 = bd.xf(gi1), x2 = bd.xf(gi2);
                        dist = a2.w + dot3(xform(x1, xyz(cs.pp(PR4_LP1, k, s))) - xform(x2, xyz(cs.pp(PR4_LP2, k, s))), dir);
                    }
                    float rhs = max2(dist, 0.0f) * P.sub_inv_dt;
                    rhs = rhs + clampf(dist * erp, -P.max_corrective_velocity, 0.0f);
                    pre[j].cfm = dist <= 0.0f ? cfm_soft : 1.0f;
                    pre[j].rhs = rhs;
                }
                if (MODE == MODE_RESTITUTION) {
                    seed[j] = crow(w, CR_LP1 + k, q0 + s).w;
                    own_seed = own_seed || seed[j] < 0.0f;
                }
                if (MODE == MODE_WARMSTART) {
                    acc[j] = acc[j] + imp[j];
                    imp[j] = imp[j] * P.warmstart_coeff;
                }
            }
        }
        bool skip = false;
        if (MODE == MODE_RESTITUTION) skip = !lane_any<L>(own_seed);

        // ---- sequential part: the points in order; every lane evaluates its own row against the current
        //      velocities (SIMT: same instructions), the owner's result is broadcast and applied by all ----
#pragma unroll
        for (int kk = 0; kk < MAX_PTS; ++kk) {
            const int owner = kk % L, j = kk / L;
            float nl = imp[j], dl_own;
            if (MODE == MODE_WARMSTART) dl_own = imp[j];
            else if (MODE == MODE_RESTITUTION) dl_own = point_restitution(pre[j], r[j], imp[j], acc[j], seed[j], dir, v1, w1, v2, w2, nl);
            else dl_own = point_solve(pre[j], r[j], imp[j], dir, v1, w1, v2, w2, nl);
            const bool mine = sub == owner && kk < nc;
            imp[j] = mine ? nl : imp[j];
            const float dl = lane_bcast<L>(dl_own, owner);
            const vec3 i1 = lane_bcast3<L>(pre[j].itd1, owner), i2 = lane_bcast3<L>(pre[j].itd2, owner);
            if (kk < nc) apply_normal(lin1, lin2, i1, i2, dl, v1, w1, v2, w2);
        }

        float4 ti4 = mu.mr(MR_TI, s);
        float ti0 = ti4.x, ti1 = ti4.y, wi = wi4.x;
        float ta0 = ti4.z, ta1 = ti4.w, wa = wi4.y;
        if (MODE == MODE_WARMSTART || (MODE != MODE_RESTITUTION && solve_friction)) {
            const FrictionJac fj = coop_get_jac(cs, s);
            if (MODE == MODE_WARMSTART) {
                ta0 = ta0 + ti0; ta1 = ta1 + ti1;
                ti0 = ti0 * P.warmstart_coeff; ti1 = ti1 * P.warmstart_coeff;
                wa = wa + wi;
                wi = wi * P.warmstart_coeff;
                friction_warmstart_jac(g1, g2, t1, t2, nc, fj, ti0, ti1, wi, v1, w1, v2, w2);
            } else {
                const float4 twd = cs.pc(CR4_TWD, s);
                float tlimit = 0.0f, wlimit = 0.0f;
#pragma unroll
                for (int kk = 0; kk < MAX_PTS; ++kk) {
                    const float ik = lane_bcast<L>(imp[kk / L], kk % L);
                    if (kk < nc) {
                        tlimit = tlimit + ik;
                        wlimit = fma_(ik, kk == 0 ? twd.x : (kk == 1 ? twd.y : (kk == 2 ? twd.z : twd.w)), wlimit);
                    }
                }
                tlimit = tlimit * dirf.w;
                wlimit = wlimit * dirf.w;
                constexpr bool relax = MODE == MODE_RELAX;
                vec3 lfc1 = zero3(), lfc2 = zero3();
                if (!relax) { lfc1 = xyz(crow(w, CR_LFC1, q0 + s)); lfc2 = xyz(crow(w, CR_LFC2, q0 + s)); }
                FrictionState f;
                f.ti0 = ti0; f.ti1 = ti1; f.wi = wi;
                friction_solve_jac(P, g1, g2, dir, t1, t2, nc, tlimit, wlimit, t1w.w, fj, trn.x, trn.y, trn.z, relax, lfc1, lfc2, f, v1,
                                   w1, v2, w2);
                ti0 = f.ti0; ti1 = f.ti1; wi = f.wi;
            }
        }
        // ---- write back: each lane its own point impulses, lane 0 the shared state ----
        if (active && !skip) {
#pragma unroll
            for (int j = 0; j < PPL; ++j) {
                const int k = sub + j * L;
                if (k < nc) {
                    mu.mf(MR_IMP, k, s) = imp[j];
                    if (MODE == MODE_WARMSTART) mu.mf(MR_ACC, k, s) = acc[j];
                    if (MODE == MODE_RELAX) mu.mf(MR_DIST, k, s) = dist_new[j];
                }
            }
            if (sub == 0) {
                if (MODE != MODE_RESTITUTION) {
                    mu.mr(MR_TI, s) = make_float4(ti0, ti1, ta0, ta1);
                    mu.mr(MR_WI, s) = make_float4(wi, wa, 0.0f, 0.0f);
                }
                bd.set_vel(id1 < 0 ? (wslot + 1) : id1, v1, w1);
                bd.set_vel(id2 < 0 ? (wslot + 1) : id2, v2, w2);
            }
        }
    }
}

// coop_stage for a sweep mode known only at run time.
template <int L, class B>
RB_HD void coop_stage_mode(int mode, const World& w, const B& bd, const RowView& cs, const RowView& mu, int wslot, int q0, int a, int e,
                           int tid, int nth, bool solve_friction) {
    if (mode == MODE_WARMSTART) coop_stage<L, MODE_WARMSTART>(w, bd, cs, mu, wslot, q0, a, e, tid, nth, solve_friction);
    else if (mode == MODE_BIASED) coop_stage<L, MODE_BIASED>(w, bd, cs, mu, wslot, q0, a, e, tid, nth, solve_friction);
    else if (mode == MODE_RELAX) coop_stage<L, MODE_RELAX>(w, bd, cs, mu, wslot, q0, a, e, tid, nth, solve_friction);
    else coop_stage<L, MODE_RESTITUTION>(w, bd, cs, mu, wslot, q0, a, e, tid, nth, solve_friction);
}

// Bank the impulses of constraint s into their accumulators and scale them by `scale`: the warm-start
// coefficient, or 0 when the step has no warm start (the impulses are then banked without being applied).
RB_HD void coop_bank(const RowView& mu, int s, float scale) {
    float4 im = mu.mr(MR_IMP, s), ac = mu.mr(MR_ACC, s), ti = mu.mr(MR_TI, s), wi = mu.mr(MR_WI, s);
    ac.x = ac.x + im.x; ac.y = ac.y + im.y; ac.z = ac.z + im.z; ac.w = ac.w + im.w;
    im.x = im.x * scale; im.y = im.y * scale; im.z = im.z * scale; im.w = im.w * scale;
    ti.z = ti.z + ti.x; ti.w = ti.w + ti.y; ti.x = ti.x * scale; ti.y = ti.y * scale;
    wi.y = wi.y + wi.x; wi.x = wi.x * scale;
    mu.mr(MR_IMP, s) = im; mu.mr(MR_ACC, s) = ac; mu.mr(MR_TI, s) = ti; mu.mr(MR_WI, s) = wi;
}

// ---- the streaming / grid-wide solve ------------------------------------------------------------------
// Constraint-row policies of solve_item: where a constraint's rows live between sweeps and which sweep reads them.
//
// HbmRows<FM, JM>: the Cons tables in HBM/L2, loaded, swept (cons_sweep) and stored back by one thread per
// constraint.  The only rows with Coulomb friction (FM = 1) and generic joints (JM = 1).  generate / bank / writeback
// work in the caller's Cons scratch `c` (see solve_item).
template <int FM, int JM>
struct HbmRows {
    static constexpr bool solve_groups = true;   // a world with substep solve-groups takes these rows
    static constexpr bool generic_joints = JM != 0;
    RB_HD explicit HbmRows(const World&) {}
    template <class B>
    static RB_HD void begin(const World&, const B&) {}
    template <class B>
    static RB_HD void generate(const World& w, const B& bd, int q, int buf, int item, Cons& c) {
        cons_generate<FM>(w, bd, q, buf, item, c);
        cons_store_static<FM>(w, q, c);
        cons_store_dyn<FM>(w, q, c);
    }
    // The constraints of colour stage [a, e) in the launch's solve-group: strided over the threads, or by thread 0 alone (serial).
    template <class B>
    static RB_HD void stage(const World& w, const B& bd, int a, int e, bool serial, int mode, bool fric, int tid, int nth, bool grp,
                            unsigned char gk) {
        if (serial) {
            if (tid == 0)
                for (int q = a; q < e; ++q) { if (grp && w.cons_key[q] != gk) continue; Cons cc; cons_load<FM>(w, q, cc); cons_sweep<FM>(w, bd, q, cc, mode, fric); cons_store_dyn<FM>(w, q, cc); }
        } else {
            for (int q = a + tid; q < e; q += nth) { if (grp && w.cons_key[q] != gk) continue; Cons cc; cons_load<FM>(w, q, cc); cons_sweep<FM>(w, bd, q, cc, mode, fric); cons_store_dyn<FM>(w, q, cc); }
        }
    }
    static RB_HD void bank(const World& w, int q, Cons& c) {   // bank and zero the impulses (no velocity change)
        cons_load<FM>(w, q, c);
#pragma unroll
        for (int k = 0; k < MAX_PTS; ++k)
            if (k < c.nc) { c.acc[k] = c.acc[k] + c.imp[k]; c.imp[k] = c.imp[k] * 0.0f; }
        c.ta0 = c.ta0 + c.ti0; c.ta1 = c.ta1 + c.ti1; c.ti0 = c.ti0 * 0.0f; c.ti1 = c.ti1 * 0.0f;
        c.wa = c.wa + c.wi; c.wi = c.wi * 0.0f;
        if (FM) {
#pragma unroll
            for (int k = 0; k < MAX_PTS; ++k)
                if (k < c.nc) {
                    c.pta0[k] = c.pta0[k] + c.pti0[k]; c.pta1[k] = c.pta1[k] + c.pti1[k];
                    c.pti0[k] = c.pti0[k] * 0.0f; c.pti1[k] = c.pti1[k] * 0.0f;
                }
        }
        cons_store_dyn<FM>(w, q, c);
    }
    static RB_HD void writeback(const World& w, int q, int buf, Cons& c) { cons_load<FM>(w, q, c); cons_writeback<FM>(w, q, buf, c); }
    template <class B>
    static RB_HD void update_joint(const World& w, const B& bd, int q, int sub) { if (JM) joint_update_generic(w, bd, q, sub); else joint_update(w, bd, q); }
    template <class B>   // warm: the generic joints' warm start, fused into the first biased pass (worker.rs:548)
    static RB_HD void solve_joint(const World& w, const B& bd, int q, bool relax, bool warm) {
        if (JM) joint_solve_generic(w, bd, q, relax, warm); else joint_solve(w, bd, q, relax);
    }
    static RB_HD void writeback_joint(const World& w, int q) { if (JM) joint_writeback_generic(w, q); else joint_writeback(w, q); }
};

// PoolRows<L>: the lane-cooperative rows of coop_stage (L lanes per constraint) in the L2-resident World::large_pool /
// large_mut (row stride cons_cap, indexed by schedule slot).  For the grid-wide item 0 of the twist path: the solver
// bodies are the global s_* tables (ids are body indices), the world pseudo body is entry nb, the garbage slot nb + 1.
// No Coulomb friction, no generic joints and no substep solve-groups: a world with any of them takes HbmRows.
template <int L>
struct PoolRows {
    static constexpr bool solve_groups = false;   // (the key filter costs k_collide and k_solve_large stack and spills)
    static constexpr bool generic_joints = false;
    RowView rows, mu;
    int wslot;
    RB_HD explicit PoolRows(const World& w) {
        wslot = w.nb;
        rows.p = w.large_pool; rows.stride = w.cons_cap;
        mu.p = w.large_mut; mu.stride = w.cons_cap;
    }
    template <class B>
    RB_HD void begin(const World& w, const B& bd) const {
        bd.set_vel(wslot, zero3(), zero3());
        bd.set_xf(wslot, pident());
        w.b_eim[wslot] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    template <class B>
    RB_HD void generate(const World& w, const B& bd, int q, int buf, int item, Cons& c) const {
        cons_generate(w, bd, q, buf, item, c);
        coop_put(rows, mu, bd, q, c);
    }
    template <class B>
    RB_HD void stage(const World& w, const B& bd, int a, int e, bool serial, int mode, bool fric, int tid, int nth, bool, unsigned char) const {
        // the overflow colour is solved one constraint after the other by the first L lanes
        const int n = serial ? L : nth;
        if (serial && tid >= L) return;
        // stages with more constraints than lane groups are throughput-bound: one lane per constraint
        // executes fewer instructions in total than L lanes sharing it
        if (L > 1 && !serial && (e - a) * L > nth) coop_stage_mode<1>(mode, w, bd, rows, mu, wslot, 0, a, e, tid, n, fric);
        else coop_stage_mode<L>(mode, w, bd, rows, mu, wslot, 0, a, e, tid, n, fric);
    }
    RB_HD void bank(const World&, int q, Cons&) const { coop_bank(mu, q, 0.0f); }
    RB_HD void writeback(const World& w, int q, int buf, Cons& c) const {
        coop_get_for_writeback(rows, mu, q, c);
        cons_writeback(w, q, buf, c, true);
    }
    template <class B>
    static RB_HD void update_joint(const World& w, const B& bd, int q, int) { joint_update(w, bd, q); }
    template <class B>
    static RB_HD void solve_joint(const World& w, const B& bd, int q, bool relax, bool) { joint_solve(w, bd, q, relax); }
    static RB_HD void writeback_joint(const World& w, int q) { joint_writeback(w, q); }
};

// Solve one work item from solver-body init to the final positions of its bodies, with the constraint rows of policy R:
// one CTA per item with its bodies in shared memory (BlockExec, SmemBodies), or the grid-wide item 0 with the bodies in
// the global tables and grid barriers (GridExec / GridSpreadExec, GlobalBodies).
template <class R, class X, class B>
RB_PHASE void solve_item(const X& ex, const World& w, const B& bd, int item, vec3 gravity) {
    const Params& P = w.prm;
    State* st = w.st;
    const int buf = st->cur;
    const bool global_ids = item == 0;
    const int b0 = w.item_body_start[item], b1 = w.item_body_start[item + 1];
    const int c0 = w.item_cons_start[item];
    const int c1 = w.item_cons_start[item + 1] < w.cons_cap ? w.item_cons_start[item + 1] : w.cons_cap;
    const int j0 = w.item_joint_start[item], j1 = w.item_joint_start[item + 1];
    const int* coff = w.item_color_off + (size_t)item * (NUM_COLORS + 1);
    const int* joff = w.item_jcolor_off + (size_t)item * (NUM_COLORS + 1);
    const int ncol = st->nused_colors, njcol = st->njused_colors;
    const int ovf = w.color_pos[COLOR_OVERFLOW], jovf = w.jcolor_pos[COLOR_OVERFLOW];
    const int tid = ex.tid(), nth = ex.nth();
    // substep solve-groups: this launch solves the islands whose key is pass_key, at the cadence w.prm was derived for
    const bool grp = R::solve_groups && w.any_extra != 0;
    const unsigned char gk = (unsigned char)w.pass_key;
    const R rows(w);

    // The kernels of the general path sit at 255 registers with stack frames of 1-4 KB, and this function's shape decides
    // them: the Cons scratch of generate / bank / writeback is declared by the loops here (not inside the policy), and the
    // three colour-stage loops stay written out (not one lambda).  Either alternative costs those kernels 8-32 B of stack.
    auto stage = [&](int a, int e, bool serial, int mode, bool fric) { rows.stage(w, bd, a, e, serial, mode, fric, tid, nth, grp, gk); };

    if (tid == 0) {
        w.item_flags[item] = 0;   // bit 0: some contact of this item holds a restitution seed
        rows.begin(w, bd);
    }
    for (int l = b0 + tid; l < b1; l += nth) {
        int b = w.item_bodies[l];
        if (grp && w.b_key[b] != gk) continue;
        body_init(w, bd, b, global_ids ? b : l - b0, gravity);
    }
    ex.sync();
    // S2 generate
    for (int q = c0 + tid; q < c1; q += nth) {
        if (grp && w.cons_key[q] != gk) continue;
        Cons c;
        rows.generate(w, bd, q, buf, item, c);
    }
    ex.sync();

    for (int sub = 0; sub < P.num_substeps; ++sub) {
        for (int l = b0 + tid; l < b1; l += nth) {
            int b = w.item_bodies[l];
            if (grp && w.b_key[b] != gk) continue;
            body_increment(w, bd, b, global_ids ? b : l - b0);
        }
        ex.sync();
        // S4 joint rows from the current poses
        if (j1 > j0) {
            for (int q = j0 + tid; q < j1; q += nth) { if (grp && w.j_key[q] != gk) continue; rows.update_joint(w, bd, q, sub); }
            ex.sync();
        }
        // S5 update + warmstart, colour by colour
        if (P.warmstart_coeff != 0.0f) {
            for (int c = 0; c < ncol; ++c) {
                int a = c0 + coff[c], e = c0 + coff[c + 1];
                if (e > c1) e = c1;
                if (a >= e) continue;
                stage(a, e, c == ovf, MODE_WARMSTART, false);
                ex.sync();
            }
        } else {
            // warmstart_coefficient == 0: update only banks and zeroes the impulses (no velocity change)
            for (int q = c0 + tid; q < c1; q += nth) {
                if (grp && w.cons_key[q] != gk) continue;
                Cons c;
                rows.bank(w, q, c);
            }
            ex.sync();
        }
        for (int pass = 0; pass < 2; ++pass) {
            const bool relax = pass == 1;
            const int iters = relax ? P.num_relax : P.num_pgs;
            const bool fric = relax || P.friction_in_bias || P.num_relax == 0;
            for (int it = 0; it < iters; ++it) {
                const bool jwarm = R::generic_joints && P.warmstart_joints && !relax && it == 0;   // fused into the first biased pass (worker.rs:548)
                // joints first (solve.rs:89-92), then contacts
                for (int c = 0; c < njcol; ++c) {
                    int a = j0 + joff[c], e = j0 + joff[c + 1];
                    if (a >= e) continue;
                    if (c == jovf) {
                        if (tid == 0) for (int q = a; q < e; ++q) { if (grp && w.j_key[q] != gk) continue; rows.solve_joint(w, bd, q, relax, jwarm); }
                    } else {
                        for (int q = a + tid; q < e; q += nth) { if (grp && w.j_key[q] != gk) continue; rows.solve_joint(w, bd, q, relax, jwarm); }
                    }
                    ex.sync();
                }
                for (int c = 0; c < ncol; ++c) {
                    int a = c0 + coff[c], e = c0 + coff[c + 1];
                    if (e > c1) e = c1;
                    if (a >= e) continue;
                    stage(a, e, c == ovf, relax ? MODE_RELAX : MODE_BIASED, fric);
                    ex.sync();
                }
            }
            if (!relax) {
                for (int l = b0 + tid; l < b1; l += nth) {
                    int b = w.item_bodies[l];
                    if (grp && w.b_key[b] != gk) continue;
                    body_integrate(w, bd, b, global_ids ? b : l - b0);
                }
                ex.sync();
            }
        }
    }
    // S9 restitution
    if (w.item_flags[item]) {
        for (int c = 0; c < ncol; ++c) {
            int a = c0 + coff[c], e = c0 + coff[c + 1];
            if (e > c1) e = c1;
            if (a >= e) continue;
            stage(a, e, c == ovf, MODE_RESTITUTION, false);
            ex.sync();
        }
    }
    // S10 impulse writeback
    for (int q = c0 + tid; q < c1; q += nth) { if (grp && w.cons_key[q] != gk) continue; Cons c; rows.writeback(w, q, buf, c); }
    for (int q = j0 + tid; q < j1; q += nth) { if (grp && w.j_key[q] != gk) continue; rows.writeback_joint(w, q); }
    for (int l = b0 + tid; l < b1; l += nth) {
        int b = w.item_bodies[l];
        if (grp && w.b_key[b] != gk) continue;
        body_writeback(w, bd, b, global_ids ? b : l - b0);
    }
}

RB_HD bool item_is_coop(const World& w, int item) {
    const int nbod = w.item_body_start[item + 1] - w.item_body_start[item];
    const int ncons = w.item_cons_start[item + 1] - w.item_cons_start[item];
    const int njoints = w.item_joint_start[item + 1] - w.item_joint_start[item];
    const int ovf = w.color_pos[COLOR_OVERFLOW];
    const int* coff = w.item_color_off + (size_t)item * (NUM_COLORS + 1);
    const bool has_ovf = ovf >= 0 && coff[ovf + 1] > coff[ovf];
    return item > 0 && njoints == 0 && !has_ovf && !w.prm.friction_model && ncons < 65536 && w.item_cons_start[item + 1] <= w.cons_cap &&
           coop_plan(w.coop_small_floats, nbod, ncons).ok;
}

// Streaming pipeline of one CTA: two shared-memory staging buffers filled by bulk (TMA) copies from the
// L2-resident pool, one chunk ahead of the sweep.  A chunk is a run of at most `cap` slots of one colour
// stage; its 36 constant rows are stored as ONE contiguous block in the pool (row stride = cnt | 1), so
// staging a chunk is a single bulk copy.  Only rows that are constant during the step are streamed (the
// impulses stay resident), so chunks can be prefetched at any time.  `t` counts the chunks consumed since
// the kernel started (buffer = t & 1, mbarrier phase = (t >> 1) & 1) and lives across items.
struct CoopPipe {
    float4* buf[2];
    unsigned long long* mbar;   // [2], shared memory
    float4* pool;               // the item's region of the pool: chunk q starts at COOP_ROWS * (chunk[q] + q)
    const int* chunk;           // [nchunks + 1] first slot of every chunk (shared memory)
    int nchunks;
    unsigned t;
    int sweep_threads;          // threads that take part in the sweeps (a multiple of the warp size, <= block size)
};
RB_HD RowView coop_chunk_rows(const CoopPipe& pp, int q) {   // pool rows of chunk q, indexed by item slot
    const int o = pp.chunk[q], cnt = pp.chunk[q + 1] - o;
    RowView v;
    v.p = pp.pool + (size_t)COOP_ROWS * (o + q) - o;
    v.stride = cnt | 1;
    return v;
}
RB_HD RowView coop_slot_rows(const CoopPipe& pp, int s) {   // ... of the chunk that holds slot s
    int lo = 0, hi = pp.nchunks - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (pp.chunk[mid] <= s) lo = mid; else hi = mid - 1;
    }
    return coop_chunk_rows(pp, lo);
}
RB_HD void coop_pipe_issue(const CoopPipe& pp, int q, int b) {   // one thread: stage chunk q into buffer b
    const int o = pp.chunk[q], cnt = pp.chunk[q + 1] - o;
    const unsigned bytes = (unsigned)(COOP_ROWS * (cnt | 1) * 16);
    mbar_expect_tx(pp.mbar + b, bytes);
    bulk_g2s(b ? pp.buf[1] : pp.buf[0], pp.pool + (size_t)COOP_ROWS * (o + q), bytes, pp.mbar + b);
}

// One sweep over all colour stages of the item.  Resident items read their shared-memory rows; streamed
// items consume the pipeline, whose first chunk is already in flight (issued after generate, or by the sweep
// before).  `wrap`: another sweep follows, its first chunk is prefetched by the last one here.
template <int L, int MODE>
RB_PHASE void coop_sweep(const BlockCtx& ctx, const World& w, const SmemBodies& bd, const RowView& res, const RowView& mu, bool resident,
                         CoopPipe& pp, const int* s_stage, int nstages, int wslot, int c0, bool fric, bool wrap) {
    const int tid = ctx.btid, nth = pp.sweep_threads;   // warps beyond the sweep width only take part in the barriers
#ifdef RB_DEBUG
    if (w.debug_flags & 1) return;   // profiling experiment (debug build only): skip the sweeps
#endif
    if (resident) {
        for (int c = 0; c < nstages; ++c) {
            const int ae = s_stage[c];
            if (tid < nth) coop_stage<L, MODE>(w, bd, res, mu, wslot, c0, ae & 0xffff, ae >> 16, tid, nth, fric);
            ctx.block_sync();
        }
        return;
    }
    for (int q = 0; q < pp.nchunks; ++q) {
        const int o = pp.chunk[q], e = pp.chunk[q + 1];
        const int b = pp.t & 1;
        mbar_wait(pp.mbar + b, (pp.t >> 1) & 1);
        if (tid == 0) {   // prefetch the next chunk into the buffer the previous chunk was read from
            if (q + 1 < pp.nchunks) coop_pipe_issue(pp, q + 1, b ^ 1);
            else if (wrap) coop_pipe_issue(pp, 0, b ^ 1);
        }
        RowView rd;
        rd.p = (b ? pp.buf[1] : pp.buf[0]) - o;   // (a select, not a dynamically indexed array: keeps the pointers in registers and the loads LDS)
        rd.stride = (e - o) | 1;
        if (tid < nth) coop_stage<L, MODE>(w, bd, rd, mu, wslot, c0, o, e, tid, nth, fric);
        ctx.block_sync();
        pp.t += 1;
    }
}

// ---- warm start of a shared-memory item, body-centric ------------------------------------------------
// The reference applies the banked impulses constraint by constraint, colour by colour (update + warmstart,
// contact_with_twist_friction.rs:426-522, :633-678).  A warm start only ADDS to the two bodies of its
// constraint, so what a body ends up with is the sequence of additions of ITS constraints in colour order.
// Walking each body's adjacency list (slot order = colour order, built by the schedule) reproduces exactly
// that sequence -- same operands, same order, same bits -- with one barrier instead of one per colour.
// Streamed items gather the same way, reading the constant rows from the L2 pool instead of shared memory.
RB_HD void coop_warmstart_bank(const Params& P, const RowView& mu, int s) {   // the per-constraint half: bank and scale
    coop_bank(mu, s, P.warmstart_coeff);
}
// The rows one side of constraint s adds to its body in the warm start, loaded apart from their use so that a
// body's gather can fetch the next constraint's rows (L2 latency for a streamed item) while it applies the
// current one.  The rows of points beyond nc are loaded too (generate writes every point row) and never used.
struct WarmSide { float4 dirf, t1w, trn, itd[MAX_PTS], jac[5], imp, ti, wi; };
RB_HD WarmSide coop_warmstart_load(const RowView& cs, const RowView& mu, int s, int side) {
    WarmSide o;
    o.dirf = cs.pc(CR4_DIRF, s); o.t1w = cs.pc(CR4_T1W, s); o.trn = cs.pc(CR4_TR, s);
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) o.itd[k] = cs.pp(side == 0 ? PR4_ITD1I : PR4_ITD2A, k, s);
#pragma unroll
    for (int r = 0; r < 5; ++r) o.jac[r] = cs.pc(CR4_J3 + r, s);   // i10 i11 i20 i21 tw1 tw2 (see coop_put_jac)
    o.imp = mu.mr(MR_IMP, s); o.ti = mu.mr(MR_TI, s); o.wi = mu.mr(MR_WI, s);
    return o;
}
// One side of one constraint applied to its body (v, wv): the operations coop_stage<MODE_WARMSTART> performs on that side.
RB_HD void coop_warmstart_apply(const WarmSide& o, int side, vec3 im, vec3& v, vec3& wv) {
    const int nc = as_int(o.trn.w);
    const vec3 dir = xyz(o.dirf), t1 = xyz(o.t1w);
    const vec3 t2 = cross3(dir, t1);
    const vec3 lin = had(dir, im);
    const float imp[MAX_PTS] = {o.imp.x, o.imp.y, o.imp.z, o.imp.w};
#pragma unroll
    for (int k = 0; k < MAX_PTS; ++k) {
        if (k < nc) {
            const vec3 itd = xyz(o.itd[k]);
            v = madd3(v, lin, side == 0 ? imp[k] : -imp[k]);
            wv = madd3(wv, itd, imp[k]);
        }
    }
    const float4 d = o.jac[0], e = o.jac[1], f = o.jac[2], g = o.jac[3], h = o.jac[4];
    const float ti0 = o.ti.x, ti1 = o.ti.y, wi = o.wi.x;
    if (side == 0) {
        v = madd3v(v, madd3(t1 * ti0, t2, ti1), im);
        wv = madd3(madd3(wv, mk3(d.x, d.y, d.z), ti0), mk3(d.w, e.x, e.y), ti1);
        if (nc > 1) wv = madd3(wv, mk3(g.x, g.y, g.z), wi);
    } else {
        v = madd3v(v, madd3(t1 * (-ti0), t2, -ti1), im);
        wv = madd3(madd3(wv, mk3(e.z, e.w, f.x), ti0), mk3(f.y, f.z, f.w), ti1);
        if (nc > 1) wv = madd3(wv, mk3(g.w, h.x, h.y), -wi);
    }
}

// One work item, start to finish, by one CTA: bodies and impulses in shared memory; the constant
// constraint rows resident in shared memory when they fit, else streamed from the L2 pool through the
// staging pipeline (L lanes / constraint).
template <int L>
RB_PHASE void solve_item_coop(const BlockCtx& ctx, const World& w, float* smem, int smem_floats, CoopPipe& pp, int item, vec3 gravity) {
    const Params& P = w.prm;
    State* st = w.st;
    const int buf = st->cur;
    const int b0 = w.item_body_start[item], b1 = w.item_body_start[item + 1];
    const int c0 = w.item_cons_start[item], n = w.item_cons_start[item + 1] - c0;
    const int tid = ctx.btid, nth = ctx.bsize;
    const CoopPlan plan = coop_plan(smem_floats, b1 - b0, n);
    const bool resident = plan.resident != 0;
    const int wslot = b1 - b0;
    SmemBodies bd;
    bd.s = smem;
    RowView mu;     // impulses
    mu.p = reinterpret_cast<float4*>(smem + plan.body_slots * SB_STRIDE); mu.stride = plan.mstride;
    float4* cbase = mu.p + MR_COUNT * plan.mstride;
    RowView res;    // the resident constant rows
    res.p = cbase; res.stride = plan.stride;
    // The non-empty colour stages of this item, staged once (no HBM/L2 reads between sweeps), and for
    // streamed items the chunks they are cut into.
    RB_SHARED int s_stage[NUM_COLORS + 2];
    RB_SHARED int s_nstages;
    RB_SHARED int s_chunk[COOP_MAX_CHUNKS + 1];
    RB_SHARED int s_nchunks;
    RB_SHARED int s_width;
    pp.buf[0] = cbase; pp.buf[1] = cbase + (size_t)COOP_ROWS * plan.stride;
    pp.pool = w.coop_pool + (size_t)2 * COOP_ROWS * c0; pp.chunk = s_chunk;
    if (tid == 0) {
        const int* coff = w.item_color_off + (size_t)item * (NUM_COLORS + 1);
        const int ncol = st->nused_colors;
        int ns = 0;
        for (int c = 0; c < ncol; ++c)
            if (coff[c + 1] > coff[c]) s_stage[ns++] = coff[c] | (coff[c + 1] << 16);
        s_nstages = ns;
        // sweep width: enough lanes for the longest colour stage in one pass, at least 4 warps; the other warps
        // of the CTA only help with generation, integration and writeback (fewer warps = shorter issue queues)
        int longest = 0;
        for (int c = 0; c < ns; ++c) longest = max2i(longest, (s_stage[c] >> 16) - (s_stage[c] & 0xffff));
        const int width = (longest * L + 31) & ~31;
        s_width = min2i(nth, max2i(width, 128));
        int nq = 0;
        if (!resident)
            for (int c = 0; c < ns; ++c)
                for (int o = s_stage[c] & 0xffff; o < (s_stage[c] >> 16); o += plan.stride) s_chunk[nq++] = o;
        s_chunk[nq] = n;
        s_nchunks = nq;
        w.item_flags[item] = 0;
        bd.set_vel(wslot, zero3(), zero3());
        bd.set_xf(wslot, pident());
        bd.set_mass(wslot, sym_zero(), zero3());
        if (!coop_plan(w.coop_small_floats, b1 - b0, n).resident) st->need_big = 1;
        atomic_add(resident ? &st->coop_resident : &st->coop_streamed, 1);
    }
#ifdef RB_DEBUG   // phase timeline of one item (debug build only: librapier_b200_dbg.so, tests/prof_phases.py)
    const bool trace = (w.debug_flags & 2) && ctx.bid == 0 && tid == 0;
    int tr = 0;
#define RB_TRACE() if (trace && tr < 32) w.dbg_times[tr++] = rb_clock()
#else
#define RB_TRACE() do {} while (0)
#endif
    RB_TRACE();
    for (int l = b0 + tid; l < b1; l += nth) body_init(w, bd, w.item_bodies[l], l - b0, gravity);
    ctx.block_sync();
    RB_TRACE();
    const int nstages = s_nstages;
    pp.nchunks = s_nchunks;
    pp.sweep_threads = s_width;
    for (int s = tid; s < n; s += nth) {   // S2 generate, one thread per constraint
        Cons c;
        cons_generate(w, bd, c0 + s, buf, item, c);
        coop_put(resident ? res : coop_slot_rows(pp, s), mu, bd, s, c);
    }
    if (!resident) fence_async_proxy();   // pool rows written above are read by bulk copies from here on
    ctx.block_sync();
    RB_TRACE();
    const bool bouncy_item = w.item_flags[item] != 0;
    const bool warm = P.warmstart_coeff != 0.0f;
    // The pipeline sweeps of a streamed item.  The first chunk of the first one is staged from here on: nothing
    // before that sweep reads the staging buffers (the warm start reads the rows from the pool).
    int total_sweeps = P.num_substeps * (P.num_pgs + P.num_relax) + (bouncy_item ? 1 : 0);
#ifdef RB_DEBUG
    if (w.debug_flags & 1) total_sweeps = 0;   // (the sweeps are skipped: no chunk may be left in flight)
#endif
    if (!resident && total_sweeps > 0 && tid == 0) coop_pipe_issue(pp, 0, pp.t & 1);
    int done = 0;
    for (int sub = 0; sub < P.num_substeps; ++sub) {
        for (int l = b0 + tid; l < b1; l += nth) body_increment(w, bd, w.item_bodies[l], l - b0);
        if (warm) {   // body-centric (one barrier instead of one per colour)
            if (sub == 0) RB_TRACE();
            for (int s = tid; s < n; s += nth) coop_warmstart_bank(P, mu, s);
            ctx.block_sync();   // (also orders the increments above before the gathers below)
#ifdef RB_DEBUG
            if (!(w.debug_flags & 1))
#endif
                for (int l = tid; l < b1 - b0; l += nth) {
                    const int* adj = w.adj_list + w.adj_off[b0 + l];
                    const int cnt = w.adj_cnt[b0 + l];
                    vec3 v = bd.lin(l), wv = bd.ang(l);
                    const vec3 im = bd.im(l);
                    if (cnt > 0) {
                        // software pipeline: the rows of entry i + 1 and list entry i + 2 are in flight while entry i is applied
                        int e = adj[0], e_after = cnt > 1 ? adj[1] : 0;
                        WarmSide next = coop_warmstart_load(resident ? res : coop_slot_rows(pp, e >> 1), mu, e >> 1, e & 1);
                        for (int i = 0; i < cnt; ++i) {
                            const WarmSide cur = next;
                            const int side = e & 1;
                            if (i + 1 < cnt) {
                                e = e_after;
                                if (i + 2 < cnt) e_after = adj[i + 2];
                                next = coop_warmstart_load(resident ? res : coop_slot_rows(pp, e >> 1), mu, e >> 1, e & 1);
                            }
                            coop_warmstart_apply(cur, side, im, v, wv);
                        }
                    }
                    bd.set_vel(l, v, wv);
                }
            ctx.block_sync();
            if (sub == 0) RB_TRACE();
        } else {   // bank the impulses without applying them
            for (int s = tid; s < n; s += nth) coop_bank(mu, s, 0.0f);
            ctx.block_sync();
        }
        for (int pass = 0; pass < 2; ++pass) {
            const bool relax = pass == 1;
            const int iters = relax ? P.num_relax : P.num_pgs;
            const bool fric = relax || P.friction_in_bias || P.num_relax == 0;
            for (int it = 0; it < iters; ++it) {
                ++done;
                if (relax) coop_sweep<L, MODE_RELAX>(ctx, w, bd, res, mu, resident, pp, s_stage, nstages, wslot, c0, fric, done < total_sweeps);
                else coop_sweep<L, MODE_BIASED>(ctx, w, bd, res, mu, resident, pp, s_stage, nstages, wslot, c0, fric, done < total_sweeps);
                if (sub == 0) RB_TRACE();
            }
            if (!relax) {
                for (int l = b0 + tid; l < b1; l += nth) body_integrate(w, bd, w.item_bodies[l], l - b0);
                ctx.block_sync();
                if (sub == 0) RB_TRACE();
            }
        }
    }
    if (bouncy_item) coop_sweep<L, MODE_RESTITUTION>(ctx, w, bd, res, mu, resident, pp, s_stage, nstages, wslot, c0, false, false);
    RB_TRACE();
    for (int s = tid; s < n; s += nth) {
        Cons c;
        coop_get_for_writeback(resident ? res : coop_slot_rows(pp, s), mu, s, c);
        cons_writeback(w, c0 + s, buf, c, true);
    }
#ifdef RB_DEBUG
    if (w.debug_flags & 2) ctx.block_sync();   // (uniform: only to attribute the two writebacks separately)
#endif
    RB_TRACE();
    for (int l = b0 + tid; l < b1; l += nth) body_writeback(w, bd, w.item_bodies[l], l - b0);
    RB_TRACE();
#undef RB_TRACE
}

}  // namespace rb
