// TEST INFRASTRUCTURE ONLY -- CPU oracle: scene state, collision detection bookkeeping, colouring
// (see oracle.h header note; PARITY UNPINNED).
//
// Follows, in order: src/pipeline/physics_pipeline/substep.rs:267-581 (step_inner),
// src/pipeline/physics_pipeline/solve.rs:45-157 (detect_collisions),
// src/geometry/broad_phase_bvh/{mod.rs:170-263, update.rs:334-396,484-537} (pair-set semantics),
// src/geometry/narrow_phase/pair_update.rs:67-680 (process_pair),
// src/geometry/narrow_phase/{contacts.rs:300-385, mod.rs:87-172} (transitions + colouring).
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <vector>
#include <cstdio>
#include <cstring>
#include <string>
#include "oracle_internal.h"

namespace orc {

void solve_island(World& w, V3 gravity);  // oracle_solver.cpp
void ccd_motion_clamping(World& w);       // oracle_ccd.cpp

// ---------------------------------------------------------------------------------------------
// Mass properties: parry MassProperties::{from_cuboid, from_ball, new, world_com, world_inv_inertia}
// as consumed by RigidBodyMassProps::recompute_mass_properties_from_colliders
// (src/dynamics/rigid_body_components.rs:421) and update_world_mass_properties (:528-572).
// ---------------------------------------------------------------------------------------------
static inline float inv_exact0(float x) { return x == 0.0f ? 0.0f : 1.0f / x; }

static void collider_mass(const Collider& c, float& mass, V3& principal) {
    if (c.shape == RB_SHAPE_CUBOID) {
        float vol = c.he.x * c.he.y * c.he.z * 8.0f;
        V3 sq = cmul(c.he, c.he);
        float third = 1.0f / 3.0f;
        V3 unit = V3{(sq.y + sq.z) * third, (sq.x + sq.z) * third, (sq.x + sq.y) * third};
        mass = vol * c.density;
        principal = unit * mass;
    } else if (c.shape == RB_SHAPE_CAPSULE) {   // parry MassProperties::from_capsule (restated: cylinder + two half balls)
        const float hh = c.he.x, r = c.he.y;
        const int ax = (int)c.he.z;
        const float pi_ = 3.14159265358979323846f;
        const float cyl_vol = hh * r * r * pi_ * 2.0f, ball_vol = pi_ * r * r * r * 4.0f / 3.0f;
        const float sq_r = r * r, sq_h = hh * hh * 4.0f;
        const float cyl_off = (sq_r * 3.0f + sq_h) / 12.0f, cyl_axis = sq_r / 2.0f, ball_unit = sq_r * 2.0f / 5.0f;
        const float h = hh * 2.0f;
        const float extra = (h * h * 0.25f + h * r * 3.0f / 8.0f) * ball_vol * c.density;
        const float i_off = (cyl_off * cyl_vol + ball_unit * ball_vol) * c.density + extra;
        const float i_axis = (cyl_axis * cyl_vol + ball_unit * ball_vol) * c.density;
        mass = (cyl_vol + ball_vol) * c.density;
        principal = V3{i_off, i_off, i_off};
        vset(principal, ax, i_axis);
    } else {
        float r = c.he.x;
        float vol = 3.14159265358979323846f * r * r * r * 4.0f / 3.0f;
        float unit = r * r * 2.0f / 5.0f;
        mass = vol * c.density;
        principal = V3{unit * mass, unit * mass, unit * mass};
    }
}

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

// `first_body` / `first_collider`: only the bodies from first_body on, from the colliders from first_collider on
// (insertion appends bodies that carry appended colliders only).
static int recompute_mass_properties(World& w, int first_body = 0, int first_collider = 0) {
    int nb = (int)w.bodies.size();
    std::vector<int> count(nb, 0), first(nb, -1);
    for (int ci = first_collider; ci < (int)w.colliders.size(); ++ci) {
        int p = w.colliders[ci].parent;
        if (w.colliders[ci].sensor && w.colliders[ci].density == 0.0f) continue;   // a massless sensor adds nothing
        if (p >= 0) {
            if (count[p] == 0) first[p] = ci;
            count[p]++;
        }
    }
    for (int bi = first_body; bi < nb; ++bi) {
        Body& b = w.bodies[bi];
        b.local_com = vzero();
        b.inv_mass = 0.0f;
        b.inv_principal_inertia = vzero();
        b.principal_inertia = vzero();
        b.principal_frame = qidentity();
        if (count[bi] == 1 && w.colliders[first[bi]].shape == RB_SHAPE_CONVEX) {
            // MassProperties::from_convex_polyhedron [parry]: unit-density properties of the hull times the density; its centre
            // of mass and principal frame go through the collider's pose (in double, rounded once)
            const Collider& c = w.colliders[first[bi]];
            const Hull& h = w.hulls[(int)c.he.x];
            const float mass = h.volume * c.density;
            const V3 pi = h.principal_inertia * c.density;
            const double q[4] = {c.pos_wrt_parent.q.x, c.pos_wrt_parent.q.y, c.pos_wrt_parent.q.z, c.pos_wrt_parent.q.w};
            const double v[3] = {h.com.x, h.com.y, h.com.z};
            double t[3] = {q[1] * v[2] - q[2] * v[1], q[2] * v[0] - q[0] * v[2], q[0] * v[1] - q[1] * v[0]};
            for (int k = 0; k < 3; ++k) t[k] *= 2.0;
            const double u[3] = {q[1] * t[2] - q[2] * t[1], q[2] * t[0] - q[0] * t[2], q[0] * t[1] - q[1] * t[0]};
            b.local_com = V3{(float)((double)c.pos_wrt_parent.t.x + (v[0] + q[3] * t[0] + u[0])),
                             (float)((double)c.pos_wrt_parent.t.y + (v[1] + q[3] * t[1] + u[1])),
                             (float)((double)c.pos_wrt_parent.t.z + (v[2] + q[3] * t[2] + u[2]))};
            const double g[4] = {h.principal_frame.x, h.principal_frame.y, h.principal_frame.z, h.principal_frame.w};
            b.principal_frame = Q4{(float)(q[3] * g[0] + q[0] * g[3] + q[1] * g[2] - q[2] * g[1]),
                                   (float)(q[3] * g[1] - q[0] * g[2] + q[1] * g[3] + q[2] * g[0]),
                                   (float)(q[3] * g[2] + q[0] * g[1] - q[1] * g[0] + q[2] * g[3]),
                                   (float)(q[3] * g[3] - q[0] * g[0] - q[1] * g[1] - q[2] * g[2])};
            b.inv_mass = inv_exact0(mass);
            b.inv_principal_inertia = V3{inv_exact0(pi.x), inv_exact0(pi.y), inv_exact0(pi.z)};
        } else if (count[bi] == 1) {
            const Collider& c = w.colliders[first[bi]];
            float mass;
            V3 pi;
            collider_mass(c, mass, pi);
            b.local_com = c.pos_wrt_parent.t;
            b.inv_mass = inv_exact0(mass);
            b.inv_principal_inertia = V3{inv_exact0(pi.x), inv_exact0(pi.y), inv_exact0(pi.z)};
            b.principal_frame = c.pos_wrt_parent.q;
        } else if (count[bi] > 1) {
            // Sum of axis-aligned parts only (composite bodies whose summed tensor is diagonal).
            float M = 0.0f;
            V3 com = vzero();
            for (size_t ci = (size_t)first_collider; ci < w.colliders.size(); ++ci) {
                const Collider& c = w.colliders[ci];
                if (c.parent != bi || (c.sensor && c.density == 0.0f)) continue;
                if (c.shape == RB_SHAPE_CONVEX) return RB_ERR_INVALID;   // polyhedra in multi-collider bodies: not supported
                float mass; V3 pi;
                collider_mass(c, mass, pi);
                M = M + mass;
                com = com + c.pos_wrt_parent.t * mass;
            }
            if (M != 0.0f) {   // (a massless compound still reaches the additional mass and the extents below)
            com = com * (1.0f / M);
            bool simple = true;   // axis-aligned parts offset from the centre of mass along one axis: the summed tensor is diagonal
            for (size_t ci = (size_t)first_collider; ci < w.colliders.size(); ++ci) {
                const Collider& c = w.colliders[ci];
                if (c.parent != bi || (c.sensor && c.density == 0.0f)) continue;
                Q4 q = c.pos_wrt_parent.q;
                if (!(q.x == 0.0f && q.y == 0.0f && q.z == 0.0f)) simple = false;
                V3 d = c.pos_wrt_parent.t - com;
                if ((d.x != 0.0f) + (d.y != 0.0f) + (d.z != 0.0f) > 1) simple = false;
            }
            if (simple) {
                V3 I = vzero();
                for (size_t ci = (size_t)first_collider; ci < w.colliders.size(); ++ci) {
                    const Collider& c = w.colliders[ci];
                    if (c.parent != bi || (c.sensor && c.density == 0.0f)) continue;
                    float mass; V3 pi;
                    collider_mass(c, mass, pi);
                    V3 d = c.pos_wrt_parent.t - com;
                    float d2 = dot(d, d);
                    I = I + pi + V3{(d2 - d.x * d.x) * mass, (d2 - d.y * d.y) * mass, (d2 - d.z * d.z) * mass};
                }
                b.local_com = com;
                b.inv_principal_inertia = V3{inv_exact0(I.x), inv_exact0(I.y), inv_exact0(I.z)};
            } else {   // compound bodies in general: full tensor, principal axes by eigen-decomposition
                std::vector<float> pm;
                std::vector<std::array<float, 3>> ppi, pt;
                std::vector<std::array<float, 4>> pq;
                for (size_t ci = (size_t)first_collider; ci < w.colliders.size(); ++ci) {
                    const Collider& c = w.colliders[ci];
                    if (c.parent != bi || (c.sensor && c.density == 0.0f)) continue;
                    float mass; V3 pi;
                    collider_mass(c, mass, pi);
                    pm.push_back(mass);
                    ppi.push_back({pi.x, pi.y, pi.z});
                    pt.push_back({c.pos_wrt_parent.t.x, c.pos_wrt_parent.t.y, c.pos_wrt_parent.t.z});
                    pq.push_back({c.pos_wrt_parent.q.x, c.pos_wrt_parent.q.y, c.pos_wrt_parent.q.z, c.pos_wrt_parent.q.w});
                }
                float lc[3], I[3], fr[4];
                composite_inertia((int)pm.size(), pm.data(), reinterpret_cast<const float(*)[3]>(ppi.data()), reinterpret_cast<const float(*)[4]>(pq.data()),
                                  reinterpret_cast<const float(*)[3]>(pt.data()), lc, I, fr);
                b.local_com = V3{lc[0], lc[1], lc[2]};
                b.principal_frame = Q4{fr[0], fr[1], fr[2], fr[3]};
                b.inv_principal_inertia = V3{inv_exact0(I[0]), inv_exact0(I[1]), inv_exact0(I[2])};
            }
            b.inv_mass = inv_exact0(M);
            }
        }
        // RigidBodyAdditionalMassProps::Mass (rigid_body_components.rs:454-486); MassProperties::set_mass(m, true)
        // [parry] rescales the angular inertia by new_mass / old_mass, i.e. its inverse by inv(new) * old.
        if (b.additional_mass > 0.0f) {
            const float add = b.additional_mass;
            const float prev = inv_exact0(b.inv_mass);
            if (prev > 0.0f) {
                const float inv_new = inv_exact0(prev + add);
                b.inv_principal_inertia = b.inv_principal_inertia * (inv_new * prev);
                b.inv_mass = inv_new;
            } else if (count[bi] == 1 && w.colliders[first[bi]].shape == RB_SHAPE_CONVEX) {
                return RB_ERR_INVALID;          // additional mass on a massless polyhedron: not supported
            } else if (count[bi] == 1) {
                // massless collider: inertia and centre of mass of the shape at unit density, rescaled to the mass
                Collider u = w.colliders[first[bi]];
                u.density = 1.0f;
                float um; V3 upi;
                collider_mass(u, um, upi);
                const float inv_new = inv_exact0(add);
                b.local_com = u.pos_wrt_parent.t;
                b.principal_frame = u.pos_wrt_parent.q;
                b.inv_principal_inertia = V3{inv_exact0(upi.x), inv_exact0(upi.y), inv_exact0(upi.z)} * (inv_new * um);
                b.inv_mass = inv_new;
            } else if (count[bi] == 0) {
                b.inv_mass = inv_exact0(add);   // no shape to derive an inertia from: just the mass
            } else {
                return RB_ERR_INVALID;          // massless multi-collider bodies with additional mass: not supported
            }
        }
        b.principal_inertia = V3{inv_exact0(b.inv_principal_inertia.x), inv_exact0(b.inv_principal_inertia.y),
                                 inv_exact0(b.inv_principal_inertia.z)};
        // recompute_max_extent (rigid_body_components.rs:491-515): bounding spheres about the local centre of mass
        b.max_extent = 0.0f;
        b.ccd_thickness = 3.4028235e38f;   // RigidBodyCcd::default (:1076); min over the colliders' Shape::ccd_thickness (:1224-1228)
        for (size_t ci = (size_t)first_collider; ci < w.colliders.size(); ++ci) {
            const Collider& c = w.colliders[ci];
            if (c.parent != bi) continue;
            if (c.shape != RB_SHAPE_CAPSULE && c.shape != RB_SHAPE_CONVEX)   // (capsules and polyhedra are never swept here: they do not count)
                b.ccd_thickness = fmin2(b.ccd_thickness, c.shape == RB_SHAPE_BALL ? c.he.x : fmin2(c.he.x, fmin2(c.he.y, c.he.z)));
            const float radius = c.shape == RB_SHAPE_CONVEX ? w.hulls[(int)c.he.x].radius + c.he.y
                               : c.shape == RB_SHAPE_BALL ? c.he.x : (c.shape == RB_SHAPE_CAPSULE ? c.he.x + c.he.y : length(c.he));
            b.max_extent = fmax2(b.max_extent, length(c.pos_wrt_parent.t - b.local_com) + radius);
        }
    }
    return RB_OK;
}

// rigid_body_components.rs:528-572
void update_world_mass_properties(Body& b) {
    b.world_com = pose_point(b.pos, b.local_com);
    bool dyn = b.is_strict_dynamic();
    b.eff_inv_mass = V3{b.inv_mass, b.inv_mass, b.inv_mass};
    V3 d = b.inv_principal_inertia;
    if (d.x != 0.0f || d.y != 0.0f || d.z != 0.0f) {
        M3 r = qto_mat(qmul(b.pos.q, b.principal_frame));
        float c0[3] = {r.c0.x, r.c0.y, r.c0.z}, c1[3] = {r.c1.x, r.c1.y, r.c1.z}, c2[3] = {r.c2.x, r.c2.y, r.c2.z};
        auto e = [&](int i, int j) {
            return (c0[i] * d.x) * c0[j] + (c1[i] * d.y) * c1[j] + (c2[i] * d.z) * c2[j];
        };
        b.eff_world_inv_inertia = Sdp3{e(0, 0), e(0, 1), e(0, 2), e(1, 1), e(1, 2), e(2, 2)};
    } else {
        b.eff_world_inv_inertia = sdp_zero();
    }
    if (!dyn || (b.flags & RB_BODY_LOCK_TX)) b.eff_inv_mass.x = 0.0f;
    if (!dyn || (b.flags & RB_BODY_LOCK_TY)) b.eff_inv_mass.y = 0.0f;
    if (!dyn || (b.flags & RB_BODY_LOCK_TZ)) b.eff_inv_mass.z = 0.0f;
    Sdp3& m = b.eff_world_inv_inertia;
    if (!dyn || (b.flags & RB_BODY_LOCK_RX)) { m.m11 = 0; m.m12 = 0; m.m13 = 0; }
    if (!dyn || (b.flags & RB_BODY_LOCK_RY)) { m.m22 = 0; m.m12 = 0; m.m23 = 0; }
    if (!dyn || (b.flags & RB_BODY_LOCK_RZ)) { m.m33 = 0; m.m13 = 0; m.m23 = 0; }
}

// ---------------------------------------------------------------------------------------------
// Collider world pose + broad-phase AABB (collider.rs:553-599) and the fat leaf AABB with change
// detection (broad_phase_bvh/mod.rs:170-201, :235-263; skin = 0.04 * length_unit).
// ---------------------------------------------------------------------------------------------
static inline Aabb loosened(const Aabb& a, float l) {
    return Aabb{V3{a.mins.x - l, a.mins.y - l, a.mins.z - l}, V3{a.maxs.x + l, a.maxs.y + l, a.maxs.z + l}};
}
static inline bool aabb_contains(const Aabb& a, const Aabb& b) {
    return a.mins.x <= b.mins.x && a.mins.y <= b.mins.y && a.mins.z <= b.mins.z && a.maxs.x >= b.maxs.x &&
           a.maxs.y >= b.maxs.y && a.maxs.z >= b.maxs.z;
}
static inline bool aabb_intersects(const Aabb& a, const Aabb& b) {
    return a.mins.x <= b.maxs.x && a.mins.y <= b.maxs.y && a.mins.z <= b.maxs.z && a.maxs.x >= b.mins.x &&
           a.maxs.y >= b.mins.y && a.maxs.z >= b.mins.z;
}

// substep.rs:103-146 (collider pose + AABB harvest) followed by refresh_moved_collider_aabbs
// (substep.rs:229-240) -> BroadPhaseBvh::set_aabb.
void refresh_collider(World& w, Collider& c) {
    if (c.parent >= 0)
        c.pos = pose_mul(w.bodies[c.parent].pos, c.pos_wrt_parent);
    else
        c.pos = c.pos_wrt_parent;
    float pred = w.params.prediction_distance();
    c.aabb = loosened(c.shape == RB_SHAPE_CONVEX ? convex_aabb(w.hulls, c.he, c.pos) : shape_aabb(c.shape, c.he, c.pos), c.contact_skin + pred / 2.0f);
    if (!c.fat_valid || !aabb_contains(c.fat, c.aabb)) {
        c.fat = loosened(c.aabb, 4.0e-2f * w.params.p.length_unit);
        c.fat_valid = true;
        w.bp_dirty = true;
    }
}

// ---------------------------------------------------------------------------------------------
// Broad phase: the pair set is exactly the set of collider pairs whose fat AABBs intersect,
// minus same-parent / fixed-fixed / collision-group filtered pairs (update.rs:334-396); pairs
// leave the set only when a changed leaf stops intersecting (update.rs:484-537).  Because fat
// AABBs only change together with `changed`, the set is a pure function of the fat AABBs.
// Realised here as a sort-and-sweep along x (the GPU build uses a device radix sort + sweep).
// ---------------------------------------------------------------------------------------------
static bool pair_allowed(const World& w, int c1, int c2) {
    const Collider& a = w.colliders[c1];
    const Collider& b = w.colliders[c2];
    if (a.parent >= 0 && a.parent == b.parent) return false;
    bool dyn1 = a.parent >= 0 && w.bodies[a.parent].is_strict_dynamic();
    bool dyn2 = b.parent >= 0 && w.bodies[b.parent].is_strict_dynamic();
    if (!dyn1 && !dyn2) return false;  // ActiveCollisionTypes::default(): DYNAMIC_DYNAMIC | DYNAMIC_KINEMATIC | DYNAMIC_FIXED
    if (!((a.memberships & b.filter) != 0 && (b.memberships & a.filter) != 0)) return false;
    if (!w.nocontact_body_pairs.empty() && a.parent >= 0 && b.parent >= 0) {
        uint32_t lo = (uint32_t)std::min(a.parent, b.parent), hi = (uint32_t)std::max(a.parent, b.parent);
        uint64_t key = ((uint64_t)lo << 32) | hi;
        if (std::binary_search(w.nocontact_body_pairs.begin(), w.nocontact_body_pairs.end(), key)) return false;
    }
    return true;
}

static void clear_pair_color(World& w, Pair& p) {  // narrow_phase/mod.rs:154-172
    if (p.color < COLOR_OVERFLOW) {
        for (int k = 0; k < 2; ++k)
            if (p.color_bodies[k] != NO_BODY) w.color_masks[p.color_bodies[k]].clear(p.color);
    }
    p.color = COLOR_UNCOLORED;
    p.color_bodies[0] = p.color_bodies[1] = NO_BODY;
}

// A pair that leaves the broad phase while touching stops (pair_management.rs: emit_stop_event) and frees its colour.
static void removed_pair(World& w, Pair& o) {
    if ((o.nsc > 0 || o.intersecting) && ((w.colliders[o.c1].active_events | w.colliders[o.c2].active_events) & RB_EVENT_COLLISION))
        w.collision_events.push_back(RbCollisionEvent{o.c1, o.c2, 0, (int)w.counters.steps + 1});
    clear_pair_color(w, o);
    if (o.nsc > 0) w.islands_dirty = true;   // a touching pair that leaves the broad phase may split its island (persistent.rs; the kernels relabel whenever the pair table changes)
}
static void update_pairs(World& w) {
    int nc = (int)w.colliders.size();
    // Only pairs with a collider that can move matter (static-static pairs are filtered anyway), so the sweep runs
    // over the movers, and each mover searches the static colliders, which are sorted once (they never move).
    auto is_static = [&](const Collider& c) { return c.parent < 0 || !w.bodies[c.parent].is_dynamic(); };
    if (w.static_dirty) {
        w.static_sorted.clear();
        w.static_max_width = 0.0f;
        for (int i = 0; i < nc; ++i) {
            const Collider& c = w.colliders[i];
            if (c.shape < 0 || !is_static(c)) continue;
            w.static_sorted.push_back(i);
            w.static_max_width = fmax2(w.static_max_width, c.fat.maxs.x - c.fat.mins.x);
        }
        std::stable_sort(w.static_sorted.begin(), w.static_sorted.end(), [&](int a, int b) {
            return w.colliders[a].fat.mins.x < w.colliders[b].fat.mins.x;
        });
        w.static_dirty = false;
    }
    std::vector<int> idx;
    for (int i = 0; i < nc; ++i)
        if (w.colliders[i].shape >= 0 && !is_static(w.colliders[i])) idx.push_back(i);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) {
        return w.colliders[a].fat.mins.x < w.colliders[b].fat.mins.x;
    });
    std::vector<uint64_t> keys;
    auto emit = [&](int i, int j) {
        int c1 = std::min(i, j), c2 = std::max(i, j);
        if (!pair_allowed(w, c1, c2)) return;
        keys.push_back(((uint64_t)(uint32_t)c1 << 32) | (uint32_t)c2);
    };
    const int nd = (int)idx.size(), ns = (int)w.static_sorted.size();
    const float wn = w.static_max_width * 1.0001f + 1.0e-6f;
    for (int ii = 0; ii < nd; ++ii) {
        const Collider& a = w.colliders[idx[ii]];
        for (int jj = ii + 1; jj < nd; ++jj) {
            const Collider& b = w.colliders[idx[jj]];
            if (b.fat.mins.x > a.fat.maxs.x) break;
            if (aabb_intersects(a.fat, b.fat)) emit(idx[ii], idx[jj]);
        }
        const float x0 = a.fat.mins.x - wn;
        int lo = 0, hi = ns;
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (w.colliders[w.static_sorted[mid]].fat.mins.x < x0) lo = mid + 1; else hi = mid;
        }
        for (int jj = lo; jj < ns; ++jj) {
            const Collider& b = w.colliders[w.static_sorted[jj]];
            if (b.fat.mins.x > a.fat.maxs.x) break;
            if (aabb_intersects(a.fat, b.fat)) emit(idx[ii], w.static_sorted[jj]);
        }
    }
    std::sort(keys.begin(), keys.end());
    // Merge with the previous (sorted) pair list, carrying persistent per-pair state.
    std::vector<Pair> np;
    np.reserve(keys.size());
    size_t oi = 0;
    for (uint64_t k : keys) {
        while (oi < w.pairs.size()) {
            Pair& o = w.pairs[oi];
            uint64_t ok = ((uint64_t)(uint32_t)o.c1 << 32) | (uint32_t)o.c2;
            if (ok < k) {  // removed pair: end-touch frees its colour (contacts.rs:333-335)
                removed_pair(w, o);
                ++oi;
            } else break;
        }
        if (oi < w.pairs.size()) {
            Pair& o = w.pairs[oi];
            uint64_t ok = ((uint64_t)(uint32_t)o.c1 << 32) | (uint32_t)o.c2;
            if (ok == k) { np.push_back(o); ++oi; continue; }
        }
        Pair p;
        memset(&p, 0, sizeof(p));
        p.c1 = (int)(k >> 32);
        p.c2 = (int)(k & 0xffffffffu);
        p.b1 = w.colliders[p.c1].parent;
        p.b2 = w.colliders[p.c2].parent;
        p.color = COLOR_UNCOLORED;
        p.color_bodies[0] = p.color_bodies[1] = NO_BODY;
        np.push_back(p);
    }
    for (; oi < w.pairs.size(); ++oi) removed_pair(w, w.pairs[oi]);
    w.pairs.swap(np);
    w.bp_dirty = false;
    w.counters.broad_phase_ran = 1;
}

// ---------------------------------------------------------------------------------------------
// Narrow phase: process_pair (pair_update.rs:67-680).
// ---------------------------------------------------------------------------------------------
static float combine_coeff(float c1, float c2, int r1, int r2) {  // coefficient_combine_rule.rs:51-84
    int rule = std::max(r1, r2);
    switch (rule) {
        case RB_COMBINE_AVERAGE: return (c1 + c2) / 2.0f;
        case RB_COMBINE_MIN: return fabsf(fmin2(c1, c2));
        case RB_COMBINE_MULTIPLY: return c1 * c2;
        case RB_COMBINE_MAX: return fmax2(c1, c2);
        case RB_COMBINE_CLAMPED_SUM: return fclamp(c1 + c2, 0.0f, 1.0f);
        default: return sqrtf(fmax2(c1, 0.0f) * fmax2(c2, 0.0f));
    }
}

static float relative_pose_drift(const Pose& base, const Pose& cur, float max_extent) {  // contact_pair.rs:299-323
    float trans = length(cur.t - base.t);
    Q4 d = qmul(cur.q, qconj(base.q));
    float rot_chord = 2.0f * length(V3{d.x, d.y, d.z}) * max_extent;
    return trans + rot_chord;
}
static float relative_rot_cos(Q4 base, Q4 cur) {  // contact_pair.rs:284-293
    float c = qdot(base, cur);
    return 2.0f * c * c - 1.0f;
}

static float shape_origin_radius(const World& w, int shape, V3 he) {  // pair_update.rs:591-595 (local AABB corners)
    if (shape == RB_SHAPE_CONVEX) { const V3 a = w.hulls[(int)he.x].aabb; return length(V3{a.x + he.y, a.y + he.y, a.z + he.y}); }
    if (shape == RB_SHAPE_BALL) {
        V3 c = V3{he.x, he.x, he.x};
        return length(c);
    }
    if (shape == RB_SHAPE_CAPSULE) return length(V3{he.y, he.x + he.y, he.y});
    return length(he);
}

// manifold_reduction.rs:4-84
static void reduce_manifold_naive(const RawManifold& m, int selected[4], int& num_selected, float prediction) {
    if (m.n <= 4) return;
    for (int i = 0; i < 4; ++i) selected[i] = -1;
    float deepest = 3.4028235e38f;
    for (int i = 0; i < m.n; ++i)
        if (m.pts[i].dist < deepest) { deepest = m.pts[i].dist; selected[0] = i; }
    if (selected[0] < 0) { num_selected = 0; return; }
    V3 a = m.pts[selected[0]].local_p1;
    float furthest = -3.4028235e38f;
    for (int i = 0; i < m.n; ++i) {
        float d = length_sq(m.pts[i].local_p1 - a);
        if (i != selected[0] && m.pts[i].dist <= prediction && d > furthest) { furthest = d; selected[1] = i; }
    }
    if (selected[1] < 0) { num_selected = 1; return; }
    V3 b = m.pts[selected[1]].local_p1;
    if (veq(a, b)) { num_selected = 1; return; }
    V3 ab = b - a;
    V3 tangent = cross(ab, m.local_n1);
    float min_dot = 3.4028235e38f, max_dot = -3.4028235e38f;
    for (int i = 0; i < m.n; ++i) {
        if (i == selected[0] || i == selected[1] || m.pts[i].dist > prediction) continue;
        float d = dot(m.pts[i].local_p1 - a, tangent);
        if (d < min_dot) { min_dot = d; selected[2] = i; }
        if (d > max_dot) { max_dot = d; selected[3] = i; }
    }
    if (selected[2] < 0) num_selected = 2;
    else if (selected[2] == selected[3]) num_selected = 3;
    else num_selected = 4;
}

// Returns true when the pair's "has any active contact" state flipped.
static bool process_pair(World& w, Pair& pair) {
    const Collider& co1 = w.colliders[pair.c1];
    const Collider& co2 = w.colliders[pair.c2];
    const float prediction = w.params.prediction_distance();
    const float dt = w.params.p.dt;
    const float recycle_dist = w.params.p.contact_recycling ? w.params.contact_recycle_distance() : 0.0f;

    // Contact recycling (pair_update.rs:111-171).
    if (recycle_dist > 0.0f && pair.has_recycle) {
        Pose pos12 = pose_inv_mul(co1.pos, co2.pos);
        float drift = relative_pose_drift(pair.r_pos12, pos12, pair.r_max_extent);
        float rot_cos = fmin2(relative_rot_cos(pair.r_rot1, co1.pos.q), relative_rot_cos(pair.r_rot2, co2.pos.q));
        if (drift <= pair.r_max_drift && rot_cos > 0.98f) return false;
    }

    bool had_active = pair.nsc > 0;
    const Body* rb1 = pair.b1 >= 0 ? &w.bodies[pair.b1] : nullptr;
    const Body* rb2 = pair.b2 >= 0 ? &w.bodies[pair.b2] : nullptr;
    const int rel_dom = relative_dominance(rb1, rb2);
    bool dyn1 = rb1 && rb1->is_dynamic() && rel_dom <= 0;   // pair_update.rs:538-545: dominance-superior sides keep world anchors
    bool dyn2 = rb2 && rb2->is_dynamic() && rel_dom >= 0;

    Pose pos12 = pose_inv_mul(co1.pos, co2.pos);
    float skin_sum = co1.contact_skin + co2.contact_skin;
    float eff_prediction = prediction + skin_sum;  // pair_update.rs:319

    RawManifold raw;
    if (co1.shape == RB_SHAPE_CONVEX || co2.shape == RB_SHAPE_CONVEX) contact_manifold_convex(w.hulls, co1.shape, co1.he, co2.shape, co2.he, pos12, eff_prediction, raw);
    else contact_manifold(co1.shape, co1.he, co2.shape, co2.he, pos12, eff_prediction, raw);

    // parry ContactManifold::match_contacts: carry ContactData by (fid1, fid2); ball manifolds keep
    // their single point's data (copy_geometry_from).
    Point carried[MAX_RAW_POINTS];
    for (int i = 0; i < raw.n; ++i) {
        Point& p = carried[i];
        memset(&p, 0, sizeof(p));
        p.local_p1 = raw.pts[i].local_p1;
        p.local_p2 = raw.pts[i].local_p2;
        p.dist = raw.pts[i].dist;
        p.fid1 = raw.pts[i].fid1;
        p.fid2 = raw.pts[i].fid2;
        bool single_ball = (co1.shape == RB_SHAPE_BALL || co2.shape == RB_SHAPE_BALL);
        for (int j = 0; j < pair.npts; ++j) {
            const Point& o = pair.pts[j];
            if (single_ball || (o.fid1 == p.fid1 && o.fid2 == p.fid2)) {
                p.impulse = o.impulse;
                p.warmstart_impulse = o.warmstart_impulse;
                p.warmstart_twist = o.warmstart_twist;
                p.warmstart_tangent_world = o.warmstart_tangent_world;
                p.dp1 = o.dp1;
                p.dp2 = o.dp2;
            }
        }
    }

    pair.friction = combine_coeff(co1.friction, co2.friction, co1.friction_rule, co2.friction_rule);
    pair.restitution = combine_coeff(co1.restitution, co2.restitution, co1.restitution_rule, co2.restitution_rule);
    pair.local_n1 = raw.local_n1;
    pair.local_n2 = raw.local_n2;
    pair.normal = qrot(co1.pos.q, raw.local_n1);  // pair_update.rs:414

    // Reduce to <= 4 points and sort them on the contact plane (pair_update.rs:418-457).
    int selected[4] = {0, 1, 2, 3};
    int num_selected = raw.n < MAX_MANIFOLD_POINTS ? raw.n : MAX_MANIFOLD_POINTS;
    reduce_manifold_naive(raw, selected, num_selected, prediction);
    if (num_selected > 1) {
        V3 b0, b1;
        orthonormal_basis(raw.local_n1, b0, b1);
        float k0[4], k1[4];
        int ks[4];
        for (int i = 0; i < num_selected; ++i) {
            V3 p = raw.pts[selected[i]].local_p1;
            k0[i] = dot(p, b0);
            k1[i] = dot(p, b1);
            ks[i] = selected[i];
        }
        for (int i = 1; i < num_selected; ++i) {
            float a0 = k0[i], a1 = k1[i];
            int as = ks[i];
            int j = i;
            while (j > 0 && (k0[j - 1] > a0 || (k0[j - 1] == a0 && k1[j - 1] > a1))) {
                k0[j] = k0[j - 1]; k1[j] = k1[j - 1]; ks[j] = ks[j - 1];
                --j;
            }
            k0[j] = a0; k1[j] = a1; ks[j] = as;
        }
        for (int i = 0; i < num_selected; ++i) selected[i] = ks[i];
    }
    // Only the selected points persist (DESIGN.md: "manifold storage").
    pair.npts = num_selected;
    for (int i = 0; i < num_selected; ++i) pair.pts[i] = carried[selected[i]];

    // Solver contacts (pair_update.rs:459-498) + localisation / anchor freezing (:536-577).
    pair.nsc = 0;
    V3 normal = pair.normal;
    Pose com_pose1 = pose_identity(), com_pose2 = pose_identity();
    if (dyn1) com_pose1 = pose_prepend_translation(rb1->pos, rb1->local_com);
    if (dyn2) com_pose2 = pose_prepend_translation(rb2->pos, rb2->local_com);
    for (int k = 0; k < pair.npts; ++k) {
        Point& c = pair.pts[k];
        float eff_dist = c.dist - co1.contact_skin - co2.contact_skin;
        V3 world_pt1 = pose_point(co1.pos, c.local_p1);
        V3 world_pt2 = pose_point(co2.pos, c.local_p2);
        bool keep = eff_dist < prediction;
        if (!keep) {
            V3 vel1 = rb1 ? rb1->linvel + cross(rb1->angvel, world_pt1 - rb1->world_com) : vzero();
            V3 vel2 = rb2 ? rb2->linvel + cross(rb2->angvel, world_pt2 - rb2->world_com) : vzero();
            keep = eff_dist + dot(vel2 - vel1, normal) * dt < prediction;
        }
        if (!keep) continue;
        SolverContact& sc = pair.sc[pair.nsc++];
        sc.cid = k;
        float shift = dot(world_pt2 - world_pt1, normal) - eff_dist;
        V3 p1 = world_pt1 + normal * shift;
        V3 point = (p1 + world_pt2) * 0.5f;
        c.dp1 = dyn1 ? point - com_pose1.t : point;
        c.dp2 = dyn2 ? point - com_pose2.t : point;
        sc.anchor1 = dyn1 ? pose_inv_point(com_pose1, p1) : p1;
        sc.anchor2 = dyn2 ? pose_inv_point(com_pose2, world_pt2) : world_pt2;
    }

    // Recycle state (pair_update.rs:582-613).
    if (recycle_dist > 0.0f) {
        float max_extent = pair.has_recycle
                               ? pair.r_max_extent
                               : fmax2(shape_origin_radius(w, co1.shape, co1.he), shape_origin_radius(w, co2.shape, co2.he));
        float max_drift = pair.nsc > 0 ? recycle_dist : fmin2(recycle_dist, prediction);
        pair.has_recycle = true;
        pair.r_pos12 = pos12;
        pair.r_rot1 = co1.pos.q;
        pair.r_rot2 = co2.pos.q;
        pair.r_max_extent = max_extent;
        pair.r_max_drift = max_drift;
    }
    return (pair.nsc > 0) != had_active;
}

// narrow_phase/mod.rs:87-152
static void assign_pair_color(World& w, Pair& p) {
    if (p.color != COLOR_UNCOLORED) return;
    bool d1 = p.b1 >= 0 && w.bodies[p.b1].is_dynamic();
    bool d2 = p.b2 >= 0 && w.bodies[p.b2].is_dynamic();
    if (!d1 && !d2) {
        p.color = COLOR_OVERFLOW;
        p.color_bodies[0] = p.color_bodies[1] = NO_BODY;
        return;
    }
    int color;
    uint32_t cb[2];
    if (d1 && d2) {
        Mask128 m;
        m.lo = w.color_masks[p.b1].lo | w.color_masks[p.b2].lo;
        m.hi = w.color_masks[p.b1].hi | w.color_masks[p.b2].hi;
        color = 128;
        for (int c = 0; c < DYNAMIC_COLOR_COUNT; ++c)
            if (!m.test(c)) { color = c; break; }
        cb[0] = (uint32_t)p.b1;
        cb[1] = (uint32_t)p.b2;
    } else {
        int b = d1 ? p.b1 : p.b2;
        const Mask128& m = w.color_masks[b];
        color = 128;
        for (int c = 127; c >= 0; --c)
            if (!m.test(c)) { color = c; break; }
        cb[0] = (uint32_t)b;
        cb[1] = NO_BODY;
    }
    if (color >= 128) {
        p.color = COLOR_OVERFLOW;
        p.color_bodies[0] = p.color_bodies[1] = NO_BODY;
        return;
    }
    for (int k = 0; k < 2; ++k)
        if (cb[k] != NO_BODY) w.color_masks[cb[k]].set(color);
    p.color = (uint8_t)color;
    p.color_bodies[0] = cb[0];
    p.color_bodies[1] = cb[1];
}

// Whole-island wake (island_manager/sleep.rs:8-80): every body of the component, timers reset ("strong").
static void wake_island_of(World& w, int body) {
    if (body < 0 || body >= (int)w.island_of.size()) return;
    const int root = w.island_of[body];
    if (root < 0) { w.bodies[body].sleeping = false; w.bodies[body].sleep_time = 0.0f; return; }
    for (int i = 0; i < (int)w.bodies.size(); ++i)
        if (w.island_of[i] == root && w.bodies[i].sleeping) { w.bodies[i].sleeping = false; w.bodies[i].sleep_time = 0.0f; }
}

static void narrow_phase(World& w) {
    std::vector<int> started;
    std::vector<int> to_wake;
    for (int i = 0; i < (int)w.pairs.size(); ++i) {
        Pair& p = w.pairs[i];
        // pairs without an awake body are not updated (their bodies do not move)
        const bool a1 = p.b1 >= 0 && w.bodies[p.b1].is_awake(), a2 = p.b2 >= 0 && w.bodies[p.b2].is_awake();
        if (!a1 && !a2) continue;
        if (w.colliders[p.c1].sensor || w.colliders[p.c2].sensor) {
            // a pair with a sensor (narrow_phase/intersections.rs:17-221): no contacts, no colour, no island edge -- only whether
            // the shapes intersect (the deepest manifold point is not positive), with a CollisionEvent when that changes
            const Collider& co1 = w.colliders[p.c1];
            const Collider& co2 = w.colliders[p.c2];
            const Pose pos12 = pose_inv_mul(co1.pos, co2.pos);
            const float eff_prediction = w.params.prediction_distance() + (co1.contact_skin + co2.contact_skin);
            RawManifold raw;
            if (co1.shape == RB_SHAPE_CONVEX || co2.shape == RB_SHAPE_CONVEX) contact_manifold_convex(w.hulls, co1.shape, co1.he, co2.shape, co2.he, pos12, eff_prediction, raw);
            else contact_manifold(co1.shape, co1.he, co2.shape, co2.he, pos12, eff_prediction, raw);
            bool inter = false;
            for (int k = 0; k < raw.n; ++k) inter = inter || raw.pts[k].dist <= 0.0f;
            if (inter != p.intersecting && ((co1.active_events | co2.active_events) & RB_EVENT_COLLISION))
                w.collision_events.push_back(RbCollisionEvent{p.c1, p.c2, inter ? 1 : 0, (int)w.counters.steps + 1, RB_COLLISION_EVENT_SENSOR});
            p.intersecting = inter;
            continue;
        }
        if (process_pair(w, p)) {
            // contacts.rs:312-324: start / stop events for colliders that ask for them
            if ((w.colliders[p.c1].active_events | w.colliders[p.c2].active_events) & RB_EVENT_COLLISION)
                w.collision_events.push_back(RbCollisionEvent{p.c1, p.c2, p.nsc > 0 ? 1 : 0, (int)w.counters.steps + 1});
            if (p.nsc == 0) p.force_event_emitted = false;
            if (p.nsc > 0) {
                started.push_back(i);
                // a contact that begins wakes the sleeping side's whole island (narrow_phase/mod.rs:53-67)
                if (p.b1 >= 0 && w.bodies[p.b1].is_dynamic() && w.bodies[p.b1].sleeping) to_wake.push_back(p.b1);
                if (p.b2 >= 0 && w.bodies[p.b2].is_dynamic() && w.bodies[p.b2].sleeping) to_wake.push_back(p.b2);
            } else clear_pair_color(w, p);  // end-touch frees the colour first (contacts.rs:333-335)
            w.counters.schedule_rebuilt = 1;
            w.islands_dirty = true;
        }
    }
    for (int b : to_wake) wake_island_of(w, b);
    // Deferred greedy colouring in canonical (min body, max body, edge) order (contacts.rs:366-385).
    auto bid = [](int b) { return b < 0 ? 0xffffffffu : (uint32_t)b; };
    std::stable_sort(started.begin(), started.end(), [&](int x, int y) {
        const Pair& a = w.pairs[x];
        const Pair& b = w.pairs[y];
        uint32_t a1 = bid(a.b1), a2 = bid(a.b2), b1 = bid(b.b1), b2 = bid(b.b2);
        uint64_t ka = ((uint64_t)std::min(a1, a2) << 32) | std::max(a1, a2);
        uint64_t kb = ((uint64_t)std::min(b1, b2) << 32) | std::max(b1, b2);
        if (ka != kb) return ka < kb;
        return x < y;
    });
    for (int i : started) assign_pair_color(w, w.pairs[i]);
}

// ---------------------------------------------------------------------------------------------
// Islands and sleeping.
// ---------------------------------------------------------------------------------------------
static int dsu_find(std::vector<int>& p, int x) {
    while (p[x] != x) { p[x] = p[p[x]]; x = p[x]; }
    return x;
}
static void label_islands(World& w) {
    const int nb = (int)w.bodies.size();
    std::vector<int> parent(nb);
    for (int i = 0; i < nb; ++i) parent[i] = i;
    auto unite = [&](int a, int b) {
        a = dsu_find(parent, a); b = dsu_find(parent, b);
        if (a != b) parent[std::max(a, b)] = std::min(a, b);   // the smaller index is the root (as on the device)
    };
    for (const Pair& p : w.pairs)
        if (p.nsc > 0 && p.b1 >= 0 && p.b2 >= 0 && w.bodies[p.b1].is_dynamic() && w.bodies[p.b2].is_dynamic()) unite(p.b1, p.b2);
    for (const Joint& j : w.joints)
        if (!j.removed && w.bodies[j.body1].is_dynamic() && w.bodies[j.body2].is_dynamic()) unite(j.body1, j.body2);
    w.island_of.assign(nb, -1);
    for (int i = 0; i < nb; ++i)
        if (w.bodies[i].is_dynamic()) w.island_of[i] = dsu_find(parent, i);
    w.islands_dirty = false;
}

// RigidBodyActivation::update_energy (rigid_body_components.rs:1417-1470) for every awake body, then the
// whole-island decision (island_manager/manager.rs:367-392): an island sleeps when all of its bodies are eligible.
static void update_sleep(World& w) {
    const float dt = w.params.p.dt;
    const float linear_threshold = 0.05f * w.params.p.length_unit;   // default_normalized_linear_threshold
    const float angular_threshold = 0.5f, time_until_sleep = 0.5f;
    const int nb = (int)w.bodies.size();
    std::vector<char> blocked(nb, 0);
    bool any = false;
    for (int i = 0; i < nb; ++i) {
        Body& b = w.bodies[i];
        if (!b.is_awake()) continue;
        const bool may = !(b.flags & RB_BODY_NO_SLEEP);
        const Pose prev = b.sleep_prev_pose;
        b.sleep_prev_pose = b.pos;
        const float sq_angvel = dot(b.angvel, b.angvel);
        bool angular_ok;
        if (b.max_extent > 0.0f) angular_ok = may && sq_angvel < 1.5707963267948966f * 1.5707963267948966f;
        else angular_ok = may && sq_angvel < angular_threshold * angular_threshold;
        const float drift = relative_pose_drift(prev, b.pos, b.max_extent);
        bool can = may && angular_ok && drift * 0.5f < linear_threshold * dt;
        if (!b.is_strict_dynamic()) can = may && dot(b.linvel, b.linvel) == 0.0f && sq_angvel == 0.0f;   // platforms: exactly zero (:1457-1461)
        b.sleep_time = can ? b.sleep_time + dt : 0.0f;
        if (!(b.sleep_time >= time_until_sleep)) blocked[w.island_of[i]] = 1;
        any = true;
    }
    if (!any) return;
    for (int i = 0; i < nb; ++i) {
        Body& b = w.bodies[i];
        if (!b.is_awake() || blocked[w.island_of[i]]) continue;
        b.sleeping = true;                 // RigidBody::sleep (rigid_body.rs:804-807)
        b.sleep_time = time_until_sleep;
        b.linvel = vzero();
        b.angvel = vzero();
        w.counters.schedule_rebuilt = 1;
    }
}

// ---------------------------------------------------------------------------------------------
// One step (substep.rs:267-581).
// ---------------------------------------------------------------------------------------------
static inline double now_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

void step_once(World& w, V3 gravity) {
    w.counters.broad_phase_ran = 0;
    w.counters.schedule_rebuilt = 0;
    double t0 = now_ms();
    // 5. detect_collisions
    if (w.bp_dirty) update_pairs(w);
    double t1 = now_ms();
    narrow_phase(w);
    double t2 = now_ms();
    // 7a. islands (connected components of touching contacts and joints between dynamic bodies; the reference keeps
    //     them incrementally, island_manager/persistent.rs) and the whole-island sleep decision (solve.rs:234-306).
    if (w.islands_dirty) label_islands(w);
    update_sleep(w);
    // 7b. build_islands_and_solve_velocity_constraints
    solve_island(w, gravity);
    // 7c. CCD motion clamping of the fast bodies' next_position (substep.rs:492-520)
    ccd_motion_clamping(w);
    double t3 = now_ms();
    // 7d. advance_to_final_positions (substep.rs:84-224) + 7f refresh_moved_collider_aabbs
    for (Body& b : w.bodies) {
        if (!b.is_awake()) continue;
        b.pos = b.next_pos;
        update_world_mass_properties(b);
    }
    for (Collider& c : w.colliders) {
        if (c.shape >= 0 && c.parent >= 0 && w.bodies[c.parent].is_awake()) refresh_collider(w, c);
    }
    // NarrowPhase::emit_contact_force_events (solver_graph.rs:462-498; ContactForceEvent::from_contact_pair, geometry/mod.rs:223-258)
    {
        const float inv_dt = w.params.p.dt == 0.0f ? 0.0f : 1.0f / w.params.p.dt;
        for (Pair& p : w.pairs) {
            if (p.nsc <= 0) continue;
            const bool a1 = p.b1 >= 0 && w.bodies[p.b1].is_awake(), a2 = p.b2 >= 0 && w.bodies[p.b2].is_awake();
            if (!a1 && !a2) continue;   // solver-active pairs only
            const Collider &c1 = w.colliders[p.c1], &c2 = w.colliders[p.c2];
            const float t1 = (c1.active_events & RB_EVENT_CONTACT_FORCE) ? c1.force_event_threshold : 3.4028235e38f;
            const float t2 = (c2.active_events & RB_EVENT_CONTACT_FORCE) ? c2.force_event_threshold : 3.4028235e38f;
            const float threshold = fmin2(t1, t2);
            if (!(threshold < 3.4028235e38f)) continue;
            float total = 0.0f, maxi = 0.0f;
            for (int k = 0; k < p.nsc; ++k) {
                const float imp = p.pts[p.sc[k].cid].impulse;
                total = total + imp;
                if (imp > maxi) maxi = imp;
            }
            const float magnitude = total * inv_dt;
            if (magnitude > threshold) {
                RbContactForceEvent e{};
                e.collider1 = p.c1; e.collider2 = p.c2;
                const V3 tf = (p.normal * total) * inv_dt;
                e.total_force[0] = tf.x; e.total_force[1] = tf.y; e.total_force[2] = tf.z;
                e.total_force_magnitude = magnitude;
                if (maxi > 0.0f) { e.max_force_direction[0] = p.normal.x; e.max_force_direction[1] = p.normal.y; e.max_force_direction[2] = p.normal.z; }
                e.max_force_magnitude = maxi * inv_dt;
                e.started = p.force_event_emitted ? 0 : 1;
                e.step = (int)w.counters.steps + 1;
                w.force_events.push_back(e);
                p.force_event_emitted = true;
            } else p.force_event_emitted = false;
        }
    }
    double t4 = now_ms();
    w.counters.broad_phase_ms = (float)(t1 - t0);
    w.counters.narrow_phase_ms = (float)(t2 - t1);
    w.counters.collision_detection_ms = (float)(t2 - t0);
    w.counters.solver_ms = (float)(t3 - t2);
    w.counters.update_ms = (float)(t4 - t3);
    w.counters.step_ms = (float)(t4 - t0);
    w.counters.steps++;
    w.counters.num_pairs = (int)w.pairs.size();
}

// ---------------------------------------------------------------------------------------------
// Scene upload (RigidBodySet / ColliderSet / ImpulseJointSet user changes, substep.rs:303-334).
// ---------------------------------------------------------------------------------------------
static inline V3 f3(const float* p) { return V3{p[0], p[1], p[2]}; }
static inline Q4 f4(const float* p) { return Q4{p[0], p[1], p[2], p[3]}; }

// One joint of the ImpulseJointSet from its descriptor (generic_joint.rs:142-300; AngularLimitParams::new,
// joint_constraint_helper.rs:44-73); impulses start at zero.
static int fill_joint(World& w, Joint& j, const RbJointDesc& d) {
    const int nb = (int)w.bodies.size();
    if (d.body1 < 0 || d.body1 >= nb || d.body2 < 0 || d.body2 >= nb) return RB_ERR_INVALID;
    j.removed = false;
    j.body1 = d.body1;
    j.body2 = d.body2;
    j.local_frame1 = Pose{f4(d.local_frame1_q), f3(d.local_frame1_t)};
    j.local_frame2 = Pose{f4(d.local_frame2_q), f3(d.local_frame2_t)};
    j.locked_axes = d.locked_axes;
    j.contacts_enabled = d.contacts_enabled;
    j.natural_frequency = d.natural_frequency;
    j.damping_ratio = d.damping_ratio;
    j.limit_axes = d.limit_axes; j.motor_axes = d.motor_axes; j.coupled_axes = d.coupled_axes & 63u;
    for (int k = 0; k < 6; ++k) {
        j.impulses[k] = 0.0f; j.limit_impulses[k] = 0.0f; j.motor_impulses[k] = 0.0f;
        j.limits[k][0] = d.limits[k][0]; j.limits[k][1] = d.limits[k][1];
        j.motors[k] = d.motors[k];
    }
    for (int k = 0; k < 3; ++k) {   // AngularLimitParams::new (joint_constraint_helper.rs:44-73)
        const float lo = d.limits[3 + k][0], hi = d.limits[3 + k][1];
        const float half_range = (hi - lo) * 0.5f;
        if (half_range >= 3.14159265358979323846f || half_range != half_range) {
            j.ang_limit_center[k][0] = 1.0f; j.ang_limit_center[k][1] = 0.0f; j.ang_limit_half_range[k] = 10.0f;
        } else {
            const float center = (lo + hi) * 0.5f;
            j.ang_limit_center[k][0] = cosf(center * 0.5f); j.ang_limit_center[k][1] = sinf(center * 0.5f);
            j.ang_limit_half_range[k] = half_range;
        }
    }
    return RB_OK;
}

// Everything derived from the joint set as a whole, recomputed whenever it changes (scene upload, insert_joints,
// remove_joints -- as the library's upload_joints does): the body pairs whose contacts a joint disables, and the greedy first-fit
// colouring in joint order (interaction_groups.rs:59-165: dyn-dyn from colour 0 up (< 120), dyn-fixed from 127 down).
static void refresh_joint_set(World& w) {
    const int nb = (int)w.bodies.size();
    w.nocontact_body_pairs.clear();
    for (const Joint& j : w.joints) {
        if (j.removed || j.contacts_enabled) continue;
        uint32_t lo = (uint32_t)std::min(j.body1, j.body2), hi = (uint32_t)std::max(j.body1, j.body2);
        w.nocontact_body_pairs.push_back(((uint64_t)lo << 32) | hi);
    }
    std::sort(w.nocontact_body_pairs.begin(), w.nocontact_body_pairs.end());
    std::vector<Mask128> jm(nb);
    for (Joint& j : w.joints) {
        if (j.removed) { j.color = -1; continue; }
        bool d1 = w.bodies[j.body1].is_dynamic(), d2 = w.bodies[j.body2].is_dynamic();
        j.sid1 = d1 ? (uint32_t)j.body1 : NO_BODY;
        j.sid2 = d2 ? (uint32_t)j.body2 : NO_BODY;
        j.color = 128;
        if (d1 && d2) {
            for (int c = 0; c < DYNAMIC_COLOR_COUNT; ++c)
                if (!jm[j.body1].test(c) && !jm[j.body2].test(c)) { j.color = c; break; }
            if (j.color < 128) { jm[j.body1].set(j.color); jm[j.body2].set(j.color); }
        } else if (d1 || d2) {
            int b = d1 ? j.body1 : j.body2;
            for (int c = 127; c >= 0; --c)
                if (!jm[b].test(c)) { j.color = c; break; }
            if (j.color < 128) jm[b].set(j.color);
        } else {
            j.color = -1;  // both fixed: never selected (impulse_joint_set.rs:548-553)
        }
    }
    w.bp_dirty = true;        // (the pair filter changed)
    w.islands_dirty = true;
}

// Mirrors of rb_world_insert_joints / rb_world_remove_joints (ImpulseJointSet::insert / remove after the upload).
static void wake_island_of(World& w, int body);
int insert_joints(World& w, int n, const RbJointDesc* jd) {
    const size_t n0 = w.joints.size();
    w.joints.resize(n0 + n, Joint{});
    for (int i = 0; i < n; ++i) {
        int rc = fill_joint(w, w.joints[n0 + i], jd[i]);
        if (rc != RB_OK) { w.joints.resize(n0); return rc; }
    }
    refresh_joint_set(w);
    w.counters.num_joints = (int)w.joints.size();
    for (int i = 0; i < n; ++i) { wake_island_of(w, jd[i].body1); wake_island_of(w, jd[i].body2); }   // insert(.., wake_up = true)
    return RB_OK;
}
static void wake_island_of(World& w, int body);
int update_joints(World& w, int n, const int* indices, const RbJointDesc* jd, int wake_up) {   // rb_world_update_joints
    for (int k = 0; k < n; ++k) {   // every entry is checked before any is applied
        if (indices[k] < 0 || indices[k] >= (int)w.joints.size() || w.joints[indices[k]].removed) return RB_ERR_INVALID;
        if (jd[k].body1 != w.joints[indices[k]].body1 || jd[k].body2 != w.joints[indices[k]].body2) return RB_ERR_INVALID;
    }
    for (int k = 0; k < n; ++k) {
        Joint& j = w.joints[indices[k]];
        float imp[3][6];
        for (int a = 0; a < 6; ++a) { imp[0][a] = j.impulses[a]; imp[1][a] = j.limit_impulses[a]; imp[2][a] = j.motor_impulses[a]; }
        int rc = fill_joint(w, j, jd[k]);
        if (rc != RB_OK) return rc;
        for (int a = 0; a < 6; ++a) { j.impulses[a] = imp[0][a]; j.limit_impulses[a] = imp[1][a]; j.motor_impulses[a] = imp[2][a]; }
    }
    refresh_joint_set(w);
    if (wake_up)
        for (int k = 0; k < n; ++k) { wake_island_of(w, jd[k].body1); wake_island_of(w, jd[k].body2); }
    return RB_OK;
}
int remove_joints(World& w, int n, const int* indices) {
    for (int k = 0; k < n; ++k)
        if (indices[k] < 0 || indices[k] >= (int)w.joints.size()) return RB_ERR_INVALID;
    for (int k = 0; k < n; ++k) w.joints[indices[k]].removed = true;
    refresh_joint_set(w);
    return RB_OK;
}

int set_scene(World& w, int nb, const RbBodyDesc* bd, int nc, const RbColliderDesc* cd, int nj,
              const RbJointDesc* jd) {
    w.bodies.assign(nb, Body{});
    w.colliders.assign(nc, Collider{});
    w.joints.assign(nj, Joint{});
    w.pairs.clear();
    w.color_masks.assign(nb, Mask128{});
    w.bp_dirty = true;
    w.static_dirty = true;
    w.islands_dirty = true;
    w.island_of.clear();
    for (int i = 0; i < nb; ++i) {
        Body& b = w.bodies[i];
        const RbBodyDesc& d = bd[i];
        b.type = d.body_type;
        b.flags = d.flags;
        b.pos = Pose{f4(d.rotation), f3(d.translation)};
        b.next_pos = b.pos;
        b.kin_target = b.pos;
        b.linvel = f3(d.linvel);
        b.angvel = f3(d.angvel);
        b.lin_damping = d.linear_damping;
        b.ang_damping = d.angular_damping;
        b.gravity_scale = d.gravity_scale;
        b.additional_mass = d.additional_mass;
        b.user_force = f3(d.user_force);
        b.user_torque = f3(d.user_torque);
        b.force = vzero();
        b.torque = vzero();
    }
    for (int i = 0; i < nc; ++i) {
        Collider& c = w.colliders[i];
        const RbColliderDesc& d = cd[i];
        if (d.shape != RB_SHAPE_BALL && d.shape != RB_SHAPE_CUBOID && d.shape != RB_SHAPE_CAPSULE && d.shape != RB_SHAPE_CONVEX) return RB_ERR_INVALID;
        if (d.shape == RB_SHAPE_CONVEX && !(d.half_extents[0] >= 0.0f && d.half_extents[0] < (float)w.hulls.size())) return RB_ERR_INVALID;
        if (d.parent >= nb) return RB_ERR_INVALID;
        c.shape = d.shape;
        c.he = f3(d.half_extents);
        c.parent = d.parent;
        c.pos_wrt_parent = Pose{f4(d.pos_wrt_parent_q), f3(d.pos_wrt_parent_t)};
        c.density = d.density;
        c.friction = d.friction;
        c.restitution = d.restitution;
        c.friction_rule = d.friction_combine_rule;
        c.restitution_rule = d.restitution_combine_rule;
        c.contact_skin = d.contact_skin;
        c.active_events = d.active_events;
        c.sensor = d.sensor;
    c.force_event_threshold = d.contact_force_event_threshold;
    c.memberships = d.collision_memberships;
        c.filter = d.collision_filter;
        c.fat_valid = false;
    }
    int rc = recompute_mass_properties(w);
    if (rc != RB_OK) return rc;
    for (Body& b : w.bodies) update_world_mass_properties(b);
    for (Collider& c : w.colliders) refresh_collider(w, c);
    for (int i = 0; i < nj; ++i) {
        int rcj = fill_joint(w, w.joints[i], jd[i]);
        if (rcj != RB_OK) return rcj;
    }
    refresh_joint_set(w);
    w.counters = RbCounters{};
    w.counters.num_bodies = nb;
    w.counters.num_colliders = nc;
    w.counters.num_joints = nj;
    return RB_OK;
}


// Incremental changes of the sets (src/pipeline/user_changes.rs:11-46): appended bodies / colliders keep every
// existing index, so the persistent pair list (merged by collider key), colours and warm-start data survive.
static void fill_body(Body& b, const RbBodyDesc& d) {
    b.type = d.body_type;
    b.flags = d.flags;
    b.pos = Pose{f4(d.rotation), f3(d.translation)};
    b.next_pos = b.pos;
    b.kin_target = b.pos;
    b.linvel = f3(d.linvel);
    b.angvel = f3(d.angvel);
    b.lin_damping = d.linear_damping;
    b.ang_damping = d.angular_damping;
    b.gravity_scale = d.gravity_scale;
    b.additional_mass = d.additional_mass;
    b.user_force = f3(d.user_force);
    b.user_torque = f3(d.user_torque);
    b.force = vzero();
    b.torque = vzero();
}
static void fill_collider(Collider& c, const RbColliderDesc& d) {
    c.shape = d.shape;
    c.he = f3(d.half_extents);
    c.parent = d.parent;
    c.pos_wrt_parent = Pose{f4(d.pos_wrt_parent_q), f3(d.pos_wrt_parent_t)};
    c.density = d.density;
    c.friction = d.friction;
    c.restitution = d.restitution;
    c.friction_rule = d.friction_combine_rule;
    c.restitution_rule = d.restitution_combine_rule;
    c.contact_skin = d.contact_skin;
    c.active_events = d.active_events;
    c.sensor = d.sensor;
    c.force_event_threshold = d.contact_force_event_threshold;
    c.memberships = d.collision_memberships;
    c.filter = d.collision_filter;
    c.fat_valid = false;
}
int insert(World& w, int nb, const RbBodyDesc* bd, int nc, const RbColliderDesc* cd) {
    const int nb0 = (int)w.bodies.size(), nc0 = (int)w.colliders.size();
    for (int i = 0; i < nc; ++i) {
        if (cd[i].shape != RB_SHAPE_BALL && cd[i].shape != RB_SHAPE_CUBOID && cd[i].shape != RB_SHAPE_CAPSULE && cd[i].shape != RB_SHAPE_CONVEX) return RB_ERR_INVALID;
        if (cd[i].shape == RB_SHAPE_CONVEX && !(cd[i].half_extents[0] >= 0.0f && cd[i].half_extents[0] < (float)w.hulls.size())) return RB_ERR_INVALID;
        if (cd[i].parent >= nb0 + nb || (cd[i].parent >= 0 && cd[i].parent < nb0)) return RB_ERR_INVALID;
    }
    w.bodies.resize(nb0 + nb);
    w.colliders.resize(nc0 + nc);
    w.color_masks.resize(nb0 + nb, Mask128{});
    for (int i = 0; i < nb; ++i) { w.bodies[nb0 + i] = Body{}; fill_body(w.bodies[nb0 + i], bd[i]); }
    for (int i = 0; i < nc; ++i) { w.colliders[nc0 + i] = Collider{}; fill_collider(w.colliders[nc0 + i], cd[i]); }
    int rc = recompute_mass_properties(w, nb0, nc0);
    if (rc != RB_OK) return rc;
    for (int i = nb0; i < nb0 + nb; ++i) update_world_mass_properties(w.bodies[i]);
    for (int i = nc0; i < nc0 + nc; ++i) refresh_collider(w, w.colliders[i]);
    w.bp_dirty = true;
    w.static_dirty = true;
    w.islands_dirty = true;
    w.counters.num_bodies = nb0 + nb;
    w.counters.num_colliders = nc0 + nc;
    return RB_OK;
}
int remove_bodies(World& w, int n, const int* indices) {
    for (int k = 0; k < n; ++k)
        if (indices[k] < 0 || indices[k] >= (int)w.bodies.size()) return RB_ERR_INVALID;
    for (int k = 0; k < n; ++k) {
        w.bodies[indices[k]].type = 7;   // removed: not dynamic, never simulated again
        for (Collider& c : w.colliders)
            if (c.parent == indices[k]) c.shape = -1;   // leaves the broad phase: its pairs end at the next step
    }
    for (Body& b : w.bodies)
        if (b.sleeping) { b.sleeping = false; b.sleep_time = 0.0f; }   // (the reference wakes what touched the removed body; here: everything)
    w.bp_dirty = true;
    w.static_dirty = true;
    w.islands_dirty = true;
    return RB_OK;
}

// Unit-level known-answer entry points of this file (see kat_solver in oracle_solver.cpp).
int kat_world(const char* name_c, const float* in, int n_in, float* out, int n_out) {
    const std::string name(name_c);
    if (name == "pose_drift") {   // contact_pair.rs:299-323
        if (n_in < 15 || n_out < 1) return -3;
        Pose base{Q4{in[3], in[4], in[5], in[6]}, V3{in[0], in[1], in[2]}};
        Pose cur{Q4{in[10], in[11], in[12], in[13]}, V3{in[7], in[8], in[9]}};
        out[0] = relative_pose_drift(base, cur, in[14]);
        return 0;
    }
    if (name == "combine_coeff") {   // coefficient_combine_rule.rs:51-84: c1, c2, rule1, rule2
        if (n_in < 4 || n_out < 1) return -3;
        out[0] = combine_coeff(in[0], in[1], (int)in[2], (int)in[3]);
        return 0;
    }
    if (name == "reduce_manifold") {   // manifold_reduction.rs:4-84
        if (n_in < 5 || n_out < 5) return -3;
        RawManifold m{};
        m.n = (int)in[0];
        if (m.n < 0 || m.n > MAX_RAW_POINTS || n_in < 5 + 4 * m.n) return -3;
        m.local_n1 = V3{in[2], in[3], in[4]};
        for (int i = 0; i < m.n; ++i) { m.pts[i].local_p1 = V3{in[5 + 4 * i], in[6 + 4 * i], in[7 + 4 * i]}; m.pts[i].dist = in[8 + 4 * i]; }
        int sel[4] = {0, 1, 2, 3};
        int nsel = m.n < MAX_MANIFOLD_POINTS ? m.n : MAX_MANIFOLD_POINTS;
        reduce_manifold_naive(m, sel, nsel, in[1]);
        out[0] = (float)nsel;
        for (int i = 0; i < 4; ++i) out[1 + i] = i < nsel ? (float)sel[i] : -1.0f;
        return 0;
    }
    return -100;
}

}  // namespace orc
