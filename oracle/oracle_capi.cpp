// TEST INFRASTRUCTURE ONLY -- C entry points of the CPU oracle (see oracle.h header note).
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include "oracle_internal.h"

namespace orc {
void step_once(World& w, V3 gravity);
int set_scene(World& w, int nb, const RbBodyDesc* bd, int nc, const RbColliderDesc* cd, int nj, const RbJointDesc* jd);
int insert(World& w, int nb, const RbBodyDesc* bd, int nc, const RbColliderDesc* cd);
int remove_bodies(World& w, int n, const int* indices);
int insert_joints(World& w, int n, const RbJointDesc* jd);
int remove_joints(World& w, int n, const int* indices);
int update_joints(World& w, int n, const int* indices, const RbJointDesc* jd, int wake_up);
void update_world_mass_properties(Body& b);
void refresh_collider(World& w, Collider& c);
void set_threads(int n);
int get_threads();
}  // namespace orc

using namespace orc;

struct OrcWorld {
    World w;
};

static void default_params(RbIntegrationParameters* p) {  // integration_parameters.rs:379-407
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

static int64_t copy_out(const std::vector<uint8_t>& buf, void* dst, int64_t cap) {
    int64_t n = (int64_t)buf.size() < cap ? (int64_t)buf.size() : cap;
    if (dst && n > 0) memcpy(dst, buf.data(), (size_t)n);
    return (int64_t)buf.size();
}
template <class T>
static void put(std::vector<uint8_t>& b, T v) {
    size_t o = b.size();
    b.resize(o + sizeof(T));
    memcpy(b.data() + o, &v, sizeof(T));
}
static void put3(std::vector<uint8_t>& b, V3 v) { put(b, v.x); put(b, v.y); put(b, v.z); }

extern "C" {

OrcWorld* orc_world_create(const RbIntegrationParameters* params) {
    OrcWorld* o = new OrcWorld();
    if (params) o->w.params.p = *params;
    else default_params(&o->w.params.p);
    o->w.hulls.emplace_back();
    hull_unit_cube(o->w.hulls[0]);
    return o;
}
int32_t orc_world_add_hull(OrcWorld* o, int32_t nv, const float* verts, int32_t nf, const int32_t* face_sizes, const int32_t* face_indices) {
    if (!o || !verts || !face_sizes || !face_indices) return RB_ERR_INVALID;
    Hull h;
    if (!hull_from_mesh(nv, verts, nf, face_sizes, face_indices, h)) return RB_ERR_INVALID;
    o->w.hulls.push_back(h);
    return (int32_t)o->w.hulls.size() - 1;
}
void orc_world_destroy(OrcWorld* w) { delete w; }
int orc_world_set_params(OrcWorld* w, const RbIntegrationParameters* params) {
    if (!w || !params) return RB_ERR_INVALID;
    w->w.params.p = *params;
    return RB_OK;
}
int orc_world_set_scene(OrcWorld* w, int32_t nb, const RbBodyDesc* bodies, int32_t nc, const RbColliderDesc* colliders,
                        int32_t nj, const RbJointDesc* joints) {
    if (!w) return RB_ERR_INVALID;
    return set_scene(w->w, nb, bodies, nc, colliders, nj, joints);
}
// rb_world_* checks every index of a set-editing call before it changes anything; so do these mirrors.
static bool bodies_valid(const World& w, int n, const int32_t* indices, int type = -1) {
    for (int k = 0; k < n; ++k)
        if (indices[k] < 0 || indices[k] >= (int)w.bodies.size() || (type >= 0 && w.bodies[indices[k]].type != type)) return false;
    return true;
}
int orc_world_wake_up(OrcWorld* o, int32_t n, const int32_t* indices) {
    if (!o || n < 0 || !bodies_valid(o->w, n, indices)) return RB_ERR_INVALID;
    World& w = o->w;
    for (int k = 0; k < n; ++k) {
        const int i = indices[k];
        if (!w.bodies[i].is_dynamic()) continue;
        const int root = i < (int)w.island_of.size() ? w.island_of[i] : -1;
        for (int b = 0; b < (int)w.bodies.size(); ++b) {
            const bool same = b == i || (root >= 0 && b < (int)w.island_of.size() && w.island_of[b] == root);
            if (same && w.bodies[b].sleeping) { w.bodies[b].sleeping = false; w.bodies[b].sleep_time = 0.0f; }
        }
    }
    return RB_OK;
}
int orc_world_get_quarantine(OrcWorld* o, int32_t* bodies, int32_t cap) {
    if (!o) return RB_ERR_INVALID;
    std::vector<int>& q = o->w.quarantine;
    const int n = (int)q.size();
    if (bodies && cap > 0 && n > 0) {
        std::sort(q.begin(), q.end());
        for (int i = 0; i < n && i < cap; ++i) bodies[i] = q[i];
        q.clear();
    }
    return n;
}
int orc_world_get_sleeping(OrcWorld* o, uint8_t* out) {
    if (!o || !out) return RB_ERR_INVALID;
    for (size_t i = 0; i < o->w.bodies.size(); ++i) out[i] = o->w.bodies[i].sleeping ? 1 : 0;
    return RB_OK;
}
int orc_world_insert(OrcWorld* w, int32_t nb, const RbBodyDesc* bodies, int32_t nc, const RbColliderDesc* colliders) {
    if (!w || nb < 0 || nc < 0) return RB_ERR_INVALID;
    return insert(w->w, nb, bodies, nc, colliders);
}
int orc_world_remove_bodies(OrcWorld* w, int32_t n, const int32_t* indices) {
    if (!w || n < 0) return RB_ERR_INVALID;
    return remove_bodies(w->w, n, indices);
}
int orc_world_insert_joints(OrcWorld* w, int32_t n, const RbJointDesc* joints) {
    if (!w || n < 0 || (n && !joints)) return RB_ERR_INVALID;
    return insert_joints(w->w, n, joints);
}
int orc_world_update_joints(OrcWorld* w, int32_t n, const int32_t* indices, const RbJointDesc* joints, int32_t wake_up) {
    if (!w || n < 0 || (n && (!indices || !joints))) return RB_ERR_INVALID;
    return update_joints(w->w, n, indices, joints, wake_up);
}
int orc_world_remove_joints(OrcWorld* w, int32_t n, const int32_t* indices) {
    if (!w || n < 0 || (n && !indices)) return RB_ERR_INVALID;
    return remove_joints(w->w, n, indices);
}
int orc_world_set_body_states(OrcWorld* o, int32_t n, const int32_t* indices, const float* pose7, const float* vel6) {
    if (!o || n < 0 || !bodies_valid(o->w, n, indices)) return RB_ERR_INVALID;
    World& w = o->w;
    for (int k = 0; k < n; ++k) {
        int i = indices[k];
        Body& b = w.bodies[i];
        if (pose7) {
            b.pos.t = V3{pose7[k * 7 + 0], pose7[k * 7 + 1], pose7[k * 7 + 2]};
            b.pos.q = Q4{pose7[k * 7 + 3], pose7[k * 7 + 4], pose7[k * 7 + 5], pose7[k * 7 + 6]};
            b.next_pos = b.pos;
            b.kin_target = b.pos;
            if (!b.is_dynamic()) w.static_dirty = true;   // a teleported fixed body moves static colliders
            update_world_mass_properties(b);
            for (Collider& c : w.colliders)
                if (c.parent == i) refresh_collider(w, c);
        }
        if (vel6) {
            b.linvel = V3{vel6[k * 6 + 0], vel6[k * 6 + 1], vel6[k * 6 + 2]};
            b.angvel = V3{vel6[k * 6 + 3], vel6[k * 6 + 4], vel6[k * 6 + 5]};
        }
    }
    return orc_world_wake_up(o, n, indices);   // a user change wakes the body's island (user_changes.rs)
}
int orc_world_set_body_forces(OrcWorld* o, int32_t n, const int32_t* indices, const float* force3, const float* torque3) {
    if (!o || n < 0 || !bodies_valid(o->w, n, indices)) return RB_ERR_INVALID;
    World& w = o->w;
    for (int k = 0; k < n; ++k) {
        int i = indices[k];
        if (force3) w.bodies[i].user_force = V3{force3[k * 3], force3[k * 3 + 1], force3[k * 3 + 2]};
        if (torque3) w.bodies[i].user_torque = V3{torque3[k * 3], torque3[k * 3 + 1], torque3[k * 3 + 2]};
    }
    return orc_world_wake_up(o, n, indices);
}
int orc_world_set_next_kinematic_positions(OrcWorld* o, int32_t n, const int32_t* indices, const float* pose7) {
    if (!o || !pose7 || n < 0 || !bodies_valid(o->w, n, indices, RB_BODY_KINEMATIC_POSITION_BASED)) return RB_ERR_INVALID;
    World& w = o->w;
    for (int k = 0; k < n; ++k) {
        int i = indices[k];
        w.bodies[i].kin_target = Pose{Q4{pose7[k * 7 + 3], pose7[k * 7 + 4], pose7[k * 7 + 5], pose7[k * 7 + 6]}, V3{pose7[k * 7], pose7[k * 7 + 1], pose7[k * 7 + 2]}};
    }
    return orc_world_wake_up(o, n, indices);
}
int orc_world_drain_collision_events(OrcWorld* o, int32_t cap, RbCollisionEvent* out) {
    if (!o) return RB_ERR_INVALID;
    std::vector<RbCollisionEvent>& ev = o->w.collision_events;
    const int n = (int)ev.size();
    std::sort(ev.begin(), ev.end(), [](const RbCollisionEvent& a, const RbCollisionEvent& b) {   // the drain order of the C ABI: (step, collider1, collider2, started)
        if (a.step != b.step) return a.step < b.step;
        if (a.collider1 != b.collider1) return a.collider1 < b.collider1;
        if (a.collider2 != b.collider2) return a.collider2 < b.collider2;
        return a.started < b.started;
    });
    auto is_sensor = [&](int c) { return c >= 0 && c < (int)o->w.colliders.size() && o->w.colliders[c].sensor != 0; };
    for (int i = 0; i < n && i < cap && out; ++i) {
        out[i] = ev[i];
        out[i].flags = (is_sensor(ev[i].collider1) || is_sensor(ev[i].collider2)) ? RB_COLLISION_EVENT_SENSOR : 0;
    }
    ev.clear();
    return n;
}
int orc_world_drain_contact_force_events(OrcWorld* o, int32_t cap, RbContactForceEvent* out) {
    if (!o) return RB_ERR_INVALID;
    std::vector<RbContactForceEvent>& ev = o->w.force_events;
    const int n = (int)ev.size();
    for (int i = 0; i < n && i < cap && out; ++i) out[i] = ev[i];
    ev.clear();
    return n;
}
int orc_world_step(OrcWorld* w, const float gravity[3], int32_t nsteps) {
    if (!w || !gravity) return RB_ERR_INVALID;
    for (int i = 0; i < nsteps; ++i) step_once(w->w, V3{gravity[0], gravity[1], gravity[2]});
    return RB_OK;
}
int orc_world_get_body_states(OrcWorld* o, float* pose7, float* vel6) {
    if (!o) return RB_ERR_INVALID;
    World& w = o->w;
    for (size_t i = 0; i < w.bodies.size(); ++i) {
        const Body& b = w.bodies[i];
        if (pose7) {
            float* p = pose7 + i * 7;
            p[0] = b.pos.t.x; p[1] = b.pos.t.y; p[2] = b.pos.t.z;
            p[3] = b.pos.q.x; p[4] = b.pos.q.y; p[5] = b.pos.q.z; p[6] = b.pos.q.w;
        }
        if (vel6) {
            float* v = vel6 + i * 6;
            v[0] = b.linvel.x; v[1] = b.linvel.y; v[2] = b.linvel.z;
            v[3] = b.angvel.x; v[4] = b.angvel.y; v[5] = b.angvel.z;
        }
    }
    return RB_OK;
}
int orc_world_num_bodies(OrcWorld* w) { return w ? (int)w->w.bodies.size() : RB_ERR_INVALID; }
int orc_world_get_counters(OrcWorld* w, RbCounters* out) {
    if (!w || !out) return RB_ERR_INVALID;
    *out = w->w.counters;
    out->num_pairs = (int)w->w.pairs.size();
    return RB_OK;
}
int orc_world_get_contact_pairs(OrcWorld* o, int32_t cap, int32_t* pair_colliders, int32_t* num_contacts, int32_t* color,
                                float* normal, float* impulses) {
    if (!o) return RB_ERR_INVALID;
    World& w = o->w;
    int n = (int)w.pairs.size();
    for (int i = 0; i < n && i < cap; ++i) {
        const Pair& p = w.pairs[i];
        if (pair_colliders) { pair_colliders[2 * i] = p.c1; pair_colliders[2 * i + 1] = p.c2; }
        if (num_contacts) num_contacts[i] = p.nsc;
        if (color) color[i] = p.color;
        if (normal) { normal[3 * i] = p.normal.x; normal[3 * i + 1] = p.normal.y; normal[3 * i + 2] = p.normal.z; }
        if (impulses)
            for (int k = 0; k < 4; ++k) impulses[4 * i + k] = k < p.nsc ? p.pts[p.sc[k].cid].impulse : 0.0f;
    }
    return n;
}

int64_t orc_world_debug_read(OrcWorld* o, const char* table, void* dst, int64_t cap) {
    if (!o || !table) return RB_ERR_INVALID;
    World& w = o->w;
    std::string t(table);
    std::vector<uint8_t> b;
    if (t == "pair_keys") {
        for (const Pair& p : w.pairs) put<uint64_t>(b, ((uint64_t)(uint32_t)p.c1 << 32) | (uint32_t)p.c2);
    } else if (t == "pair_nsc") {
        for (const Pair& p : w.pairs) put<int32_t>(b, p.nsc);
    } else if (t == "pair_npts") {
        for (const Pair& p : w.pairs) put<int32_t>(b, p.npts);
    } else if (t == "pair_color") {
        for (const Pair& p : w.pairs) put<int32_t>(b, p.color);
    } else if (t == "pair_normal") {
        for (const Pair& p : w.pairs) put3(b, p.normal);
    } else if (t == "pair_points") {  // 4 x {local_p1, local_p2, dist, fid1, fid2}
        for (const Pair& p : w.pairs)
            for (int k = 0; k < 4; ++k) {
                const Point& q = p.pts[k];
                bool v = k < p.npts;
                put3(b, v ? q.local_p1 : vzero()); put3(b, v ? q.local_p2 : vzero());
                put<float>(b, v ? q.dist : 0.0f); put<uint32_t>(b, v ? q.fid1 : 0u); put<uint32_t>(b, v ? q.fid2 : 0u);
            }
    } else if (t == "pair_data") {  // 4 x {impulse, warmstart_impulse, warmstart_twist, tangent_world, dp1, dp2}
        for (const Pair& p : w.pairs)
            for (int k = 0; k < 4; ++k) {
                const Point& q = p.pts[k];
                bool v = k < p.npts;
                put<float>(b, v ? q.impulse : 0.0f); put<float>(b, v ? q.warmstart_impulse : 0.0f);
                put<float>(b, v ? q.warmstart_twist : 0.0f);
                put3(b, v ? q.warmstart_tangent_world : vzero()); put3(b, v ? q.dp1 : vzero()); put3(b, v ? q.dp2 : vzero());
            }
    } else if (t == "pair_sc") {  // 4 x {anchor1, anchor2, cid}
        for (const Pair& p : w.pairs)
            for (int k = 0; k < 4; ++k) {
                bool v = k < p.nsc;
                put3(b, v ? p.sc[k].anchor1 : vzero()); put3(b, v ? p.sc[k].anchor2 : vzero());
                put<int32_t>(b, v ? p.sc[k].cid : -1);
            }
    } else if (t == "collider_aabb") {
        for (const Collider& c : w.colliders) { put3(b, c.aabb.mins); put3(b, c.aabb.maxs); }
    } else if (t == "collider_fat") {
        for (const Collider& c : w.colliders) { put3(b, c.fat.mins); put3(b, c.fat.maxs); }
    } else if (t == "body_mprops") {  // local_com(3), inv_mass, inv_principal(3), world_com(3), eff_ii(6)
        for (const Body& q : w.bodies) {
            put3(b, q.local_com); put<float>(b, q.inv_mass); put3(b, q.inv_principal_inertia); put3(b, q.world_com);
            put<float>(b, q.eff_world_inv_inertia.m11); put<float>(b, q.eff_world_inv_inertia.m12);
            put<float>(b, q.eff_world_inv_inertia.m13); put<float>(b, q.eff_world_inv_inertia.m22);
            put<float>(b, q.eff_world_inv_inertia.m23); put<float>(b, q.eff_world_inv_inertia.m33);
        }
    } else if (t == "body_mframe") {  // principal frame xyzw, effective inverse mass xyz
        for (const Body& q : w.bodies) {
            put<float>(b, q.principal_frame.x); put<float>(b, q.principal_frame.y); put<float>(b, q.principal_frame.z);
            put<float>(b, q.principal_frame.w); put3(b, q.eff_inv_mass);
        }
    } else if (t == "hull_tables") {  // the layout of rb_world_debug_read's table, over every registered hull
        for (const Hull& h : w.hulls) {
            const int nv = (int)h.verts.size(), nf = (int)h.face_count.size(), ne = (int)h.edges.size(), nl = (int)h.loops.size();
            put<int32_t>(b, nv); put<int32_t>(b, nf); put<int32_t>(b, ne); put<int32_t>(b, nl);
            put3(b, h.aabb); put<float>(b, h.radius);
            for (const V3& v : h.verts) put3(b, v);
            for (int f = 0; f < nf; ++f) { put3(b, h.normals[f]); put<float>(b, h.offsets[f]); }
            for (int f = 0; f < nf; ++f) { put<int32_t>(b, h.face_start[f]); put<int32_t>(b, h.face_count[f]); }
            for (int l : h.loops) put<int32_t>(b, l);
            for (const HullEdge& e : h.edges) { put<int32_t>(b, e.v0); put<int32_t>(b, e.v1); put<int32_t>(b, e.f0); put<int32_t>(b, e.f1); }
        }
    } else if (t == "joint_impulses") {
        for (const Joint& j : w.joints)
            for (int k = 0; k < 6; ++k) put<float>(b, j.impulses[k]);
    } else if (t == "joint_color") {
        for (const Joint& j : w.joints) put<int32_t>(b, j.color);
    } else if (t == "island_of") {   // connected component (root body) of every dynamic / kinematic body, -1 otherwise (as of the last step)
        for (size_t i = 0; i < w.bodies.size(); ++i) put<int32_t>(b, i < w.island_of.size() ? w.island_of[i] : -1);
    } else {
        return RB_ERR_INVALID;
    }
    return copy_out(b, dst, cap);
}

void orc_set_threads(int n) { set_threads(n); }
int orc_get_threads(void) { return get_threads(); }

int orc_contact_manifold(int shape1, const float he1[3], int shape2, const float he2[3], const float pos12_t[3],
                         const float pos12_q[4], float prediction, float* out_points, float out_n1[3], float out_n2[3]) {
    RawManifold m;
    Pose pos12{Q4{pos12_q[0], pos12_q[1], pos12_q[2], pos12_q[3]}, V3{pos12_t[0], pos12_t[1], pos12_t[2]}};
    contact_manifold(shape1, V3{he1[0], he1[1], he1[2]}, shape2, V3{he2[0], he2[1], he2[2]}, pos12, prediction, m);
    for (int i = 0; i < m.n; ++i) {
        float* o = out_points + i * 9;
        o[0] = m.pts[i].local_p1.x; o[1] = m.pts[i].local_p1.y; o[2] = m.pts[i].local_p1.z;
        o[3] = m.pts[i].local_p2.x; o[4] = m.pts[i].local_p2.y; o[5] = m.pts[i].local_p2.z;
        o[6] = m.pts[i].dist;
        memcpy(&o[7], &m.pts[i].fid1, 4);
        memcpy(&o[8], &m.pts[i].fid2, 4);
    }
    out_n1[0] = m.local_n1.x; out_n1[1] = m.local_n1.y; out_n1[2] = m.local_n1.z;
    out_n2[0] = m.local_n2.x; out_n2[1] = m.local_n2.y; out_n2[2] = m.local_n2.z;
    return m.n;
}

// Unit-level known-answer entry point: evaluates ONE function of the restated path on literal inputs
// (names and float layouts: tests/golden/make_ref_vectors.py, and for ccd_toi / ccd_moving_fast / atan2_poly /
// quat_angle tests/test_ccd_reference.py; mirrored by rb_debug_kat).
static int kat_ccd(const char* name_c, const float* in, int n_in, float* out, int n_out) {
    const std::string name(name_c);
    auto v3at = [&](int o) { return V3{in[o], in[o + 1], in[o + 2]}; };
    auto poseat = [&](int o) { return Pose{Q4{in[o], in[o + 1], in[o + 2], in[o + 3]}, v3at(o + 4)}; };   // q (x, y, z, w) then t
    if (name == "ccd_toi") {
        if (n_in < 33 || n_out < 1) return -3;
        const Sweep sw = sweep_from_poses(poseat(15), poseat(22), v3at(29));
        out[0] = toi((int)in[0], v3at(1), poseat(4), (int)in[11], v3at(12), sw, in[32]);
        return 0;
    }
    if (name == "ccd_moving_fast") {
        if (n_in < 19 || n_out < 1) return -3;
        RbIntegrationParameters p;
        default_params(&p);
        out[0] = is_moving_fast(p, v3at(0), poseat(3), poseat(10), in[17], in[18]) ? 1.0f : 0.0f;
        return 0;
    }
    if (name == "atan2_poly" || name == "quat_angle") {
        if (n_in < 2 || n_out < 1) return -3;
        out[0] = name == "atan2_poly" ? atan2_poly(in[0], in[1]) : ccd_quat_angle(in[0], in[1]);
        return 0;
    }
    return -100;
}

int orc_kat(const char* name, const float* in, int32_t n_in, float* out, int32_t n_out) {
    if (!name || !in || !out) return RB_ERR_INVALID;
    int rc = kat_ccd(name, in, n_in, out, n_out);
    if (rc == -100) rc = kat_solver(name, in, n_in, out, n_out);
    if (rc == -100) rc = kat_world(name, in, n_in, out, n_out);
    return rc == -100 ? RB_ERR_INVALID : rc;
}

}  // extern "C"
