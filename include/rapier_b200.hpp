// rapier_b200.hpp -- header-only C++ host mirror of the reference's step API over the C ABI.
//
// The reference's host language is Rust (absent from this image); this is the compiled-language
// mirror of the same surface: RigidBodyBuilder / ColliderBuilder (src/dynamics/rigid_body.rs:1490-1580,
// src/geometry/collider.rs:688-707), RigidBodySet / ColliderSet / ImpulseJointSet (index handles),
// IntegrationParameters::default() (integration_parameters.rs:379-407), PhysicsPipeline::step
// (physics_pipeline/mod.rs:196-247) and the PhysicsWorld facade (physics_world.rs:120-207).
// Every method is a thin call into librapier_b200.so; no physics is computed here.
#pragma once
#include <array>
#include <cfloat>
#include <cmath>
#include <stdexcept>
#include <string>
#include <vector>

#include "rapier_b200.h"

namespace rapier_b200 {

using Vector = std::array<float, 3>;

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
inline void check(int rc) {
    if (rc < 0) throw Error(rc, std::string("rapier_b200 status ") + std::to_string(rc) + ": " + rb_last_error());
}

struct IntegrationParameters : RbIntegrationParameters {
    IntegrationParameters() { rb_integration_parameters_default(this); }
};

struct RigidBodyHandle { int index = -1; };
struct ColliderHandle { int index = -1; };
struct ImpulseJointHandle { int index = -1; };

class RigidBodyBuilder {
public:
    static RigidBodyBuilder dynamic() { return RigidBodyBuilder(RB_BODY_DYNAMIC); }
    static RigidBodyBuilder fixed() { return RigidBodyBuilder(RB_BODY_FIXED); }
    static RigidBodyBuilder kinematic_position_based() { return RigidBodyBuilder(RB_BODY_KINEMATIC_POSITION_BASED); }
    static RigidBodyBuilder kinematic_velocity_based() { return RigidBodyBuilder(RB_BODY_KINEMATIC_VELOCITY_BASED); }
    RigidBodyBuilder& translation(Vector v) { for (int i = 0; i < 3; ++i) d_.translation[i] = v[i]; return *this; }
    RigidBodyBuilder& rotation(Vector axis_angle) {   // scaled axis, like RigidBodyBuilder::rotation
        float a = std::sqrt(axis_angle[0] * axis_angle[0] + axis_angle[1] * axis_angle[1] + axis_angle[2] * axis_angle[2]);
        if (a == 0.0f) { d_.rotation[0] = d_.rotation[1] = d_.rotation[2] = 0.0f; d_.rotation[3] = 1.0f; return *this; }
        float s = std::sin(a / 2.0f) / a;
        for (int i = 0; i < 3; ++i) d_.rotation[i] = axis_angle[i] * s;
        d_.rotation[3] = std::cos(a / 2.0f);
        return *this;
    }
    RigidBodyBuilder& linvel(Vector v) { for (int i = 0; i < 3; ++i) d_.linvel[i] = v[i]; return *this; }
    RigidBodyBuilder& angvel(Vector v) { for (int i = 0; i < 3; ++i) d_.angvel[i] = v[i]; return *this; }
    RigidBodyBuilder& linear_damping(float x) { d_.linear_damping = x; return *this; }
    RigidBodyBuilder& angular_damping(float x) { d_.angular_damping = x; return *this; }
    RigidBodyBuilder& gravity_scale(float x) { d_.gravity_scale = x; return *this; }
    RigidBodyBuilder& additional_mass(float m) { d_.additional_mass = m; return *this; }
    RigidBodyBuilder& dominance_group(int group) {   // RigidBodyBuilder::dominance_group (i8)
        d_.flags = (d_.flags & ~(0xffu << RB_BODY_DOMINANCE_SHIFT)) | RB_BODY_DOMINANCE(group); return *this;
    }
    RigidBodyBuilder& additional_solver_iterations(unsigned n) {   // RigidBodyBuilder::additional_solver_iterations (0..255)
        d_.flags = (d_.flags & ~(0xffu << RB_BODY_EXTRA_ITERS_SHIFT)) | RB_BODY_EXTRA_ITERS(n); return *this;
    }
    RigidBodyBuilder& ccd_enabled(bool on) { if (on) d_.flags |= RB_BODY_CCD_ENABLED; else d_.flags &= ~RB_BODY_CCD_ENABLED; return *this; }
    RigidBodyBuilder& can_sleep(bool on) {   // RigidBodyActivation::cannot_sleep() when false
        if (on) d_.flags &= ~RB_BODY_NO_SLEEP; else d_.flags |= RB_BODY_NO_SLEEP;
        return *this;
    }
    RigidBodyBuilder& gyroscopic_forces_enabled(bool on) {
        if (on) d_.flags |= RB_BODY_GYROSCOPIC; else d_.flags &= ~RB_BODY_GYROSCOPIC;
        return *this;
    }
    const RbBodyDesc& desc() const { return d_; }

private:
    explicit RigidBodyBuilder(int type) : d_{} {
        d_.body_type = type;
        d_.flags = RB_BODY_GYROSCOPIC;   // rigid_body.rs:1579
        d_.rotation[3] = 1.0f;
        d_.gravity_scale = 1.0f;
    }
    RbBodyDesc d_;
};

class ColliderBuilder {
public:
    static ColliderBuilder cuboid(float hx, float hy, float hz) { return ColliderBuilder(RB_SHAPE_CUBOID, hx, hy, hz); }
    static ColliderBuilder ball(float r) { return ColliderBuilder(RB_SHAPE_BALL, r, 0.0f, 0.0f); }
    static ColliderBuilder capsule_y(float half_height, float radius) { return ColliderBuilder(RB_SHAPE_CAPSULE, half_height, radius, 1.0f); }
    ColliderBuilder& density(float x) { d_.density = x; return *this; }
    ColliderBuilder& mass(float m) {   // ColliderMassProps::Mass: the density that gives the shape this mass
        const float* h = d_.half_extents;
        float vol = d_.shape == RB_SHAPE_CUBOID ? 8.0f * h[0] * h[1] * h[2] : 4.18879020478639f * h[0] * h[0] * h[0];
        d_.density = vol > 0.0f ? m / vol : 0.0f;
        return *this;
    }
    ColliderBuilder& friction(float x) { d_.friction = x; return *this; }
    ColliderBuilder& restitution(float x) { d_.restitution = x; return *this; }
    ColliderBuilder& friction_combine_rule(int r) { d_.friction_combine_rule = r; return *this; }
    ColliderBuilder& restitution_combine_rule(int r) { d_.restitution_combine_rule = r; return *this; }
    ColliderBuilder& translation(Vector v) { for (int i = 0; i < 3; ++i) d_.pos_wrt_parent_t[i] = v[i]; return *this; }
    ColliderBuilder& contact_skin(float x) { d_.contact_skin = x; return *this; }
    ColliderBuilder& collision_groups(unsigned memberships, unsigned filter, int test_mode = RB_TEST_AND) {   // RB_TEST_*
        d_.collision_memberships = memberships; d_.collision_filter = filter; f_.collision_test_mode = test_mode; return *this;
    }
    // ColliderBuilder::solver_groups / active_collision_types (RbColliderFilter, applied by PhysicsPipeline after the upload)
    ColliderBuilder& solver_groups(unsigned memberships, unsigned filter, int test_mode = RB_TEST_AND) {
        f_.solver_memberships = memberships; f_.solver_filter = filter; f_.solver_test_mode = test_mode; return *this;
    }
    ColliderBuilder& active_collision_types(unsigned bits) { f_.active_collision_types = bits; return *this; }   // RB_ACT_*
    // The collider's filters; false when everything but the collision groups (which the descriptor carries) is the default.
    bool filter(RbColliderFilter& out) const {
        out = f_;
        out.collision_memberships = d_.collision_memberships; out.collision_filter = d_.collision_filter;
        return f_.collision_test_mode != RB_TEST_AND || f_.solver_memberships != 0xffffffffu || f_.solver_filter != 0xffffffffu ||
               f_.solver_test_mode != RB_TEST_AND || f_.active_collision_types != RB_ACT_DEFAULT;
    }
    ColliderBuilder& active_events(unsigned events) { d_.active_events = events; return *this; }   // RB_EVENT_*
    ColliderBuilder& contact_force_event_threshold(float t) { d_.contact_force_event_threshold = t; return *this; }
    ColliderBuilder& sensor(bool on = true) { d_.sensor = on ? 1 : 0; return *this; }   // ColliderBuilder::sensor
    RbColliderDesc desc(int parent) const { RbColliderDesc d = d_; d.parent = parent; return d; }

private:
    ColliderBuilder(int shape, float a, float b, float c) : d_{} {
        d_.shape = shape;
        d_.half_extents[0] = a; d_.half_extents[1] = b; d_.half_extents[2] = c;
        d_.parent = -1;
        d_.pos_wrt_parent_q[3] = 1.0f;
        d_.density = 1.0f; d_.friction = 0.5f; d_.restitution = 0.0f;           // collider.rs:688-707
        d_.friction_combine_rule = RB_COMBINE_AVERAGE; d_.restitution_combine_rule = RB_COMBINE_AVERAGE;
        d_.collision_memberships = 0xffffffffu; d_.collision_filter = 0xffffffffu;
        f_ = RbColliderFilter{0xffffffffu, 0xffffffffu, RB_TEST_AND, 0xffffffffu, 0xffffffffu, RB_TEST_AND, RB_ACT_DEFAULT};
    }
    RbColliderDesc d_;
    RbColliderFilter f_;
};

// GenericJoint / GenericJointBuilder (src/dynamics/joint/generic_joint.rs): locked axes, limits and motors on the free
// ones.  `axis` arguments are JointAxis indices 0..5 (LinX LinY LinZ AngX AngY AngZ).
class GenericJointBuilder {
public:
    explicit GenericJointBuilder(unsigned locked_axes) : d_{} {
        d_.local_frame1_q[3] = 1.0f; d_.local_frame2_q[3] = 1.0f;
        d_.locked_axes = locked_axes; d_.contacts_enabled = 1;
        d_.natural_frequency = 1.0e6f; d_.damping_ratio = 1.0f;                 // integration_parameters.rs:78-83
        for (int ax = 0; ax < 6; ++ax) {
            d_.limits[ax][0] = -FLT_MAX; d_.limits[ax][1] = FLT_MAX;            // JointLimits::default
            d_.motors[ax].max_force = FLT_MAX;                                  // JointMotor::default
        }
    }
    GenericJointBuilder& local_anchor1(Vector v) { for (int i = 0; i < 3; ++i) d_.local_frame1_t[i] = v[i]; return *this; }
    GenericJointBuilder& local_anchor2(Vector v) { for (int i = 0; i < 3; ++i) d_.local_frame2_t[i] = v[i]; return *this; }
    // GenericJoint::set_local_axis{1,2}: the joint's X axis in the body's frame (generic_joint.rs:374-389)
    GenericJointBuilder& local_axis1(Vector axis) { arc_from_x(axis, d_.local_frame1_q); return *this; }
    GenericJointBuilder& local_axis2(Vector axis) { arc_from_x(axis, d_.local_frame2_q); return *this; }
    GenericJointBuilder& contacts_enabled(bool on) { d_.contacts_enabled = on ? 1 : 0; return *this; }
    // generic_joint.rs:470-560
    GenericJointBuilder& limits(int axis, float lo, float hi) {
        d_.limit_axes |= 1u << axis; d_.limits[axis][0] = lo; d_.limits[axis][1] = hi; return *this;
    }
    GenericJointBuilder& motor(int axis, float target_pos, float target_vel, float stiffness, float damping) {
        d_.motor_axes |= 1u << axis;
        RbJointMotor& m = d_.motors[axis];
        m.target_pos = target_pos; m.target_vel = target_vel; m.stiffness = stiffness; m.damping = damping;
        return *this;
    }
    GenericJointBuilder& motor_velocity(int axis, float target_vel, float factor) { return motor(axis, 0.0f, target_vel, 0.0f, factor); }
    GenericJointBuilder& motor_position(int axis, float target_pos, float stiffness, float damping) {
        return motor(axis, target_pos, 0.0f, stiffness, damping);
    }
    GenericJointBuilder& motor_max_force(int axis, float max_force) { d_.motor_axes |= 1u << axis; d_.motors[axis].max_force = max_force; return *this; }
    GenericJointBuilder& motor_model(int axis, int model) { d_.motor_axes |= 1u << axis; d_.motors[axis].model = model; return *this; }   // 0 acceleration-, 1 force-based
    GenericJointBuilder& coupled_axes(unsigned mask) { d_.coupled_axes = mask & 63u; return *this; }   // GenericJointBuilder::coupled_axes
    RbJointDesc desc(int b1, int b2) const { RbJointDesc d = d_; d.body1 = b1; d.body2 = b2; return d; }

private:
    // minimal rotation taking +X to `axis`, written as (x, y, z, w)
    static void arc_from_x(Vector axis, float q[4]) {
        const float n = std::sqrt(axis[0] * axis[0] + axis[1] * axis[1] + axis[2] * axis[2]);
        const float ax = axis[0] / n, ay = axis[1] / n, az = axis[2] / n;
        if (ax > 1.0f - 1e-7f) { q[0] = q[1] = q[2] = 0.0f; q[3] = 1.0f; return; }
        if (ax < -1.0f + 1e-7f) { q[0] = q[1] = 0.0f; q[2] = 1.0f; q[3] = 0.0f; return; }   // half turn about Z
        const float s = std::sqrt((1.0f + ax) * 2.0f);
        q[0] = 0.0f; q[1] = -az / s; q[2] = ay / s; q[3] = s * 0.5f;
    }
    RbJointDesc d_;
};
// SphericalJointBuilder / FixedJointBuilder / RevoluteJointBuilder / PrismaticJointBuilder (src/dynamics/joint/*.rs)
struct SphericalJointBuilder : GenericJointBuilder { SphericalJointBuilder() : GenericJointBuilder(0x07u) {} };
struct FixedJointBuilder : GenericJointBuilder { FixedJointBuilder() : GenericJointBuilder(0x3fu) {} };
struct SpringJointBuilder : GenericJointBuilder {      // spring_joint.rs:32-38: LIN_AXES coupled, force-based position motor on the distance
    SpringJointBuilder(float rest_length, float stiffness, float damping) : GenericJointBuilder(0u) {
        coupled_axes(0x07u); motor_position(0, rest_length, stiffness, damping); motor_model(0, 1);
    }
};
struct RopeJointBuilder : GenericJointBuilder {        // rope_joint.rs:32-38, :153-156: LIN_AXES coupled, distance <= max_dist
    explicit RopeJointBuilder(float max_dist) : GenericJointBuilder(0u) { coupled_axes(0x07u); limits(0, 0.0f, max_dist); }
};
struct RevoluteJointBuilder : GenericJointBuilder {   // free: the rotation about `axis` (the X axis of both joint frames)
    explicit RevoluteJointBuilder(Vector axis) : GenericJointBuilder(0x37u) { local_axis1(axis); local_axis2(axis); }
};
struct PrismaticJointBuilder : GenericJointBuilder {  // free: the translation along `axis`
    explicit PrismaticJointBuilder(Vector axis) : GenericJointBuilder(0x3eu) { local_axis1(axis); local_axis2(axis); }
};

struct RigidBodySet {
    std::vector<RbBodyDesc> bodies;
    bool modified = true;
    RigidBodyHandle insert(const RigidBodyBuilder& b) { bodies.push_back(b.desc()); modified = true; return {int(bodies.size()) - 1}; }
    size_t len() const { return bodies.size(); }
};
struct ColliderSet {
    std::vector<RbColliderDesc> colliders;
    std::vector<int32_t> filtered;              // colliders whose filters are not the defaults ...
    std::vector<RbColliderFilter> filters;      // ... and those filters
    bool modified = true;
    ColliderHandle insert(const ColliderBuilder& c) { return add(c, -1); }
    ColliderHandle insert_with_parent(const ColliderBuilder& c, RigidBodyHandle parent, RigidBodySet&) { return add(c, parent.index); }
    ColliderHandle add(const ColliderBuilder& c, int parent) {
        colliders.push_back(c.desc(parent));
        RbColliderFilter f;
        if (c.filter(f)) { filtered.push_back(int(colliders.size()) - 1); filters.push_back(f); }
        modified = true;
        return {int(colliders.size()) - 1};
    }
    size_t len() const { return colliders.size(); }
};
struct ImpulseJointSet {
    std::vector<RbJointDesc> joints;
    bool modified = true;
    ImpulseJointHandle insert(RigidBodyHandle b1, RigidBodyHandle b2, const GenericJointBuilder& j, bool = true) {
        joints.push_back(j.desc(b1.index, b2.index)); modified = true; return {int(joints.size()) - 1};
    }
};

// PhysicsPipeline: owns the device-resident mirror (the reference's pipeline owns only scratch memory).
class PhysicsPipeline {
public:
    explicit PhysicsPipeline(int device = 0) : device_(device) {}
    ~PhysicsPipeline() { if (w_) rb_world_destroy(w_); }
    PhysicsPipeline(const PhysicsPipeline&) = delete;
    PhysicsPipeline& operator=(const PhysicsPipeline&) = delete;

    // PhysicsPipeline::step(gravity, &integration_parameters, ..., &mut bodies, &mut colliders, &mut impulse_joints, ...)
    void step(const Vector& gravity, const IntegrationParameters& params, RigidBodySet& bodies, ColliderSet& colliders,
              ImpulseJointSet& joints, int nsteps = 1, bool sync = true) {
        if (!w_) {
            w_ = rb_world_create(&params, device_);
            if (!w_) throw Error(RB_ERR_NO_DEVICE, rb_last_error());
        } else {
            check(rb_world_set_params(w_, &params));
        }
        if (bodies.modified || colliders.modified || joints.modified) {   // handle_user_changes (substep.rs:303-334)
            check(rb_world_set_scene(w_, int(bodies.bodies.size()), bodies.bodies.data(), int(colliders.colliders.size()),
                                     colliders.colliders.data(), int(joints.joints.size()), joints.joints.data()));
            if (!colliders.filtered.empty())
                check(rb_world_set_collider_filters(w_, int(colliders.filtered.size()), colliders.filtered.data(), colliders.filters.data()));
            bodies.modified = colliders.modified = joints.modified = false;
        }
        check(rb_world_step(w_, gravity.data(), nsteps, sync ? 1 : 0));
    }
    // Writes poses / velocities back into the caller's set (worker.rs:809-897 + substep.rs:84-224 on the CPU).
    void writeback(RigidBodySet& bodies) {
        size_t n = bodies.bodies.size();
        std::vector<float> pose(n * 7), vel(n * 6);
        check(rb_world_get_body_states(w_, pose.data(), vel.data()));
        for (size_t i = 0; i < n; ++i) {
            RbBodyDesc& d = bodies.bodies[i];
            for (int k = 0; k < 3; ++k) { d.translation[k] = pose[i * 7 + k]; d.linvel[k] = vel[i * 6 + k]; d.angvel[k] = vel[i * 6 + 3 + k]; }
            for (int k = 0; k < 4; ++k) d.rotation[k] = pose[i * 7 + 3 + k];
        }
    }
    RbCounters counters() { RbCounters c; check(rb_world_get_counters(w_, &c)); return c; }
    RbWorld* raw() { return w_; }

private:
    RbWorld* w_ = nullptr;
    int device_;
};

// PhysicsWorld facade (src/pipeline/physics_world.rs).
class PhysicsWorld {
public:
    Vector gravity{0.0f, -9.81f, 0.0f};
    IntegrationParameters integration_parameters;
    RigidBodySet bodies;
    ColliderSet colliders;
    ImpulseJointSet impulse_joints;
    PhysicsPipeline physics_pipeline;

    RigidBodyHandle insert(const RigidBodyBuilder& b, const ColliderBuilder& c) {
        RigidBodyHandle h = bodies.insert(b);
        colliders.insert_with_parent(c, h, bodies);
        return h;
    }
    void step(int n = 1) {
        physics_pipeline.step(gravity, integration_parameters, bodies, colliders, impulse_joints, n, true);
        physics_pipeline.writeback(bodies);
    }
};

}  // namespace rapier_b200
