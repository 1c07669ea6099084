/* rapier_b200.h -- C ABI of librapier_b200.so, the H100-native (sm_90a) replacement for the per-step
 * hot path of dimforge/rapier 0.35.2 (3-D, f32).
 *
 * The reference has no FFI layer for this path: the seam is the Rust method
 *   PhysicsPipeline::step(gravity, &IntegrationParameters, &mut IslandManager, &mut BroadPhaseBvh,
 *                         &mut NarrowPhase, &mut RigidBodySet, &mut ColliderSet, &mut ImpulseJointSet,
 *                         &mut MultibodyJointSet, &mut CCDSolver, &dyn PhysicsHooks, &dyn EventHandler)
 *   (src/pipeline/physics_pipeline/mod.rs:196-247; reached through PhysicsWorld::step,
 *    src/pipeline/physics_world.rs:120-156).
 * A Rust shim replacing `step_inner` (src/pipeline/physics_pipeline/substep.rs:267-581) binds the
 * entry points below with `extern "C"` (see INTEGRATION.md).  All pointers are caller-owned host
 * memory; the library copies.  One RbWorld is not re-entrant (the reference takes `&mut self`).
 * Every function returns RB_OK (0) or a negative RbStatus; rb_last_error() describes the failure.
 * The calls that edit the sets -- rb_world_set_body_states, rb_world_set_body_forces, rb_world_set_next_kinematic_positions,
 * rb_world_wake_up, rb_world_insert, rb_world_remove_bodies, rb_world_insert_joints, rb_world_remove_joints and
 * rb_world_update_joints -- check all of their input before they change anything: a call that returns RB_ERR_INVALID
 * has applied none of its entries and woken no body.
 * There is NO CPU fallback: without a CUDA device rb_world_create fails with RB_ERR_NO_DEVICE.
 */
#ifndef RAPIER_B200_H
#define RAPIER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB_ABI_VERSION 6

typedef struct RbWorld RbWorld;

typedef enum RbStatus {
    RB_OK = 0,
    RB_ERR_NO_DEVICE = -1,   /* no CUDA device / driver: the product path never falls back to CPU */
    RB_ERR_CUDA = -2,        /* a CUDA runtime call or kernel failed */
    RB_ERR_INVALID = -3,     /* bad argument (null pointer, index out of range, unsupported shape) */
    RB_ERR_CAPACITY = -4,    /* a device-side table overflowed (pairs, islands); state is unchanged */
    RB_ERR_NONFINITE = -5, RB_ERR_SHARD = -6    /* a body went non-finite (reference: Quarantine, quarantine.rs:14-47) */
} RbStatus;

/* Mirror of IntegrationParameters (src/dynamics/integration_parameters.rs:181-304), #[repr(C)]. */
typedef struct RbIntegrationParameters {
    float dt;                                   /* :185  default 1/60 */
    float min_ccd_dt;                           /*       default 1/60/100 (only read by the multi-substep CCD splitter, which is not supported) */
    float contact_natural_frequency;            /* contact_softness.natural_frequency, default 30 */
    float contact_damping_ratio;                /* contact_softness.damping_ratio,     default 10 */
    float static_contact_natural_frequency;     /* static_contact_softness, default 60 */
    float static_contact_damping_ratio;         /*                          default 10 */
    float warmstart_coefficient;                /* default 1 */
    float length_unit;                          /* default 1 */
    float normalized_allowed_linear_error;      /* default 0.005 */
    float normalized_max_corrective_velocity;   /* default 3 */
    float normalized_prediction_distance;       /* default 0.02 */
    float normalized_max_linear_velocity;       /* default 400 */
    int32_t num_solver_iterations;              /* substeps, default 4 */
    int32_t num_internal_pgs_iterations;        /* default 1 */
    int32_t num_internal_stabilization_iterations; /* default 1 */
    int32_t max_ccd_substeps;                   /* default 1: CCD motion clamping of fast bodies vs fixed colliders; 0 = off; > 1: RB_ERR_INVALID */
    int32_t contact_clustering;                 /* default 1 (no effect: single-manifold pairs only) */
    int32_t contact_recycling;                  /* default 1 */
    float normalized_contact_recycle_distance;  /* default 0.05 */
    int32_t friction_in_bias_pass;              /* default 0 */
    int32_t warmstart_joints;                   /* default 0; 1: joint rows are seeded with last step's impulses (joint_constraint_builder.rs:116-150) */
    int32_t friction_model;                     /* 0 = Simplified (twist, default); 1 = Coulomb (one friction part per point) */
} RbIntegrationParameters;

/* Fills *p with IntegrationParameters::default() (integration_parameters.rs:379-407). */
void rb_integration_parameters_default(RbIntegrationParameters* p);

/* RigidBodyType (src/dynamics/rigid_body_components.rs:20-46). */
enum { RB_BODY_DYNAMIC = 0, RB_BODY_FIXED = 1, RB_BODY_KINEMATIC_POSITION_BASED = 2, RB_BODY_KINEMATIC_VELOCITY_BASED = 3 };   /* RigidBodyType */

/* Body flags */
enum {
    RB_BODY_GYROSCOPIC = 1,          /* forces.gyroscopic_forces_enabled (default on, rigid_body.rs:1579) */
    RB_BODY_ALLOW_FAST_ROTATION = 2, /* ccd.allow_fast_rotation */
    RB_BODY_LOCK_TX = 4, RB_BODY_LOCK_TY = 8, RB_BODY_LOCK_TZ = 16,   /* LockedAxes */
    RB_BODY_LOCK_RX = 32, RB_BODY_LOCK_RY = 64, RB_BODY_LOCK_RZ = 128,
    RB_BODY_CCD_ENABLED = 512,       /* RigidBodyCcd::ccd_enabled: a "bullet" also sweeps against kinematic / dynamic bodies (never other bullets) */
    RB_BODY_NO_SLEEP = 256           /* RigidBodyActivation::cannot_sleep() (RigidBodyBuilder::can_sleep(false)); default: may sleep */
};
/* RigidBodyDominance (rigid_body_components.rs:1255-1276): a signed 8-bit group carried in bits 16..23 of `flags`
 * (default 0).  In a contact between bodies of different groups the body of the HIGHER group is seen as world-attached
 * (infinite mass, zero velocity: contact_with_twist_friction.rs:71-84); fixed bodies dominate every group. */
#define RB_BODY_DOMINANCE_SHIFT 16
#define RB_BODY_DOMINANCE(group) (((uint32_t)(uint8_t)(int8_t)(group)) << RB_BODY_DOMINANCE_SHIFT)
#define RB_BODY_DOMINANCE_OF(flags) ((int)(int8_t)(uint8_t)(((flags) >> RB_BODY_DOMINANCE_SHIFT) & 0xffu))
/* RigidBody::additional_solver_iterations (rigid_body.rs; island_manager/substep_groups.rs): 0..255 in bits 24..31 of
 * `flags` (default 0; ABI 5).  The body's whole connected component of awake dynamic bodies (touching contacts + joints)
 * runs num_solver_iterations + max-over-members substeps of dt / that count; other components keep the base cadence. */
#define RB_BODY_EXTRA_ITERS_SHIFT 24
#define RB_BODY_EXTRA_ITERS(n) (((uint32_t)(n) & 0xffu) << RB_BODY_EXTRA_ITERS_SHIFT)
#define RB_BODY_EXTRA_ITERS_OF(flags) ((int)(((flags) >> RB_BODY_EXTRA_ITERS_SHIFT) & 0xffu))

/* One rigid body as the caller's RigidBodySet holds it (src/dynamics/rigid_body.rs:48-70).
 * Mass properties are recomputed by the library from the attached colliders
 * (RigidBodyMassProps::recompute_mass_properties_from_colliders, rigid_body_components.rs:421)
 * plus `additional_mass`; pose quaternions are (x, y, z, w). */
typedef struct RbBodyDesc {
    int32_t body_type;            /* RB_BODY_* */
    uint32_t flags;               /* RB_BODY_GYROSCOPIC | ... */
    float translation[3];
    float rotation[4];
    float linvel[3];
    float angvel[3];
    float linear_damping;
    float angular_damping;
    float gravity_scale;
    float additional_mass;        /* RigidBodyAdditionalMassProps::Mass: added to the colliders' mass, angular inertia rescaled
                                   * (derived from the shape at unit density when the colliders are massless); 0 = none */
    float user_force[3];
    float user_torque[3];
} RbBodyDesc;

enum { RB_SHAPE_BALL = 0, RB_SHAPE_CUBOID = 1, RB_SHAPE_CAPSULE = 2, RB_SHAPE_CONVEX = 3 };

/* CoefficientCombineRule (src/dynamics/coefficient_combine_rule.rs:8-22). */
enum { RB_COMBINE_AVERAGE = 0, RB_COMBINE_MIN = 1, RB_COMBINE_MULTIPLY = 2, RB_COMBINE_MAX = 3,
       RB_COMBINE_CLAMPED_SUM = 4, RB_COMBINE_GEOMETRIC_MEAN = 5 };

/* One collider (src/geometry/collider.rs; ColliderBuilder defaults :688-707). */
typedef struct RbColliderDesc {
    int32_t shape;                /* RB_SHAPE_* */
    float half_extents[3];        /* cuboid half extents; ball: [radius, 0, 0]; capsule: [half height, radius, axis 0 | 1 | 2];
                                   * convex polyhedron: [hull id of rb_world_add_hull, border radius (round_convex_hull), 0] */
    int32_t parent;               /* body index, or -1 for a parentless (fixed) collider */
    float pos_wrt_parent_t[3];    /* pose relative to the parent (world pose if parent == -1) */
    float pos_wrt_parent_q[4];
    float density;                /* default 1 */
    float friction;               /* default 0.5 */
    float restitution;            /* default 0 */
    int32_t friction_combine_rule;     /* RB_COMBINE_* */
    int32_t restitution_combine_rule;
    float contact_skin;           /* default 0 */
    uint32_t collision_memberships;    /* InteractionGroups::all() = 0xffffffff */
    uint32_t collision_filter;
    uint32_t active_events;            /* RB_EVENT_* (ActiveEvents, collider.rs); default 0 */
    float contact_force_event_threshold;   /* default 0; only read with RB_EVENT_CONTACT_FORCE */
    int32_t sensor;                    /* ColliderBuilder::sensor (collider.rs; ABI 6): a sensor takes no part in contacts -- its pairs
                                        * are tested for intersection only (narrow_phase/intersections.rs) and report CollisionEvents
                                        * carrying RB_COLLISION_EVENT_SENSOR; it still counts for the mass of its body.  Default 0. */
} RbColliderDesc;

/* ActiveEvents (src/pipeline/event_handler.rs). */
enum { RB_EVENT_COLLISION = 1, RB_EVENT_CONTACT_FORCE = 2 };

/* CollisionEvent::{Started, Stopped} (src/geometry/mod.rs; emitted by apply_pair_transitions, narrow_phase/contacts.rs:312-324,
 * and when a touching pair leaves the broad phase).  `step` = index of the step that emitted it (1 = first step). */
enum { RB_COLLISION_EVENT_SENSOR = 1 };   /* CollisionEventFlags::SENSOR: at least one of the two colliders is a sensor */
typedef struct RbCollisionEvent { int32_t collider1, collider2, started, step, flags; } RbCollisionEvent;
/* ContactForceEvent (src/geometry/mod.rs:191-258; NarrowPhase::emit_contact_force_events, solver_graph.rs:462-498). */
typedef struct RbContactForceEvent {
    int32_t collider1, collider2;
    float total_force[3];
    float total_force_magnitude;
    float max_force_direction[3];
    float max_force_magnitude;
    int32_t started;               /* first step above the pair's threshold (coming from below or from separation) */
    int32_t step;
} RbContactForceEvent;

/* JointAxesMask bits (src/dynamics/joint/generic_joint.rs): LIN_X=1, LIN_Y=2, LIN_Z=4,
 * ANG_X=8, ANG_Y=16, ANG_Z=32 (spherical = 7 locked, fixed = 63, revolute about x = 55, prismatic along x = 62).
 * Free axes may carry limits (JointLimits, generic_joint.rs:142-160) and motors (JointMotor, :203-232); coupled
 * axes are not supported. */
typedef struct RbJointMotor {
    float target_vel, target_pos, stiffness, damping;
    float max_force;              /* default FLT_MAX */
    int32_t model;                /* 0 = AccelerationBased (default), 1 = ForceBased (motor_model.rs) */
} RbJointMotor;
typedef struct RbJointDesc {
    int32_t body1, body2;
    float local_frame1_t[3], local_frame1_q[4];
    float local_frame2_t[3], local_frame2_q[4];
    uint32_t locked_axes;
    int32_t contacts_enabled;     /* default 1 */
    float natural_frequency;      /* joint softness, default 1e6 (integration_parameters.rs:78-83) */
    float damping_ratio;          /* default 1 */
    uint32_t limit_axes;          /* JointAxesMask of the limited free axes */
    uint32_t motor_axes;          /* JointAxesMask of the motorised free axes */
    float limits[6][2];           /* [axis] min, max (distance along a linear axis, angle about an angular one) */
    RbJointMotor motors[6];
    uint32_t coupled_axes;        /* JointAxesMask of the coupled axes (GenericJoint::coupled_axes; ABI 5).  Coupled LINEAR axes share one
                                   * row on the DISTANCE between the anchors, driven by the limit (max only) and the motor of the first
                                   * coupled axis -- SpringJoint / RopeJoint (spring_joint.rs:32-38, rope_joint.rs:32-38).  Exactly two
                                   * coupled ANGULAR axes share one limit row on the angle between the third axes of the two frames; their
                                   * motors produce no row, as in the reference (joint_velocity_constraint.rs:224-226).  Default 0. */
} RbJointDesc;

/* Per-stage device times of the last step, named after the reference's Counters
 * (src/counters/mod.rs:19-35).  Milliseconds, measured with CUDA events when enabled. */
typedef struct RbCounters {
    float step_ms;
    float collision_detection_ms;   /* broad + narrow */
    float broad_phase_ms;
    float narrow_phase_ms;
    float island_construction_ms;   /* colouring + islands + schedule */
    float solver_ms;                /* velocity assembly + resolution + writeback */
    float update_ms;                /* advance_to_final_positions + AABB refresh */
    int32_t num_bodies, num_colliders, num_pairs, num_active_manifolds, num_islands, num_colors;
    int32_t num_joints;
    int32_t broad_phase_ran;        /* 1 if the pair set was recomputed in the last step */
    int32_t schedule_rebuilt;       /* 1 if colours/islands/schedule were rebuilt in the last step */
    int64_t kernels_launched;       /* cumulative count of this library's kernel launches */
    int64_t steps;                  /* cumulative steps */
} RbCounters;

/* ---- lifetime ---- */
int rb_abi_version(void);
const char* rb_last_error(void);
/* `device`: CUDA ordinal.  Fails (NULL, rb_last_error set) when no device is usable. */
RbWorld* rb_world_create(const RbIntegrationParameters* params, int device);
void rb_world_destroy(RbWorld* w);
int rb_world_set_params(RbWorld* w, const RbIntegrationParameters* params);

/* ---- state upload: RigidBodySet / ColliderSet / ImpulseJointSet (user changes, substep.rs:303-334) ----
 * rb_world_set_scene replaces the whole scene (and clears pairs, contacts, warm-start state). */
int rb_world_set_scene(RbWorld* w,
                       int32_t num_bodies, const RbBodyDesc* bodies,
                       int32_t num_colliders, const RbColliderDesc* colliders,
                       int32_t num_joints, const RbJointDesc* joints);
/* Overwrite poses/velocities of `n` bodies (indices[n]; pose7 = t(3) q(4); vel6 = lin(3) ang(3)). */
int rb_world_set_body_states(RbWorld* w, int32_t n, const int32_t* indices,
                             const float* pose7, const float* vel6);

/* ---- the hot path: PhysicsPipeline::step ---- */
/* Runs `nsteps` steps; host-synchronous on return only if `sync` != 0. */
int rb_world_step(RbWorld* w, const float gravity[3], int32_t nsteps, int32_t sync);
int rb_world_synchronize(RbWorld* w);

/* ---- state download (RigidBodySet writeback) ---- */
/* pose7 [n*7] and vel6 [n*6] may each be NULL. Synchronises the stream. */
int rb_world_get_body_states(RbWorld* w, float* pose7, float* vel6);
int rb_world_num_bodies(RbWorld* w);
int rb_world_get_counters(RbWorld* w, RbCounters* out);

/* ---- events (EventHandler, src/pipeline/event_handler.rs).  The reference calls the handler during the step; here the
 * step appends to device buffers (only for colliders with the matching RB_EVENT_* bit) that these calls drain: they
 * synchronise, copy out up to `cap` events ordered by (step, collider1, collider2), and empty the buffer.  Return
 * value: the number of events that were buffered (may exceed cap), or a negative status. */
int rb_world_drain_collision_events(RbWorld* w, int32_t cap, RbCollisionEvent* out);
int rb_world_drain_contact_force_events(RbWorld* w, int32_t cap, RbContactForceEvent* out);
/* RigidBody::reset_forces + add_force / add_torque between steps: replaces the user force / torque of the listed bodies
 * (either array may be NULL). */
int rb_world_set_body_forces(RbWorld* w, int32_t n, const int32_t* indices, const float* force3, const float* torque3);
/* RigidBody::set_next_kinematic_position (rigid_body.rs:1085-1090) of position-based kinematic bodies: the pose they
 * reach at the end of the next step; their velocity during that step is interpolated from it.  Other bodies: RB_ERR_INVALID. */
int rb_world_set_next_kinematic_positions(RbWorld* w, int32_t n, const int32_t* indices, const float* pose7);
int rb_world_enable_profiling(RbWorld* w, int32_t enabled);

/* ---- contact graph read-back (NarrowPhase::contact_pairs; used by the parity tests) ---- */
/* Returns the number of broad-phase pairs; fills up to `cap` entries of each non-NULL array.
 *   pair_colliders [cap*2]   collider1, collider2 (collider1 < collider2)
 *   num_contacts   [cap]     active solver contacts of the pair's manifold (0..4)
 *   color          [cap]     solver colour (0..127, 128 overflow, 255 uncoloured)
 *   normal         [cap*3]   world-space manifold normal (ContactManifoldData::normal)
 *   impulses       [cap*4]   total normal impulse of each solver contact (ContactData::impulse) */
int rb_world_get_contact_pairs(RbWorld* w, int32_t cap, int32_t* pair_colliders, int32_t* num_contacts,
                               int32_t* color, float* normal, float* impulses);
/* Raw device-table dump for debugging / parity (name-addressed; see DESIGN.md "debug tables").
 * Returns bytes copied or a negative status. */
int64_t rb_world_debug_read(RbWorld* w, const char* table, void* dst, int64_t cap_bytes);

/* ---- incremental changes of the sets (src/pipeline/user_changes.rs:11-46; substep.rs:303-334) ----
 * rb_world_set_scene replaces the whole world and forgets every contact; these keep it.
 * rb_world_reserve: room for later insertions, applied by the NEXT rb_world_set_scene.
 * rb_world_insert: appends bodies and colliders (RigidBodySet::insert, ColliderSet::insert_with_parent); existing
 *   indices, contact pairs, warm-start impulses, colours and islands are untouched.  collider.parent is the FINAL body
 *   index; new colliders may only be attached to the new bodies (or have no parent).  Returns the first new indices.
 * rb_world_remove_bodies: RigidBodySet::remove(handle, .., remove_attached_colliders = true); slots stay allocated
 *   (tombstones), the colliders leave the broad phase and their contact pairs end at the next step. */
int rb_world_reserve(RbWorld* w, int32_t max_bodies, int32_t max_colliders);
int rb_world_insert(RbWorld* w, int32_t num_bodies, const RbBodyDesc* bodies, int32_t num_colliders,
                    const RbColliderDesc* colliders, int32_t* first_body_index, int32_t* first_collider_index);
int rb_world_remove_bodies(RbWorld* w, int32_t n, const int32_t* body_indices);
/* ImpulseJointSet::insert / remove after the upload (src/dynamics/joint/impulse_joint/impulse_joint_set.rs; ABI 6).
 * rb_world_reserve_joints: the TOTAL number of joint slots (scene + later insertions, like rb_world_reserve), applied by the NEXT
 * rb_world_set_scene; generic != 0 also reserves the
 * generic joint path (limits / motors / coupled axes / warmstart_joints) for a scene that has no such joint yet.
 * rb_world_insert_joints: appended joints keep every existing index; *first_joint receives the index of the first new one;
 * the islands of the attached bodies are woken (insert(.., wake_up = true)).
 * rb_world_remove_joints: the slots stay allocated; the joints are no longer solved, no longer island edges, and the
 * contacts they disabled come back.  Both recompute the joint colours and the stage order from the whole joint set. */
int rb_world_reserve_joints(RbWorld* w, int32_t max_joints, int32_t generic);
int rb_world_insert_joints(RbWorld* w, int32_t n, const RbJointDesc* joints, int32_t* first_joint);
int rb_world_remove_joints(RbWorld* w, int32_t n, const int32_t* joint_indices);
/* ImpulseJointSet::get_mut(handle, wake_up) + edits: the listed joints take the new descriptors in place (motor targets, limits,
 * frames, softness ...).  Bodies must stay the same; warm-start impulses are kept; wake_up != 0 wakes the attached bodies'
 * islands (crates/rapier3d/tests/issue_692_joint_get_mut_wakes_bodies.rs). */
int rb_world_update_joints(RbWorld* w, int32_t n, const int32_t* joint_indices, const RbJointDesc* joints, int32_t wake_up);

/* ---- convex polyhedra (ColliderBuilder::{convex_hull, convex_mesh, round_convex_hull}, src/geometry/collider.rs:1039-1090;
 *      parry ConvexPolyhedron) ----
 * rb_world_add_hull registers a closed convex mesh -- at most 32 vertices, 32 polygonal faces of 3..8 vertices (either
 * winding), 64 edges -- and returns the hull id (>= 1; hull 0 is the unit cube) that RB_SHAPE_CONVEX colliders carry in
 * half_extents[0]; half_extents[1] is the border radius of a "round" polyhedron (0 = sharp).  Planes, edges, volume,
 * centre of mass and principal inertia are derived here.  Hulls persist across rb_world_set_scene; ids are per world.
 * rb_convex_hull (host only, no world needed) computes the hull mesh of 4..32 points: buffers need room for 32 vertices
 * (96 floats), 32 face sizes and 256 face indices. */
int32_t rb_world_add_hull(RbWorld* w, int32_t num_vertices, const float* vertices3, int32_t num_faces,
                          const int32_t* face_sizes, const int32_t* face_indices);
int32_t rb_convex_hull(int32_t num_points, const float* points3, int32_t* num_vertices, float* vertices3,
                       int32_t* num_faces, int32_t* face_sizes, int32_t* face_indices);

/* ---- sleeping (src/dynamics/island_manager/sleep.rs, manager.rs:320-425; rigid_body_components.rs:1417-1470) ----
 * A connected component of touching contacts / joints falls asleep as a whole once EVERY body in it has moved less
 * than 0.05 length units / s for 0.5 s (and may sleep at all: RB_BODY_NO_SLEEP); it wakes as a whole when a contact
 * with one of its bodies begins, when one of its bodies is changed through rb_world_set_body_states / rb_world_wake_up,
 * or when a body is removed.  Sleeping bodies keep their contact pairs and warm-start data but are neither solved nor
 * integrated.  sleeping[num_bodies]: 1 = asleep. */
int rb_world_get_sleeping(RbWorld* w, uint8_t* sleeping);
/* Quarantine (src/pipeline/physics_pipeline/quarantine.rs:14-47): a body whose state goes non-finite during a step keeps
 * its last valid pose, loses its velocities and forces and is disabled like a removed body; the step reports
 * RB_ERR_NONFINITE at the next synchronising call.  Returns the number of bodies quarantined since the last call and
 * writes up to `cap` indices (ascending); the list is cleared by a call that reads it. */
int rb_world_get_quarantine(RbWorld* w, int32_t* bodies, int32_t cap);
int rb_world_wake_up(RbWorld* w, int32_t n, const int32_t* body_indices);

/* Unit-level known-answer evaluation for parity tests: runs ONE device function of the path (named: "pose_drift"
 * contact_pair.rs:299-323, "reduce_manifold" manifold_reduction.rs:4-84, "normal_solve" / "tangent_solve"
 * contact_constraint_element.rs:481-504 / :650-705, "generate" contact_with_twist_friction.rs:58-424) on literal
 * inputs and returns its outputs (float layouts: tests/golden/make_ref_vectors.py). Needs a CUDA device. */
int rb_debug_kat(const char* name, const float* in, int32_t n_in, float* out, int32_t n_out);

/* ---- multi-GPU sharding (SURVEY 8e): each rank owns whole connected components ---- */
/* Restricts this world to the bodies whose component id (as labelled by rb_world_label_components)
 * satisfies component % world_size == rank; the other dynamic bodies become inert. */
int rb_world_label_components(RbWorld* w, int32_t* component_of_body /* [num_bodies], host */);
int rb_world_set_owned_bodies(RbWorld* w, const uint8_t* owned /* [num_bodies]: 1 = simulated here, 0 = elsewhere; before the first step */);
/* Halo bodies: bodies of other ranks close enough to be tracked here (proximity detection only; a CONTACT with one
 * raises RB_ERR_SHARD: the islands of two shards merged).  flags_dev: DEVICE array [num_bodies], non-zero = track;
 * stream-ordered, keeps all contact state.  rb_world_import_halo copies their states out of the packed state table. */
int rb_world_set_halo_bodies(RbWorld* w, const uint8_t* flags_dev);
int rb_world_import_halo(RbWorld* w);
/* Device pointers to the packed per-body state (13 floats/body: t3 q4 lin3 ang3) for NCCL
 * all-gather of boundary body states, and the byte size. */
int rb_world_state_buffer(RbWorld* w, void** device_ptr, int64_t* bytes);

/* Scatter externally simulated body states (device pointers: idx[n], src[n*13]) into the world.
 * src_dev == NULL: the rows were all-gathered in place into rb_world_state_buffer; body idx[k] is
 * imported from its own row. */
int rb_world_import_states(RbWorld* w, const int32_t* idx_dev, const float* src_dev, int32_t n);
/* ... from a whole [num_bodies][13] state table (device pointer; typically one of the two buffers below). */
int rb_world_import_states_from(RbWorld* w, const int32_t* idx_dev, const float* table_dev, int32_t n);
/* Double-buffers the packed state: counted from this call, step k writes buffer (k & 1), so the buffer just
 * written can be all-gathered in place, asynchronously, under the next step.  rb_world_get_body_states and
 * rb_world_step_host keep reading / writing the most recent buffer. */
int rb_world_state_buffers(RbWorld* w, void** device_ptr0, void** device_ptr1, int64_t* bytes);
/* The CUDA stream all of this world's work is enqueued on / replace it by a caller-owned stream. */
void* rb_world_stream(RbWorld* w);
int rb_world_set_stream(RbWorld* w, void* cuda_stream);
/* One step with HOST state buffers (13 floats per body: t3 q4 linvel3 angvel3), copies included:
 * upload `in_state13` (may be NULL), step, download into `out_state13` (may be NULL). Synchronous. */
int rb_world_step_host(RbWorld* w, const float gravity[3], const float* in_state13, float* out_state13);

#ifdef __cplusplus
}
#endif
#endif /* RAPIER_B200_H */
