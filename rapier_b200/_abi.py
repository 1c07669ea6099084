"""ctypes mirror of include/rapier_b200.h (the C-ABI drop-in boundary).

Field order and types must match the header exactly; tests/test_abi.py checks sizeof() against the
values the shared library reports.
"""
import ctypes as C

RB_OK = 0
RB_ERR_NO_DEVICE = -1
RB_ERR_CUDA = -2
RB_ERR_INVALID = -3
RB_ERR_CAPACITY = -4
RB_ERR_NONFINITE = -5
RB_ERR_SHARD = -6

RB_BODY_DYNAMIC = 0
RB_BODY_FIXED = 1
RB_BODY_KINEMATIC_POSITION_BASED = 2
RB_BODY_KINEMATIC_VELOCITY_BASED = 3
RB_BODY_GYROSCOPIC = 1
RB_BODY_ALLOW_FAST_ROTATION = 2
RB_BODY_LOCK_TX, RB_BODY_LOCK_TY, RB_BODY_LOCK_TZ = 4, 8, 16
RB_BODY_LOCK_RX, RB_BODY_LOCK_RY, RB_BODY_LOCK_RZ = 32, 64, 128
RB_BODY_NO_SLEEP = 256
RB_BODY_CCD_ENABLED = 512
RB_BODY_DOMINANCE_SHIFT = 16   # RB_BODY_DOMINANCE(group): signed 8-bit dominance group in bits 16..23 of flags
RB_BODY_EXTRA_ITERS_SHIFT = 24  # RB_BODY_EXTRA_ITERS(n): additional_solver_iterations (0..255) in bits 24..31 of flags
RB_FAT_SKIN_FACTOR = 0.04     # RB_FAT_SKIN_FACTOR: fat-box skin in units of length_unit
RB_SHAPE_BALL = 0
RB_SHAPE_CUBOID = 1
RB_SHAPE_CAPSULE = 2
RB_SHAPE_CONVEX = 3
(RB_COMBINE_AVERAGE, RB_COMBINE_MIN, RB_COMBINE_MULTIPLY, RB_COMBINE_MAX, RB_COMBINE_CLAMPED_SUM,
 RB_COMBINE_GEOMETRIC_MEAN) = range(6)

f32, i32, u32 = C.c_float, C.c_int32, C.c_uint32


class RbIntegrationParameters(C.Structure):
    """IntegrationParameters (src/dynamics/integration_parameters.rs:181-304)."""
    _fields_ = [
        ("dt", f32), ("min_ccd_dt", f32),
        ("contact_natural_frequency", f32), ("contact_damping_ratio", f32),
        ("static_contact_natural_frequency", f32), ("static_contact_damping_ratio", f32),
        ("warmstart_coefficient", f32), ("length_unit", f32),
        ("normalized_allowed_linear_error", f32), ("normalized_max_corrective_velocity", f32),
        ("normalized_prediction_distance", f32), ("normalized_max_linear_velocity", f32),
        ("num_solver_iterations", i32), ("num_internal_pgs_iterations", i32),
        ("num_internal_stabilization_iterations", i32), ("max_ccd_substeps", i32),
        ("contact_clustering", i32), ("contact_recycling", i32),
        ("normalized_contact_recycle_distance", f32),
        ("friction_in_bias_pass", i32), ("warmstart_joints", i32), ("friction_model", i32),
    ]

    @classmethod
    def default(cls):
        """IntegrationParameters::default() (integration_parameters.rs:379-407)."""
        return cls(dt=1.0 / 60.0, min_ccd_dt=1.0 / 60.0 / 100.0,
                   contact_natural_frequency=30.0, contact_damping_ratio=10.0,
                   static_contact_natural_frequency=60.0, static_contact_damping_ratio=10.0,
                   warmstart_coefficient=1.0, length_unit=1.0,
                   normalized_allowed_linear_error=0.005, normalized_max_corrective_velocity=3.0,
                   normalized_prediction_distance=0.02, normalized_max_linear_velocity=400.0,
                   num_solver_iterations=4, num_internal_pgs_iterations=1,
                   num_internal_stabilization_iterations=1, max_ccd_substeps=1,
                   contact_clustering=1, contact_recycling=1,
                   normalized_contact_recycle_distance=0.05,
                   friction_in_bias_pass=0, warmstart_joints=0, friction_model=0)


class RbBodyDesc(C.Structure):
    _fields_ = [
        ("body_type", i32), ("flags", u32),
        ("translation", f32 * 3), ("rotation", f32 * 4),
        ("linvel", f32 * 3), ("angvel", f32 * 3),
        ("linear_damping", f32), ("angular_damping", f32), ("gravity_scale", f32),
        ("additional_mass", f32),
        ("user_force", f32 * 3), ("user_torque", f32 * 3),
    ]


class RbColliderDesc(C.Structure):
    _fields_ = [
        ("shape", i32), ("half_extents", f32 * 3), ("parent", i32),
        ("pos_wrt_parent_t", f32 * 3), ("pos_wrt_parent_q", f32 * 4),
        ("density", f32), ("friction", f32), ("restitution", f32),
        ("friction_combine_rule", i32), ("restitution_combine_rule", i32),
        ("contact_skin", f32),
        ("collision_memberships", u32), ("collision_filter", u32),
        ("active_events", u32), ("contact_force_event_threshold", f32), ("sensor", i32),
    ]


class RbCollisionEvent(C.Structure):
    _fields_ = [("collider1", i32), ("collider2", i32), ("started", i32), ("step", i32), ("flags", i32)]


class RbContactForceEvent(C.Structure):
    _fields_ = [("collider1", i32), ("collider2", i32), ("total_force", f32 * 3), ("total_force_magnitude", f32),
                ("max_force_direction", f32 * 3), ("max_force_magnitude", f32), ("started", i32), ("step", i32)]


RB_EVENT_COLLISION, RB_EVENT_CONTACT_FORCE = 1, 2
RB_COLLISION_EVENT_SENSOR = 1   # CollisionEventFlags::SENSOR

# ActiveCollisionTypes (collider_components.rs:282-345) and InteractionTestMode (interaction_groups.rs:74-154)
RB_ACT_DYNAMIC_DYNAMIC = 0x0001
RB_ACT_DYNAMIC_KINEMATIC = 0x000C
RB_ACT_DYNAMIC_FIXED = 0x0002
RB_ACT_KINEMATIC_KINEMATIC = 0xCC00
RB_ACT_KINEMATIC_FIXED = 0x2200
RB_ACT_FIXED_FIXED = 0x0020
RB_ACT_DEFAULT = 0x000F
RB_TEST_AND, RB_TEST_OR = 0, 1


class RbColliderFilter(C.Structure):
    """The filters of one collider (ColliderFlags, collider_components.rs:363-379)."""
    _fields_ = [
        ("collision_memberships", u32), ("collision_filter", u32), ("collision_test_mode", i32),
        ("solver_memberships", u32), ("solver_filter", u32), ("solver_test_mode", i32),
        ("active_collision_types", u32),
    ]


class RbJointMotor(C.Structure):
    _fields_ = [("target_vel", f32), ("target_pos", f32), ("stiffness", f32), ("damping", f32), ("max_force", f32), ("model", i32)]


class RbJointDesc(C.Structure):
    _fields_ = [
        ("body1", i32), ("body2", i32),
        ("local_frame1_t", f32 * 3), ("local_frame1_q", f32 * 4),
        ("local_frame2_t", f32 * 3), ("local_frame2_q", f32 * 4),
        ("locked_axes", u32), ("contacts_enabled", i32),
        ("natural_frequency", f32), ("damping_ratio", f32),
        ("limit_axes", u32), ("motor_axes", u32), ("limits", (f32 * 2) * 6), ("motors", RbJointMotor * 6),
        ("coupled_axes", u32),
    ]


class RbCounters(C.Structure):
    _fields_ = [
        ("step_ms", f32), ("collision_detection_ms", f32), ("broad_phase_ms", f32),
        ("narrow_phase_ms", f32), ("island_construction_ms", f32), ("solver_ms", f32),
        ("update_ms", f32),
        ("num_bodies", i32), ("num_colliders", i32), ("num_pairs", i32),
        ("num_active_manifolds", i32), ("num_islands", i32), ("num_colors", i32),
        ("num_joints", i32), ("broad_phase_ran", i32), ("schedule_rebuilt", i32),
        ("kernels_launched", C.c_int64), ("steps", C.c_int64),
    ]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}
