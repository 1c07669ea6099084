"""Host-side mirror of the reference's state stores for the step hot path.

Mirrors (names, argument meaning, defaults) of:
  RigidBodyBuilder / RigidBodySet     src/dynamics/rigid_body.rs:1490-1580, rigid_body_set.rs:70-79, :150
  ColliderBuilder / ColliderSet       src/geometry/collider.rs:688-707, :1125-1131
  SphericalJointBuilder / FixedJointBuilder / ImpulseJointSet
                                      src/dynamics/joint/spherical_joint.rs, impulse_joint/impulse_joint_set.rs
Handles are plain indices (the reference's generational arena index without the generation,
src/data/arena.rs): removal is outside the hot path and not mirrored.  The sets serialise to the
C-ABI descriptor arrays of include/rapier_b200.h; nothing here computes physics.
"""
import ctypes as C
import math

import numpy as np

from . import _abi as A


class RigidBodyBuilder:
    def __init__(self, body_type):
        self.body_type = body_type
        self._translation = (0.0, 0.0, 0.0)
        self._rotation = (0.0, 0.0, 0.0, 1.0)
        self._linvel = (0.0, 0.0, 0.0)
        self._angvel = (0.0, 0.0, 0.0)
        self._linear_damping = 0.0
        self._angular_damping = 0.0
        self._gravity_scale = 1.0
        self._can_sleep = True
        self._flags = A.RB_BODY_GYROSCOPIC  # gyroscopic forces on by default (rigid_body.rs:1579)
        self._additional_mass = 0.0

    @classmethod
    def dynamic(cls):
        return cls(A.RB_BODY_DYNAMIC)

    @classmethod
    def fixed(cls):
        return cls(A.RB_BODY_FIXED)

    @classmethod
    def kinematic_position_based(cls):
        return cls(A.RB_BODY_KINEMATIC_POSITION_BASED)

    @classmethod
    def kinematic_velocity_based(cls):
        return cls(A.RB_BODY_KINEMATIC_VELOCITY_BASED)

    def translation(self, v):
        self._translation = tuple(float(x) for x in v)
        return self

    def rotation(self, axis_angle):
        """Scaled-axis rotation, as RigidBodyBuilder::rotation(AngVector)."""
        ax, ay, az = (float(x) for x in axis_angle)
        ang = math.sqrt(ax * ax + ay * ay + az * az)
        if ang == 0.0:
            self._rotation = (0.0, 0.0, 0.0, 1.0)
        else:
            s = math.sin(ang / 2.0) / ang
            self._rotation = (ax * s, ay * s, az * s, math.cos(ang / 2.0))
        return self

    def rotation_quat(self, q):
        self._rotation = tuple(float(x) for x in q)
        return self

    def linvel(self, v):
        self._linvel = tuple(float(x) for x in v)
        return self

    def angvel(self, v):
        self._angvel = tuple(float(x) for x in v)
        return self

    def additional_mass(self, m):
        """RigidBodyBuilder::additional_mass (RigidBodyAdditionalMassProps::Mass)."""
        self._additional_mass = float(m)
        return self

    def linear_damping(self, d):
        self._linear_damping = float(d)
        return self

    def angular_damping(self, d):
        self._angular_damping = float(d)
        return self

    def gravity_scale(self, s):
        self._gravity_scale = float(s)
        return self

    def ccd_enabled(self, flag):
        """RigidBodyBuilder::ccd_enabled: upgrade to a bullet (sweeps against moving bodies too)."""
        if flag:
            self._flags |= A.RB_BODY_CCD_ENABLED
        else:
            self._flags &= ~A.RB_BODY_CCD_ENABLED
        return self

    def dominance_group(self, group):
        """RigidBodyBuilder::dominance_group (rigid_body.rs): signed 8-bit group; in a contact the body of the higher group
        is seen as immovable by the other one (RigidBodyDominance, rigid_body_components.rs:1255-1276)."""
        g = int(group)
        if not -128 <= g <= 127:
            raise ValueError("dominance group must fit an i8")
        self._flags = (self._flags & ~(0xFF << A.RB_BODY_DOMINANCE_SHIFT)) | ((g & 0xFF) << A.RB_BODY_DOMINANCE_SHIFT)
        return self

    def additional_solver_iterations(self, n):
        """RigidBodyBuilder::additional_solver_iterations (rigid_body.rs): the body's whole connected component runs that many
        extra substeps at a smaller dt (island_manager/substep_groups.rs)."""
        n = int(n)
        if not 0 <= n <= 255:
            raise ValueError("additional_solver_iterations must be in 0..255")
        self._flags = (self._flags & ~(0xFF << A.RB_BODY_EXTRA_ITERS_SHIFT)) | (n << A.RB_BODY_EXTRA_ITERS_SHIFT)
        return self

    def can_sleep(self, flag):
        """RigidBodyBuilder::can_sleep (rigid_body.rs; false = RigidBodyActivation::cannot_sleep())."""
        self._can_sleep = bool(flag)
        if flag:
            self._flags &= ~A.RB_BODY_NO_SLEEP
        else:
            self._flags |= A.RB_BODY_NO_SLEEP
        return self

    def gyroscopic_forces_enabled(self, flag):
        if flag:
            self._flags |= A.RB_BODY_GYROSCOPIC
        else:
            self._flags &= ~A.RB_BODY_GYROSCOPIC
        return self

    def locked_axes(self, bits):
        self._flags |= int(bits) & 0xFC
        return self

    def lock_rotations(self):
        """RigidBodyBuilder::lock_rotations (LockedAxes::ROTATION_LOCKED)."""
        return self.locked_axes(A.RB_BODY_LOCK_RX | A.RB_BODY_LOCK_RY | A.RB_BODY_LOCK_RZ)

    def lock_translations(self):
        """RigidBodyBuilder::lock_translations (LockedAxes::TRANSLATION_LOCKED)."""
        return self.locked_axes(A.RB_BODY_LOCK_TX | A.RB_BODY_LOCK_TY | A.RB_BODY_LOCK_TZ)

    def build_desc(self):
        d = A.RbBodyDesc()
        d.body_type = self.body_type
        d.flags = self._flags
        d.translation[:] = self._translation
        d.rotation[:] = self._rotation
        d.linvel[:] = self._linvel
        d.angvel[:] = self._angvel
        d.linear_damping = self._linear_damping
        d.angular_damping = self._angular_damping
        d.gravity_scale = self._gravity_scale
        d.additional_mass = self._additional_mass
        return d


class ColliderBuilder:
    def __init__(self, shape, half_extents):
        self.shape = shape
        self.half_extents = half_extents
        self._density = 1.0
        self._friction = 0.5
        self._restitution = 0.0
        self._translation = (0.0, 0.0, 0.0)
        self._rotation = (0.0, 0.0, 0.0, 1.0)
        self._friction_rule = A.RB_COMBINE_AVERAGE
        self._restitution_rule = A.RB_COMBINE_AVERAGE
        self._contact_skin = 0.0
        self._memberships = 0xFFFFFFFF
        self._filter = 0xFFFFFFFF

    @classmethod
    def cuboid(cls, hx, hy, hz):
        return cls(A.RB_SHAPE_CUBOID, (float(hx), float(hy), float(hz)))

    @classmethod
    def ball(cls, radius):
        return cls(A.RB_SHAPE_BALL, (float(radius), 0.0, 0.0))

    @classmethod
    def capsule_x(cls, half_height, radius):
        return cls(A.RB_SHAPE_CAPSULE, (float(half_height), float(radius), 0.0))

    @classmethod
    def capsule_y(cls, half_height, radius):
        """ColliderBuilder::capsule_y (collider.rs): a segment of 2 * half_height along Y, inflated by `radius`."""
        return cls(A.RB_SHAPE_CAPSULE, (float(half_height), float(radius), 1.0))

    @classmethod
    def capsule_z(cls, half_height, radius):
        return cls(A.RB_SHAPE_CAPSULE, (float(half_height), float(radius), 2.0))

    @classmethod
    def convex_mesh(cls, points, faces, border_radius=0.0):
        """ColliderBuilder::convex_mesh / round_convex_mesh (collider.rs:1070-1090): a closed convex mesh given by its
        vertices and polygonal faces (vertex index loops, either winding).  The ColliderSet registers the polyhedron
        (rb_world_add_hull) when the collider is inserted."""
        b = cls(A.RB_SHAPE_CONVEX, (0.0, float(border_radius), 0.0))
        b._hull = (np.ascontiguousarray(points, np.float32).reshape(-1, 3), [[int(i) for i in f] for f in faces])
        return b

    @classmethod
    def convex_hull(cls, points, border_radius=0.0):
        """ColliderBuilder::convex_hull (collider.rs:1039-1044): the convex hull of at most 32 points."""
        verts, faces = convex_hull_mesh(points)
        return cls.convex_mesh(verts, faces, border_radius)

    @classmethod
    def round_convex_hull(cls, points, border_radius):
        """ColliderBuilder::round_convex_hull (collider.rs:1046-1060): the hull dilated by `border_radius`."""
        return cls.convex_hull(points, border_radius)

    def density(self, d):
        self._density = float(d)
        return self

    def mass(self, m):
        """ColliderBuilder::mass (ColliderMassProps::Mass): the density that gives the shape this mass."""
        import math
        hx, hy, hz = self.half_extents
        volume = 8.0 * hx * hy * hz if self.shape == A.RB_SHAPE_CUBOID else 4.0 / 3.0 * math.pi * hx ** 3
        if self.shape == A.RB_SHAPE_CAPSULE:
            volume = 2.0 * hx * math.pi * hy ** 2 + 4.0 / 3.0 * math.pi * hy ** 3
        self._density = float(m) / volume if volume > 0.0 else 0.0
        return self

    def rotation(self, axis_angle):
        """ColliderBuilder::rotation: orientation relative to the parent body, as a scaled axis."""
        import math
        ax = [float(x) for x in axis_angle]
        a = math.sqrt(sum(x * x for x in ax))
        if a == 0.0:
            self._rotation = (0.0, 0.0, 0.0, 1.0)
        else:
            k = math.sin(a / 2.0) / a
            self._rotation = (ax[0] * k, ax[1] * k, ax[2] * k, math.cos(a / 2.0))
        return self

    def friction(self, f):
        self._friction = float(f)
        return self

    def restitution(self, r):
        self._restitution = float(r)
        return self

    def friction_combine_rule(self, r):
        self._friction_rule = int(r)
        return self

    def restitution_combine_rule(self, r):
        self._restitution_rule = int(r)
        return self

    def translation(self, v):
        self._translation = tuple(float(x) for x in v)
        return self

    def contact_skin(self, s):
        self._contact_skin = float(s)
        return self

    def collision_groups(self, memberships, filter_, test_mode=A.RB_TEST_AND):
        """ColliderBuilder::collision_groups (InteractionGroups; test_mode: RB_TEST_AND or RB_TEST_OR)."""
        self._memberships = int(memberships)
        self._filter = int(filter_)
        self._collision_test_mode = int(test_mode)
        return self

    def solver_groups(self, memberships, filter_, test_mode=A.RB_TEST_AND):
        """ColliderBuilder::solver_groups: a pair whose solver groups fail keeps its contacts and events but gets no force."""
        self._solver_groups = (int(memberships), int(filter_), int(test_mode))
        return self

    def active_collision_types(self, bits):
        """ColliderBuilder::active_collision_types (RB_ACT_* bits; default RB_ACT_DEFAULT)."""
        self._active_collision_types = int(bits)
        return self

    def build_filter(self):
        """The collider's RbColliderFilter, or None when everything but the collision groups (which travel in the
        descriptor) keeps its default."""
        mode = getattr(self, "_collision_test_mode", A.RB_TEST_AND)
        solver = getattr(self, "_solver_groups", (0xFFFFFFFF, 0xFFFFFFFF, A.RB_TEST_AND))
        types = getattr(self, "_active_collision_types", A.RB_ACT_DEFAULT)
        if mode == A.RB_TEST_AND and solver == (0xFFFFFFFF, 0xFFFFFFFF, A.RB_TEST_AND) and types == A.RB_ACT_DEFAULT:
            return None
        return A.RbColliderFilter(self._memberships, self._filter, mode, *solver, types)

    def active_events(self, events):
        """ColliderBuilder::active_events (ActiveEvents: RB_EVENT_COLLISION | RB_EVENT_CONTACT_FORCE)."""
        self._active_events = int(events)
        return self

    def sensor(self, flag=True):
        """ColliderBuilder::sensor (collider.rs): intersection events only, no contacts."""
        self._sensor = bool(flag)
        return self

    def contact_force_event_threshold(self, threshold):
        self._force_threshold = float(threshold)
        return self

    def build_desc(self, parent):
        d = A.RbColliderDesc()
        d.shape = self.shape
        d.half_extents[:] = self.half_extents
        d.parent = -1 if parent is None else int(parent)
        d.pos_wrt_parent_t[:] = self._translation
        d.pos_wrt_parent_q[:] = self._rotation
        d.density = self._density
        d.friction = self._friction
        d.restitution = self._restitution
        d.friction_combine_rule = self._friction_rule
        d.restitution_combine_rule = self._restitution_rule
        d.contact_skin = self._contact_skin
        d.collision_memberships = self._memberships
        d.collision_filter = self._filter
        d.active_events = getattr(self, "_active_events", 0)
        d.contact_force_event_threshold = getattr(self, "_force_threshold", 0.0)
        d.sensor = 1 if getattr(self, "_sensor", False) else 0
        return d


class GenericJointBuilder:
    """GenericJoint: locked axes (spherical = LIN_X|LIN_Y|LIN_Z, fixed = all six), limits and motors on the free ones."""

    def __init__(self, locked_axes):
        self.locked_axes = locked_axes
        self._a1 = (0.0, 0.0, 0.0)
        self._a2 = (0.0, 0.0, 0.0)
        self._q1 = (0.0, 0.0, 0.0, 1.0)
        self._q2 = (0.0, 0.0, 0.0, 1.0)
        self._contacts_enabled = True
        self._limits = {}
        self._motors = {}
        self._coupled_axes = 0

    def coupled_axes(self, mask):
        """GenericJointBuilder::coupled_axes (generic_joint.rs): coupled linear axes share one distance row (spring / rope
        joints), two coupled angular axes one cone-like limit row."""
        self._coupled_axes = int(mask) & 63
        return self

    def local_anchor1(self, v):
        self._a1 = tuple(float(x) for x in v)
        return self

    def local_anchor2(self, v):
        self._a2 = tuple(float(x) for x in v)
        return self

    def contacts_enabled(self, flag):
        self._contacts_enabled = bool(flag)
        return self

    def local_axis1(self, axis):
        """GenericJoint::set_local_axis1: the joint's X axis in the first body's frame (generic_joint.rs:374-389)."""
        self._q1 = _rotation_arc_from_x(axis)
        return self

    def local_axis2(self, axis):
        self._q2 = _rotation_arc_from_x(axis)
        return self

    # GenericJoint::{set_limits, set_motor_velocity, set_motor_position, set_motor, set_motor_max_force, set_motor_model}
    # (generic_joint.rs:470-560); `axis` = 0..5 (LinX LinY LinZ AngX AngY AngZ)
    def limits(self, axis, lo, hi):
        self._limits[axis] = (float(lo), float(hi))
        return self

    def _motor(self, axis):
        return self._motors.setdefault(axis, dict(target_vel=0.0, target_pos=0.0, stiffness=0.0, damping=0.0, max_force=3.4028234663852886e38, model=0))

    def motor_velocity(self, axis, target_vel, factor):
        m = self._motor(axis)
        m.update(target_vel=float(target_vel), target_pos=0.0, stiffness=0.0, damping=float(factor))   # set_motor(axis, 0, vel, 0, factor)
        return self

    def motor_position(self, axis, target_pos, stiffness, damping):
        self._motor(axis).update(target_vel=0.0, target_pos=float(target_pos), stiffness=float(stiffness), damping=float(damping))
        return self

    def motor(self, axis, target_pos, target_vel, stiffness, damping):
        self._motor(axis).update(target_vel=float(target_vel), target_pos=float(target_pos), stiffness=float(stiffness), damping=float(damping))
        return self

    def motor_max_force(self, axis, max_force):
        self._motor(axis)["max_force"] = float(max_force)
        return self

    def motor_model(self, axis, model):
        self._motor(axis)["model"] = int(model)
        return self

    def build_desc(self, body1, body2):
        d = A.RbJointDesc()
        d.body1, d.body2 = int(body1), int(body2)
        d.local_frame1_t[:] = self._a1
        d.local_frame1_q[:] = self._q1
        d.local_frame2_t[:] = self._a2
        d.local_frame2_q[:] = self._q2
        d.locked_axes = self.locked_axes
        d.contacts_enabled = 1 if self._contacts_enabled else 0
        d.natural_frequency = 1.0e6   # SpringCoefficients::joint_defaults (integration_parameters.rs:78-83)
        d.damping_ratio = 1.0
        for ax in range(6):
            d.limits[ax][0], d.limits[ax][1] = -3.4028234663852886e38, 3.4028234663852886e38   # JointLimits::default
            d.motors[ax].max_force = 3.4028234663852886e38                                        # JointMotor::default
        for ax, (lo, hi) in self._limits.items():
            d.limit_axes |= 1 << ax
            d.limits[ax][0], d.limits[ax][1] = lo, hi
        for ax, m in self._motors.items():
            d.motor_axes |= 1 << ax
            for k, v in m.items():
                setattr(d.motors[ax], k, v)
        d.coupled_axes = self._coupled_axes
        return d


def SphericalJointBuilder():
    return GenericJointBuilder(0b000111)


def FixedJointBuilder():
    return GenericJointBuilder(0b111111)


def SpringJointBuilder(rest_length, stiffness, damping):
    """SpringJointBuilder::new (spring_joint.rs:32-38): no locked axis, LIN_AXES coupled, a force-based position motor on
    LinX acting on the distance between the anchors."""
    return GenericJointBuilder(0).coupled_axes(0b000111).motor_position(0, rest_length, stiffness, damping).motor_model(0, 1)


def RopeJointBuilder(max_dist):
    """RopeJointBuilder::new (rope_joint.rs:32-38, :153-156): LIN_AXES coupled, limits [0, max_dist] on LinX = an upper bound on
    the distance between the anchors."""
    return GenericJointBuilder(0).coupled_axes(0b000111).limits(0, 0.0, max_dist)


def _rotation_arc_from_x(axis):
    """Minimal rotation taking +X to `axis` (GenericJoint::complete_ang_frame, generic_joint.rs:374-389), xyzw."""
    import math
    a = [float(x) for x in axis]
    n = math.sqrt(sum(x * x for x in a))
    a = [x / n for x in a]
    d = a[0]                       # dot(X, axis)
    if d > 1.0 - 1e-7:
        return (0.0, 0.0, 0.0, 1.0)
    if d < -1.0 + 1e-7:
        return (0.0, 0.0, 1.0, 0.0)   # half turn about Z
    c = (0.0, -a[2], a[1])         # cross(X, axis)
    s = math.sqrt((1.0 + d) * 2.0)
    return (c[0] / s, c[1] / s, c[2] / s, s * 0.5)


def RevoluteJointBuilder(axis):
    """RevoluteJointBuilder::new(axis) (revolute_joint.rs): every axis locked except the rotation about `axis`,
    which is the X axis of both joint frames."""
    b = GenericJointBuilder(0b110111)   # LIN_X | LIN_Y | LIN_Z | ANG_Y | ANG_Z
    b._q1 = b._q2 = _rotation_arc_from_x(axis)
    return b


def PrismaticJointBuilder(axis):
    """PrismaticJointBuilder::new(axis) (prismatic_joint.rs): every axis locked except the translation along `axis`,
    which is the X axis of both joint frames."""
    b = GenericJointBuilder(0b111110)   # LIN_Y | LIN_Z | ANG_X | ANG_Y | ANG_Z
    b._q1 = b._q2 = _rotation_arc_from_x(axis)
    return b


class RigidBodySet:
    def __init__(self):
        self.descs = []

    def insert(self, builder):
        self.descs.append(builder.build_desc())
        return len(self.descs) - 1

    def __len__(self):
        return len(self.descs)


class ColliderSet:
    def __init__(self):
        self.descs = []
        self.filters = {}      # collider index -> RbColliderFilter, for the colliders whose filters are not the defaults
        self.hulls = []        # convex polyhedra referred to by RB_SHAPE_CONVEX colliders: (vertices [n, 3] f32, faces); id = index + 1
        self._hull_ids = {}

    def _desc(self, builder, parent):
        d = builder.build_desc(parent)
        hull = getattr(builder, "_hull", None)
        if hull is not None:
            key = (hull[0].tobytes(), tuple(tuple(f) for f in hull[1]))
            if key not in self._hull_ids:
                self.hulls.append(hull)
                self._hull_ids[key] = len(self.hulls)
            d.half_extents[0] = float(self._hull_ids[key])
        return d

    def insert(self, builder):
        return self.insert_with_parent(builder, None)

    def insert_with_parent(self, builder, parent, bodies=None):
        self.descs.append(self._desc(builder, parent))
        f = builder.build_filter()
        if f is not None:
            self.filters[len(self.descs) - 1] = f
        return len(self.descs) - 1

    def filter(self, i):
        """The current RbColliderFilter of collider i."""
        f = self.filters.get(i)
        if f is not None:
            return A.RbColliderFilter.from_buffer_copy(f)
        d = self.descs[i]
        return A.RbColliderFilter(d.collision_memberships, d.collision_filter, A.RB_TEST_AND, 0xFFFFFFFF, 0xFFFFFFFF, A.RB_TEST_AND,
                                  A.RB_ACT_DEFAULT)

    def __len__(self):
        return len(self.descs)


class ImpulseJointSet:
    def __init__(self):
        self.descs = []

    def insert(self, body1, body2, builder, wake_up=True):
        self.descs.append(builder.build_desc(body1, body2))
        return len(self.descs) - 1

    def __len__(self):
        return len(self.descs)


def convex_hull_mesh(points):
    """Hull mesh (vertices, faces) of 4..32 points, computed by the library's host routine rb_convex_hull."""
    import ctypes as C
    from ._lib import lib
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    L = lib()
    nv, nf = C.c_int32(0), C.c_int32(0)
    verts = np.zeros((32, 3), np.float32)
    sizes = np.zeros(32, np.int32)
    idx = np.zeros(256, np.int32)
    rc = L.rb_convex_hull(len(pts), pts.ctypes.data, C.byref(nv), verts.ctypes.data, C.byref(nf), sizes.ctypes.data, idx.ctypes.data)
    if rc < 0:
        raise ValueError(L.rb_last_error().decode())
    faces, at = [], 0
    for f in range(nf.value):
        faces.append([int(i) for i in idx[at:at + sizes[f]]])
        at += int(sizes[f])
    return verts[:nv.value].copy(), faces


def hull_arrays(hull):
    """(vertices, face sizes, face indices) of a registered hull as contiguous arrays for rb_world_add_hull."""
    verts, faces = hull
    sizes = np.array([len(f) for f in faces], np.int32)
    idx = np.array([i for f in faces for i in f], np.int32)
    return np.ascontiguousarray(verts, np.float32), sizes, idx


def as_array(descs, ctype):
    arr = (ctype * max(len(descs), 1))()
    for i, d in enumerate(descs):
        arr[i] = d
    return arr
