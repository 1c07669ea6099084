"""Set-editing calls of the C ABI are all-or-nothing: a call that mixes valid entries with one invalid entry returns
RB_ERR_INVALID (-3), with its rb_last_error text, and changes nothing -- no device table, host mirror or sleep state -- so
the world then steps bit-identically to a twin that never saw the call (poses, velocities, sleeping flags and counters,
over 20 steps).

Checked on the oracle (orc_world_*), the emulated kernels and, under -m gpu, the CUDA library, for set_body_states,
set_body_forces, set_next_kinematic_positions, wake_up, remove_bodies, insert, insert_joints, remove_joints and
update_joints, with an index out of range, a negative index, and for set_next_kinematic_positions a body that is not
position-based kinematic.  The calls that wake bodies are also made on a world that has fallen asleep: it stays asleep."""
import copy

import numpy as np
import pytest

import emul_lib
import oracle_lib
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder, SphericalJointBuilder, as_array
from rapier_b200.world import PhysicsWorld

BODY_RANGE = "body index out of range"
ERRORS = {
    "set_body_states": BODY_RANGE, "set_body_forces": BODY_RANGE, "wake_up": BODY_RANGE, "remove_bodies": BODY_RANGE,
    "set_next_kinematic_positions": "rb_world_set_next_kinematic_positions: not a position-based kinematic body",
    "insert": "collider with unsupported shape, unknown hull or bad parent",
    "insert_joints": "joint with bad body index or axes",
    "remove_joints": "joint index out of range",
    "update_joints": "joint index out of range (or removed)",
}
BAD = {"out_of_range": 10 ** 6, "negative": -1, "not_kinematic": 2}   # body 2 is dynamic
WAKING = ("set_body_states", "set_body_forces", "wake_up")
CASES = [(entry, bad, False) for entry in ERRORS for bad in ("out_of_range", "negative")
         if not (entry == "insert" and bad == "negative")]   # (a collider parent of -1 is valid: no parent)
CASES += [("set_next_kinematic_positions", "not_kinematic", False)]
CASES += [(entry, bad, True) for entry in WAKING for bad in ("out_of_range", "negative")]
DYNAMIC = [1, 2, 3, 4]


def scene():
    """Bodies 0 a slab, 1..4 boxes resting on it (1 and 3 linked by a spherical joint, 4 stacked on 2), 5 a position-based
    kinematic ball out of reach."""
    s = scenes.Scene("abi_edits")
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(6.0, 0.5, 6.0))
    for t in ((-2.0, 0.5, 0.0), (0.0, 0.5, 0.0), (2.0, 0.5, 0.0), (0.0, 1.5, 0.0)):
        s.insert(RigidBodyBuilder.dynamic().translation(t), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((4.0, 4.0, 4.0)), ColliderBuilder.ball(0.5))
    s.joints.insert(1, 3, SphericalJointBuilder().local_anchor1((2.0, 0.0, 0.0)).local_anchor2((-2.0, 0.0, 0.0)))
    return s


def rejected_call(entry, bad, s):
    """The arguments after the world of a call to `entry` whose first entries are valid and whose last one is not."""
    b = BAD[bad]
    idx = lambda *v: np.array(v, np.int32)
    pose = np.tile(np.array([5.0, 5.0, 5.0, 0.0, 0.0, 0.0, 1.0], np.float32), (2, 1))
    if entry == "set_body_states":
        return [2, idx(1, b), pose, np.ones((2, 6), np.float32)]
    if entry == "set_body_forces":
        return [2, idx(2, b), np.full((2, 3), 50.0, np.float32), np.full((2, 3), 5.0, np.float32)]
    if entry == "set_next_kinematic_positions":
        return [2, idx(5, b), pose]
    if entry in ("wake_up", "remove_bodies"):
        return [2, idx(4, b)]
    if entry == "insert":
        bodies = [RigidBodyBuilder.dynamic().translation((-4.0, 0.5, 3.0)).build_desc()] * 2
        colliders = [ColliderBuilder.cuboid(0.5, 0.5, 0.5).build_desc(len(s.bodies)), ColliderBuilder.ball(0.5).build_desc(b)]
        return [2, as_array(bodies, A.RbBodyDesc), 2, as_array(colliders, A.RbColliderDesc)]
    if entry == "insert_joints":
        return [2, as_array([SphericalJointBuilder().build_desc(2, 4), SphericalJointBuilder().build_desc(2, b)], A.RbJointDesc)]
    if entry == "remove_joints":
        return [2, idx(0, b)]
    d = copy.deepcopy(s.joints.descs[0])
    d.natural_frequency = 10.0
    return [2, idx(0, b), as_array([d, d], A.RbJointDesc), 1]


class Backend:
    """A world of one backend and its raw entry points (the status of the C call, not the wrappers' exceptions)."""

    def __init__(self, kind, s):
        self.kind = kind
        if kind == "oracle":
            self.w = oracle_lib.OracleWorld(s)
            self.L, self.h = self.w.L, self.w.h
        else:
            self.w = PhysicsWorld(s, _lib=emul_lib.lib() if kind == "emulated" else None)
            self.w.reserve(len(s.bodies) + 4, len(s.colliders) + 4)
            self.w.reserve_joints(len(s.joints) + 4)
            self.L, self.h = self.w.physics_pipeline.L, self.w.physics_pipeline.h

    def call(self, entry, args):
        args = [x.ctypes.data if isinstance(x, np.ndarray) else x for x in args]
        if self.kind == "oracle":
            return getattr(self.L, "orc_world_" + entry)(self.h, *args)
        outputs = {"insert": 2, "insert_joints": 1}.get(entry, 0)   # first indices of the appended entries: not asked for
        return getattr(self.L, "rb_world_" + entry)(self.h, *args, *([None] * outputs))

    def snapshot(self):
        pose, vel = self.w.body_states()
        counters = {k: v for k, v in self.w.counters().items() if not k.endswith("_ms")}   # (times are measured, not computed)
        return dict(poses=pose.view(np.uint32), velocities=vel.view(np.uint32), sleeping=self.w.sleeping(), counters=counters)


@pytest.fixture(params=["oracle", "emulated", pytest.param("cuda", marks=pytest.mark.gpu)])
def kind(request):
    if request.param == "cuda":
        request.getfixturevalue("built")
    return request.param


@pytest.mark.parametrize("entry,bad,asleep", CASES, ids=[f"{e}-{b}" + ("-asleep" if s else "") for e, b, s in CASES])
def test_rejected_edit_changes_nothing(kind, entry, bad, asleep):
    s = scene()
    world, twin = Backend(kind, s), Backend(kind, s)
    for steps in range(600):
        world.w.step()
        twin.w.step()
        if not asleep or world.w.sleeping()[DYNAMIC].all():
            break
    else:
        raise AssertionError("the boxes never fell asleep")
    args = rejected_call(entry, bad, s)
    assert world.call(entry, args) == -3
    if kind != "oracle":
        assert world.L.rb_last_error().decode() == ERRORS[entry]
    if asleep:
        assert world.w.sleeping()[DYNAMIC].all(), "a rejected call woke bodies"
    for i in range(21):
        if i:
            world.w.step()
            twin.w.step()
        a, t = world.snapshot(), twin.snapshot()
        for what in a:
            same = a[what] == t[what] if what == "counters" else np.array_equal(a[what], t[what])
            assert same, f"{i} steps after the call: {what} differ from the twin's"
