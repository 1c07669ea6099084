"""Collider filters beyond the collision groups: solver groups, ActiveCollisionTypes and the Or test mode of InteractionGroups,
set at upload through ColliderBuilder or at run time through rb_world_set_collider_filters.

Every check runs on the emulated kernels and, under -m gpu, on the CUDA library; the last test compares the two bit for bit.
- Truth tables: a pair exists exactly when Python restatements of ActiveCollisionTypes::test (collider_components.rs:300-334)
  and InteractionGroups::test (interaction_groups.rs:136-154) say so.
- Solver groups: a box whose solver groups exclude the slab's falls through it, bit-identically to a twin whose slab the
  collision groups remove, while the pair still reports Started / Stopped, contacts with zero impulses and no force event.
- Kinematic bodies: a kinematic sensor with KINEMATIC_FIXED sees parentless colliders at the steps its motion gives; two
  kinematic bodies with KINEMATIC_KINEMATIC touch without a constraint and keep separate islands.
- Fixed-fixed pairs: the reference's fixed_fixed_pair_kept_when_opted_in, and the pair set of a large static world with a
  seeded opted-in subset against a brute-force search over the fat boxes.
- Run-time changes (also on the static side under a sleeping body), the no-op call, and rejected calls that change nothing."""
import numpy as np
import pytest

import emul_lib
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder, SphericalJointBuilder
from rapier_b200.world import PhysicsWorld

ALL = 0xFFFFFFFF
KINDS = ("dynamic", "fixed", "kinematic_position_based", "kinematic_velocity_based", "parentless")
TYPE_OF = {"dynamic": A.RB_BODY_DYNAMIC, "fixed": A.RB_BODY_FIXED, "kinematic_position_based": A.RB_BODY_KINEMATIC_POSITION_BASED,
           "kinematic_velocity_based": A.RB_BODY_KINEMATIC_VELOCITY_BASED, "parentless": A.RB_BODY_FIXED}
ACT_ALL = (A.RB_ACT_DYNAMIC_DYNAMIC | A.RB_ACT_DYNAMIC_KINEMATIC | A.RB_ACT_DYNAMIC_FIXED | A.RB_ACT_KINEMATIC_KINEMATIC |
           A.RB_ACT_KINEMATIC_FIXED | A.RB_ACT_FIXED_FIXED)   # ActiveCollisionTypes::all()
TYPE_BITS = (A.RB_ACT_DYNAMIC_DYNAMIC, A.RB_ACT_DYNAMIC_KINEMATIC, A.RB_ACT_DYNAMIC_FIXED, A.RB_ACT_KINEMATIC_KINEMATIC,
             A.RB_ACT_KINEMATIC_FIXED, A.RB_ACT_FIXED_FIXED)


def types_test(bits, t1, t2):
    """ActiveCollisionTypes::test."""
    return bool(((bits >> (t1 * 4)) & 15) & (1 << t2)) or bool(((bits >> (t2 * 4)) & 15) & (1 << t1))


def groups_test(g1, g2):
    """InteractionGroups::test on (memberships, filter, mode): Or only when both sides use it."""
    a, b = (g1[0] & g2[1]) != 0, (g2[0] & g1[1]) != 0
    return (a or b) if g1[2] == A.RB_TEST_OR and g2[2] == A.RB_TEST_OR else (a and b)


@pytest.fixture(params=["emulated", pytest.param("cuda", marks=pytest.mark.gpu)])
def kind(request):
    if request.param == "cuda":
        request.getfixturevalue("built")
    return request.param


def make_world(kind, s, params=None):
    return PhysicsWorld(s, integration_parameters=params, _lib=emul_lib.lib() if kind == "emulated" else None)


def put(s, body_kind, collider, at):
    """A collider at `at` on a body of `body_kind` (or parentless); returns the collider index."""
    if body_kind == "parentless":
        return s.colliders.insert(collider.translation(at))
    s.insert(getattr(RigidBodyBuilder, body_kind)().translation(at), collider)
    return len(s.colliders) - 1


def pair_set(w):
    return {tuple(int(x) for x in p) for p in w.contact_pairs()["colliders"]}


def snapshot(w):
    pose, vel = w.body_states()
    return pose.view(np.uint32).copy(), vel.view(np.uint32).copy()


def test_collision_types_truth_table(kind):
    """Every pair of body kinds, with each collision-type bit on collider 1, on collider 2 or on neither, overlapping once."""
    s = scenes.Scene("act_truth", gravity=(0.0, 0.0, 0.0))
    expect = {}
    x = 0.0
    for i, k1 in enumerate(KINDS):
        for k2 in KINDS[i:]:
            for bits in TYPE_BITS:
                for where in (0, 1, 2):   # 0: neither (defaults on both), 1: collider 1, 2: collider 2
                    c1 = ColliderBuilder.cuboid(0.5, 0.5, 0.5)
                    c2 = ColliderBuilder.cuboid(0.5, 0.5, 0.5)
                    if where == 1:
                        c1.active_collision_types(bits)
                    if where == 2:
                        c2.active_collision_types(bits)
                    a = put(s, k1, c1, (x, 0.0, 0.0))
                    b = put(s, k2, c2, (x + 0.8, 0.0, 0.0))
                    b1 = bits if where == 1 else A.RB_ACT_DEFAULT
                    b2 = bits if where == 2 else A.RB_ACT_DEFAULT
                    t1, t2 = TYPE_OF[k1], TYPE_OF[k2]
                    expect[(min(a, b), max(a, b))] = types_test(b1, t1, t2) or types_test(b2, t1, t2)
                    x += 10.0
    w = make_world(kind, s)
    w.step()
    got = pair_set(w)
    wrong = {p: e for p, e in expect.items() if (p in got) != e}
    assert not wrong, f"{len(wrong)} pairs disagree with ActiveCollisionTypes::test, e.g. {list(wrong.items())[:5]}"
    assert got <= set(expect), "a pair between colliders of different cases"


GROUP_MASKS = ((1, 2), (2, 1), (1, 1), (3, 4), (4, 3), (ALL, ALL), (0, ALL), (ALL, 0))


def test_interaction_groups_truth_table(kind):
    """And / Or modes on both sides over a set of masks, on dynamic-fixed pairs; plus the reference's doc example."""
    s = scenes.Scene("groups_truth", gravity=(0.0, 0.0, 0.0))
    cases = [((m1, f1, o1), (m2, f2, o2)) for (m1, f1) in GROUP_MASKS for (m2, f2) in GROUP_MASKS
             for o1 in (A.RB_TEST_AND, A.RB_TEST_OR) for o2 in (A.RB_TEST_AND, A.RB_TEST_OR)]
    cases.append(((0b001, 0b110, A.RB_TEST_AND), (0b010, 0b001, A.RB_TEST_AND)))   # interaction_groups.rs:31-50: they collide
    expect = {}
    for n, (g1, g2) in enumerate(cases):
        a = put(s, "dynamic", ColliderBuilder.cuboid(0.5, 0.5, 0.5).collision_groups(*g1), (10.0 * n, 0.0, 0.0))
        b = put(s, "fixed", ColliderBuilder.cuboid(0.5, 0.5, 0.5).collision_groups(*g2), (10.0 * n + 0.8, 0.0, 0.0))
        expect[(a, b)] = groups_test(g1, g2)
    assert expect[(2 * len(cases) - 2, 2 * len(cases) - 1)]
    w = make_world(kind, s)
    w.step()
    got = pair_set(w)
    wrong = {p: e for p, e in expect.items() if (p in got) != e}
    assert not wrong, f"{len(wrong)} pairs disagree with InteractionGroups::test, e.g. {list(wrong.items())[:5]}"


def falling_scene(exclude):
    """A slab and four boxes resting on it (0 and 1 joined), each box with events on.  exclude = "solver": the boxes' solver
    groups exclude the slab; "collision": their collision groups do; None: nothing is excluded."""
    s = scenes.Scene("solver_groups")
    slab = ColliderBuilder.cuboid(8.0, 0.5, 8.0)
    if exclude == "solver":
        slab.solver_groups(2, 2)
    if exclude == "collision":
        slab.collision_groups(2, 2)
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), slab)
    for k, t in enumerate(((-3.0, 0.5, 0.0), (-1.0, 0.5, 0.0), (2.0, 0.5, 0.0), (2.0, 1.5, 0.0))):
        c = ColliderBuilder.cuboid(0.5, 0.5, 0.5).active_events(A.RB_EVENT_COLLISION | A.RB_EVENT_CONTACT_FORCE)
        if exclude == "solver":
            c.solver_groups(1, 1)
        if exclude == "collision":
            c.collision_groups(1, 1)
        s.insert(RigidBodyBuilder.dynamic().translation(t), c)
    s.joints.insert(1, 2, SphericalJointBuilder().local_anchor1((1.0, 0.0, 0.0)).local_anchor2((-1.0, 0.0, 0.0)))
    return s


@pytest.mark.parametrize("friction_model", [0, 1], ids=["simplified", "coulomb"])
def test_solver_groups_fall_through_like_removed_slab(kind, friction_model):
    p = A.RbIntegrationParameters.default()
    p.friction_model = friction_model
    w, twin = make_world(kind, falling_scene("solver"), p), make_world(kind, falling_scene("collision"), p)
    events, saw_contact = [], False
    for step in range(90):
        w.step()
        twin.step()
        a, t = snapshot(w), snapshot(twin)
        assert np.array_equal(a[0], t[0]) and np.array_equal(a[1], t[1]), f"step {step + 1}: bodies differ from the slab-less twin"
        cp = w.contact_pairs()
        touching = (cp["num_contacts"] > 0) & (cp["colliders"][:, 0] == 0)   # (the slab's pairs; box 4 rests on box 3)
        if touching.any():
            saw_contact = True
            assert not cp["impulses"][touching].any(), "a pair without forces reports impulses"
        events += w.collision_events()
        assert not [e for e in w.contact_force_events() if e["collider1"] == 0], "a pair without forces raised a contact-force event"
    pose, _ = w.body_states()
    assert (pose[1:, 1] < -2.0).all(), "the boxes did not fall through the slab"
    assert saw_contact
    started = {(e[0], e[1]) for e in events if e[2]}
    stopped = {(e[0], e[1]) for e in events if not e[2]}
    assert {(0, k) for k in range(1, 5)} <= started and {(0, k) for k in range(1, 5)} <= stopped, events
    assert twin.collision_events() == [] or all(0 not in e[:2] for e in twin.collision_events())


def test_ccd_ignores_solver_filtered_wall(kind):
    """A fast ball against a thin wall its solver groups exclude passes through, bit-identically to the wall-less twin."""
    def scene(with_wall):
        s = scenes.Scene("ccd_solver_groups", gravity=(0.0, 0.0, 0.0))
        s.insert(RigidBodyBuilder.dynamic().translation((-3.0, 0.0, 0.0)).linvel((200.0, 0.0, 0.0)),
                 ColliderBuilder.ball(0.1).solver_groups(1, 1))
        if with_wall:
            s.colliders.insert(ColliderBuilder.cuboid(0.02, 2.0, 2.0).solver_groups(2, 2))
        else:
            s.colliders.insert(ColliderBuilder.cuboid(0.02, 2.0, 2.0).translation((0.0, 100.0, 0.0)))
        return s
    w, twin = make_world(kind, scene(True)), make_world(kind, scene(False))
    for step in range(6):
        w.step()
        twin.step()
        a, t = snapshot(w), snapshot(twin)
        assert np.array_equal(a[0], t[0]) and np.array_equal(a[1], t[1]), f"step {step + 1}: the wall changed the ball"
    assert w.body_states()[0][0, 0] > 10.0


def kinematic_sensor_scene(with_bit):
    s = scenes.Scene("kinematic_sensor", gravity=(0.0, 0.0, 0.0))
    sensor = ColliderBuilder.ball(0.5).sensor().active_events(A.RB_EVENT_COLLISION)
    if with_bit:
        sensor.active_collision_types(A.RB_ACT_DEFAULT | A.RB_ACT_KINEMATIC_FIXED)
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((-5.05, 0.0, 0.0)), sensor)
    for x in (0.0, 4.0):
        s.colliders.insert(ColliderBuilder.cuboid(0.5, 0.5, 0.5).translation((x, 0.0, 0.0)))
    return s


@pytest.mark.parametrize("with_bit", [True, False], ids=["kinematic_fixed", "default"])
def test_kinematic_sensor_sees_parentless_colliders(kind, with_bit):
    """The sensor's pose after step k is x_k = -5.05 + 0.3 k; the narrow phase of step k sees x_(k-1).  It intersects the box at
    b while |x - b| <= 1 (radius + half extent; the positions keep 0.05 away from that bound)."""
    w = make_world(kind, kinematic_sensor_scene(with_bit))
    events = []
    for k in range(1, 41):
        w.set_next_kinematic_positions([0], np.array([[-5.05 + 0.3 * k, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]], np.float32))
        w.step()
        events += w.collision_events(with_flags=True)
    if not with_bit:
        assert events == []
        return
    expect = []
    for c, b in ((1, 0.0), (2, 4.0)):
        inside = [abs(-5.05 + 0.3 * (k - 1) - b) <= 1.0 for k in range(1, 41)]
        for k in range(1, 41):
            if inside[k - 1] != (inside[k - 2] if k > 1 else False):
                expect.append((0, c, 1 if inside[k - 1] else 0, k, A.RB_COLLISION_EVENT_SENSOR))
    assert sorted(events, key=lambda e: (e[3], e[1])) == sorted(expect, key=lambda e: (e[3], e[1]))


def kinematic_pair_scene(with_bit):
    s = scenes.Scene("kinematic_pair", gravity=(0.0, 0.0, 0.0))
    for x, v in ((-2.0, 1.0), (2.0, -1.0)):
        c = ColliderBuilder.cuboid(0.5, 0.5, 0.5).active_events(A.RB_EVENT_COLLISION)
        if with_bit:
            c.active_collision_types(A.RB_ACT_DEFAULT | A.RB_ACT_KINEMATIC_KINEMATIC)
        s.insert(RigidBodyBuilder.kinematic_velocity_based().translation((x, 0.0, 0.0)).linvel((v, 0.0, 0.0)), c)
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 5.0, 0.0)), ColliderBuilder.ball(0.5))   # (a body that is solved)
    return s


def test_kinematic_bodies_touch_without_constraint(kind):
    w, twin = make_world(kind, kinematic_pair_scene(True)), make_world(kind, kinematic_pair_scene(False))
    events, touched = [], False
    for step in range(180):
        w.step()
        twin.step()
        a, t = snapshot(w), snapshot(twin)
        assert np.array_equal(a[0], t[0]) and np.array_equal(a[1], t[1]), f"step {step + 1}: kinematic motion changed"
        cp = w.contact_pairs()
        if (cp["num_contacts"] > 0).any():
            touched = True
            assert not cp["impulses"].any()
            assert (cp["color"][cp["num_contacts"] > 0] == 255).all(), "a kinematic pair took a solver colour"
            labels = w.physics_pipeline.label_components()
            assert labels[0] != labels[1], "two touching kinematic bodies share an island"
        events += w.collision_events()
    assert touched
    assert [e[2] for e in events if (e[0], e[1]) == (0, 1)] == [1, 0], events
    assert twin.collision_events() == []


def resting_scene():
    s = scenes.Scene("resting")
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)),
             ColliderBuilder.cuboid(4.0, 0.5, 4.0).active_events(A.RB_EVENT_COLLISION))
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((2.5, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    return s


def test_collision_groups_switched_at_run_time(kind):
    w = make_world(kind, resting_scene())
    w.step(20)   # (settled, not yet asleep)
    w.collision_events()
    y0 = w.body_states()[0][1, 1]
    w.set_collider_filters([1], collision_groups=(1, 0))   # the box no longer meets the slab
    w.step()
    ev = w.collision_events()
    assert (0, 1, 0) in [e[:3] for e in ev], ev
    w.step(20)
    assert w.body_states()[0][1, 1] < y0 - 0.5, "the box did not fall"
    assert abs(w.body_states()[0][2, 1] - y0) < 1e-3, "the other box moved"
    w.set_collider_filters([1], collision_groups=(ALL, ALL))
    w.set_body_states([1], np.array([[0.0, 0.505, 0.0, 0.0, 0.0, 0.0, 1.0]], np.float32), np.zeros((1, 6), np.float32))
    w.step(5)
    assert (0, 1, 1) in [e[:3] for e in w.collision_events()]


def test_solver_groups_toggled_at_run_time(kind):
    w = make_world(kind, resting_scene())
    w.step(20)
    y0 = w.body_states()[0][1, 1]
    w.set_collider_filters([1], solver_groups=(1, 1))
    w.set_collider_filters([0], solver_groups=(2, 2))
    w.step(12)
    y1 = w.body_states()[0][1, 1]
    assert y1 < y0 - 0.1, "the box did not sink without contact forces"
    cp = w.contact_pairs()
    rows = [i for i, p in enumerate(cp["colliders"]) if tuple(p) == (0, 1)]
    assert rows and cp["num_contacts"][rows[0]] > 0 and not cp["impulses"][rows[0]].any()
    w.set_collider_filters([1], solver_groups=(ALL, ALL))
    w.step(2)
    cp = w.contact_pairs()
    rows = [i for i, p in enumerate(cp["colliders"]) if tuple(p) == (0, 1)]
    assert rows and cp["impulses"][rows[0]].any(), "the contact did not get its forces back"
    assert cp["color"][rows[0]] != 255


def test_default_filters_change_nothing(kind):
    s = falling_scene(None)
    w, twin = make_world(kind, s), make_world(kind, s)
    w.step(5)
    twin.step(5)
    w.set_collider_filters(range(len(s.colliders)), collision_groups=(ALL, ALL), solver_groups=(ALL, ALL),
                           active_collision_types=A.RB_ACT_DEFAULT)
    for step in range(30):
        w.step()
        twin.step()
        a, t = snapshot(w), snapshot(twin)
        assert np.array_equal(a[0], t[0]) and np.array_equal(a[1], t[1]), f"step {step + 1}"
    assert w.counters()["num_pairs"] == twin.counters()["num_pairs"]


@pytest.mark.parametrize("what", ["collision", "solver"])
def test_static_side_change_wakes_sleeping_bodies(kind, what):
    """The slab's filters change under boxes that have fallen asleep on it: the boxes wake and fall through, as the reference
    wakes every body that shares a pair with a changed collider (pair_management.rs:230-257)."""
    w = make_world(kind, resting_scene())
    for _ in range(300):
        w.step()
        if w.sleeping()[1:].all():
            break
    else:
        raise AssertionError("the boxes never fell asleep")
    w.collision_events()
    y0 = w.body_states()[0][1:, 1].copy()
    if what == "collision":
        w.set_collider_filters([0], collision_groups=(1, 0))
    else:
        w.set_collider_filters([0], solver_groups=(2, 0))
    assert not w.sleeping()[1:].any(), "the boxes on the changed slab were not woken"
    w.step(30)
    assert (w.body_states()[0][1:, 1] < y0 - 0.5).all(), "the boxes did not fall"
    if what == "collision":   # (with solver groups the sinking box still overlaps the slab: no Stopped yet)
        assert (0, 1, 0) in [e[:3] for e in w.collision_events()]


def test_fixed_fixed_pair_kept_when_opted_in(kind):
    """crates/rapier3d/tests/broad_phase_pair_filter.rs:32-48: two overlapping parentless cuboids, one with
    ActiveCollisionTypes::all(); after 3 steps exactly one contact pair, which touches.  Without the opt-in: none."""
    pairs = []
    for opted in (True, False):
        s = scenes.Scene("fixed_fixed")
        c = ColliderBuilder.cuboid(1.0, 1.0, 1.0).active_events(A.RB_EVENT_COLLISION)
        s.colliders.insert(c.active_collision_types(ACT_ALL) if opted else c)
        s.colliders.insert(ColliderBuilder.cuboid(1.0, 1.0, 1.0).translation((0.5, 0.5, 0.0)))
        w = make_world(kind, s)
        events = []
        for _ in range(3):
            w.step()
            events += w.collision_events()
        cp = w.contact_pairs()
        pairs.append(len(cp["colliders"]))
        if opted:
            assert cp["num_contacts"][0] > 0 and not cp["impulses"].any()
            assert events == [(0, 1, 1, 1)], events
    assert pairs == [1, 0]


def static_world(n, seed):
    """n parentless cuboids over a 2-D field (a few of them wide plates), a seeded 2 % of them opted into FIXED_FIXED, and
    one dynamic ball far away."""
    rng = np.random.default_rng(seed)
    side = float(np.sqrt(n) * 3.2)
    s = scenes.Scene(f"static_{n}", gravity=(0.0, 0.0, 0.0))
    centres = rng.uniform((0.0, 0.0, 0.0), (side, 2.0, side), (n, 3))
    half = rng.uniform(0.2, 1.5, (n, 3))
    half[: n // 500] = (40.0, 0.2, 1.0)   # wide plates: over 4x the mean width along x, so in the wide list
    opted = rng.random(n) < 0.02
    for k in range(n):
        c = ColliderBuilder.cuboid(*half[k]).translation(tuple(centres[k]))
        s.colliders.insert(c.active_collision_types(A.RB_ACT_DEFAULT | A.RB_ACT_FIXED_FIXED) if opted[k] else c)
    s.insert(RigidBodyBuilder.dynamic().translation((-100.0, 0.0, -100.0)), ColliderBuilder.ball(0.5))
    return s, opted


@pytest.mark.parametrize("size", [pytest.param(4000, id="4k"), pytest.param(100000, id="100k", marks=pytest.mark.gpu)])
def test_fixed_fixed_pairs_at_size(kind, size):
    if kind == "emulated" and size > 4000:
        pytest.skip("sized for the device")
    s, opted = static_world(size, 11)
    w = make_world(kind, s)
    w.reserve(len(s.bodies), len(s.colliders) + 1000)   # (pair capacity for the fixed-fixed pairs)
    w.step(2)
    fat = w.debug_read("collider_fat", np.float32).reshape(-1, 6)[:size]
    lo, hi = fat[:, :3], fat[:, 3:]
    expect = set()
    for i in np.flatnonzero(opted):   # every pair with an opted-in side whose fat boxes overlap (closed intervals)
        hit = np.flatnonzero(((lo <= hi[i]) & (hi >= lo[i])).all(axis=1))
        expect.update((min(i, j), max(i, j)) for j in hit if j != i)
    got = pair_set(w)
    assert all(a < size and b < size for a, b in got)
    assert got == expect, (len(got), len(expect), sorted(got ^ expect)[:5])
    assert len(expect) > size // 200


BAD_FILTERS = {
    "out_of_range": (10 ** 6, {}), "negative": (-1, {}), "removed": (5, {}),
    "unknown_bit": (1, dict(active_collision_types=0x1000)), "mode_2": (1, dict(collision_test_mode=2)),
    "solver_mode_2": (1, dict(solver_test_mode=2)),
}
BAD_TEXT = {"out_of_range": "collider index out of range (or removed)", "negative": "collider index out of range (or removed)",
            "removed": "collider index out of range (or removed)", "unknown_bit": "unknown active collision type bits",
            "mode_2": "interaction test mode is neither RB_TEST_AND nor RB_TEST_OR",
            "solver_mode_2": "interaction test mode is neither RB_TEST_AND nor RB_TEST_OR"}


@pytest.mark.parametrize("bad", sorted(BAD_FILTERS))
def test_rejected_filter_call_changes_nothing(kind, bad):
    def scene():
        s = falling_scene(None)
        s.insert(RigidBodyBuilder.dynamic().translation((6.0, 3.0, 0.0)), ColliderBuilder.ball(0.3))   # body 5, collider 5: removed
        return s
    w, twin = make_world(kind, scene()), make_world(kind, scene())
    for x in (w, twin):
        x.step(3)
        x.remove(5)
        x.step(2)
    index, fields = BAD_FILTERS[bad]
    good = A.RbColliderFilter(1, 1, 0, 2, 2, 0, A.RB_ACT_DEFAULT)   # would separate box 1 from everything
    worse = A.RbColliderFilter(ALL, ALL, 0, ALL, ALL, 0, A.RB_ACT_DEFAULT)
    for k, v in fields.items():
        setattr(worse, k, v)
    from rapier_b200.sets import as_array
    idx = np.array([1, index], np.int32)
    pp = w.physics_pipeline
    assert pp.L.rb_world_set_collider_filters(pp.h, 2, idx.ctypes.data, as_array([good, worse], A.RbColliderFilter)) == -3
    assert pp.L.rb_last_error().decode() == BAD_TEXT[bad]
    for step in range(20):
        w.step()
        twin.step()
        a, t = snapshot(w), snapshot(twin)
        assert np.array_equal(a[0], t[0]) and np.array_equal(a[1], t[1]), f"{step + 1} steps after the call"
        assert np.array_equal(w.contact_pairs()["colliders"], twin.contact_pairs()["colliders"])


def mixed_scene(seed):
    """Boxes and balls over a slab with every filter kind, a sensor, a CCD bullet, a joint and two kinematic bodies."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"mixed_filters_{seed}")
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(10.0, 0.5, 10.0).solver_groups(1, 3))
    s.colliders.insert(ColliderBuilder.cuboid(0.05, 2.0, 4.0).translation((6.0, 2.0, 0.0)).collision_groups(1, 1, A.RB_TEST_OR))
    for k in range(40):
        c = (ColliderBuilder.cuboid(0.4, 0.4, 0.4) if k % 2 else ColliderBuilder.ball(0.4)).active_events(A.RB_EVENT_COLLISION)
        r = int(rng.integers(0, 4))
        if r == 1:
            c.solver_groups(2, 2)
        elif r == 2:
            c.collision_groups(int(rng.integers(1, 4)), int(rng.integers(1, 4)), int(rng.integers(0, 2)))
        elif r == 3:
            c.active_collision_types(A.RB_ACT_DYNAMIC_DYNAMIC | A.RB_ACT_DYNAMIC_KINEMATIC)
        s.insert(RigidBodyBuilder.dynamic().translation(tuple(rng.uniform((-4.0, 0.5, -4.0), (4.0, 6.0, 4.0)))), c)
    s.insert(RigidBodyBuilder.kinematic_velocity_based().translation((-3.0, 1.0, 6.0)).linvel((1.0, 0.0, 0.0)),
             ColliderBuilder.cuboid(1.0, 0.5, 0.5).sensor().active_events(A.RB_EVENT_COLLISION)
             .active_collision_types(A.RB_ACT_DEFAULT | A.RB_ACT_KINEMATIC_FIXED | A.RB_ACT_KINEMATIC_KINEMATIC))
    s.insert(RigidBodyBuilder.kinematic_velocity_based().translation((3.0, 1.0, 6.0)).linvel((-1.0, 0.0, 0.0)),
             ColliderBuilder.cuboid(0.5, 0.5, 0.5).active_events(A.RB_EVENT_COLLISION)
             .active_collision_types(A.RB_ACT_DEFAULT | A.RB_ACT_KINEMATIC_KINEMATIC))
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 2.0, 0.0)).linvel((80.0, 0.0, 0.0)).ccd_enabled(True),
             ColliderBuilder.ball(0.1).solver_groups(1, 1))
    s.joints.insert(1, 2, SphericalJointBuilder().local_anchor1((0.5, 0.0, 0.0)).local_anchor2((-0.5, 0.0, 0.0)))
    s.colliders.insert(ColliderBuilder.cuboid(1.0, 1.0, 1.0).translation((-8.0, 1.0, -8.0)).active_events(A.RB_EVENT_COLLISION)
                       .active_collision_types(ACT_ALL))
    s.colliders.insert(ColliderBuilder.cuboid(1.0, 1.0, 1.0).translation((-7.5, 1.5, -8.0)))
    return s


@pytest.mark.gpu
def test_mixed_scene_gpu_matches_emulation(built):
    s = mixed_scene(7)
    gpu, emu = make_world("cuda", s), make_world("emulated", s)
    for step in range(200):
        gpu.step()
        emu.step()
        a, t = snapshot(gpu), snapshot(emu)
        assert np.array_equal(a[0], t[0]) and np.array_equal(a[1], t[1]), f"step {step + 1}: bodies differ"
        pg, pe = gpu.contact_pairs(), emu.contact_pairs()
        for k in ("colliders", "num_contacts", "color"):
            assert np.array_equal(pg[k], pe[k]), f"step {step + 1}: {k}"
        assert np.array_equal(pg["impulses"].view(np.uint32), pe["impulses"].view(np.uint32)), f"step {step + 1}: impulses"
        assert gpu.collision_events(with_flags=True) == emu.collision_events(with_flags=True), f"step {step + 1}: events"
