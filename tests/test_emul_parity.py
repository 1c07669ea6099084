"""Kernel LOGIC check without a GPU: the phase functions of rapier_b200/csrc compiled for the host
(tests/emul, -DRB_EMULATE, one thread playing every CUDA thread) against the CPU oracle.  These do
not exercise the product library; the `-m gpu` tests do that on the GPU."""
import numpy as np
from rapier_b200 import _abi as A
import pytest

import emul_lib
import oracle_lib
from parity_util import compare_worlds, is_exact
from rapier_b200 import scenes
from rapier_b200.world import PhysicsWorld

CASES = [
    ("pyramids_2x2x10", lambda: scenes.pyramids(2, 2, 10), 25, 5),
    ("pile_with_joint_chain", lambda: scenes.box_pile(4, 4, 5), 120, 20),
    ("single_pyramid_20", lambda: scenes.single_pyramid(20), 20, 5),
    ("pyramid3_large_island", lambda: scenes.pyramid3(9), 25, 5),
    ("joint_grid_large_island", lambda: scenes.joint_grid(18), 40, 10),
    ("ball_on_slab", lambda: scenes.box_on_ground("ball", 2.0), 80, 20),
    ("keva_small", lambda: scenes.keva(1), 20, 5),
    ("large_world_reduced", lambda: scenes.large_world(grid=60, spheres=16), 150, 30),   # parentless static floor tiles
]


@pytest.mark.parametrize("name,make,steps,every", CASES, ids=[c[0] for c in CASES])
def test_emulated_kernels_match_oracle_bit_for_bit(name, make, steps, every):
    scene = make()
    w = PhysicsWorld(scene, _lib=emul_lib.lib())
    o = oracle_lib.OracleWorld(scene)
    for i in range(steps):
        w.step()
        o.step()
        if i % every == every - 1 or i < 2:
            d = compare_worlds(w, o)
            assert is_exact(d), f"{name}: step {i}: {d}"


@pytest.mark.parametrize("smem_floats", [8000, 12000])
def test_emulated_streaming_pipeline_matches_oracle(monkeypatch, smem_floats):
    """Items whose constraints do not fit the (here: artificially small) shared memory are streamed
    from the pool through the two-buffer staging pipeline; results must not change."""
    monkeypatch.setenv("RB_EMU_COOP_SMEM_FLOATS", str(smem_floats))
    scene = scenes.pyramids(2, 2, 10)
    w = PhysicsWorld(scene, _lib=emul_lib.lib())
    o = oracle_lib.OracleWorld(scene)
    for i in range(12):
        w.step()
        o.step()
        assert is_exact(compare_worlds(w, o)), f"step {i}"
    st = w.debug_read("state", np.int32)
    assert st[19] == 4, "the four pyramids must have taken the streaming path"


def test_empty_and_ragged_scenes():
    """Edge cases: no bodies, bodies without colliders, colliders without contacts."""
    from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder
    s = scenes.Scene("empty")
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w.step(3)
    s = scenes.Scene("ragged")
    s.bodies.insert(RigidBodyBuilder.dynamic().translation((0, 5, 0)))           # no collider: zero mass
    s.insert(RigidBodyBuilder.dynamic().translation((3, 5, 0)), ColliderBuilder.ball(0.5))
    s.colliders.insert(ColliderBuilder.cuboid(5, 0.5, 5))                         # parentless fixed collider
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    o = oracle_lib.OracleWorld(s)
    for _ in range(120):
        w.step()
        o.step()
    assert is_exact(compare_worlds(w, o))
    pose, _ = w.body_states()
    assert abs(pose[1, 1] - 1.0) < 0.02 and np.isfinite(pose).all()


from variant_cases import VARIANTS  # noqa: E402


@pytest.mark.parametrize("name,make,params,steps,every", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_emulated_variants_match_oracle(name, make, params, steps, every):
    scene = make()
    w = PhysicsWorld(scene, integration_parameters=params, _lib=emul_lib.lib())
    o = oracle_lib.OracleWorld(scene, params=params)
    for i in range(steps):
        w.step()
        o.step()
        if i % every == every - 1 or i < 2:
            d = compare_worlds(w, o)
            assert is_exact(d), f"{name}: step {i}: {d}"
    pose, _ = w.body_states()
    assert np.isfinite(pose).all()


def test_capacity_overflow_is_reported_after_asynchronous_steps():
    """A status raised on the device (here: more broad-phase pairs than the pair table holds) must reach the caller
    at the next synchronising call even when the steps were enqueued asynchronously (sync = 0 / step_host)."""
    from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder
    from rapier_b200.world import RapierError
    s = scenes.Scene("crowd", gravity=(0.0, 0.0, 0.0))
    for i in range(330):   # 330 balls within one ball radius of each other: 54 285 pairs > 16 per dynamic collider
        s.insert(RigidBodyBuilder.dynamic().translation((0.001 * i, 0.0, 0.0)), ColliderBuilder.ball(0.5))
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w.step(1, sync=False)
    with pytest.raises(RapierError, match="-4"):
        w.physics_pipeline.synchronize()
    w.physics_pipeline.synchronize()   # reported once, then cleared
    with pytest.raises(RapierError, match="-4"):
        w.physics_pipeline.step_host(s.gravity, None, None)


def test_large_world_insertion_protocol_emulated():
    """b3d_large_world.rs:55-77 as written: a static tiled floor, one sphere INSERTED every 5 steps (the pair table,
    colours and warm-start data of the spheres already resting must survive every insertion)."""
    from incremental_cases import large_world_protocol_case
    large_world_protocol_case(lib=emul_lib.lib())


def test_body_removal_and_insertion_emulated():
    from incremental_cases import removal_case
    removal_case(lib=emul_lib.lib())


def test_whole_island_sleep_emulated_kernels():
    from test_oracle_kat import sleeping_stack_is_woken_by_an_impact, whole_island_blocks_partial_sleep
    whole_island_blocks_partial_sleep(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))
    sleeping_stack_is_woken_by_an_impact(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))


def test_sleep_and_wake_match_oracle_bit_for_bit():
    """A pile that settles, falls asleep island by island, and is woken by a late projectile: every step of it."""
    from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder
    scene = scenes.box_pile(3, 3, 3)
    scene.insert(RigidBodyBuilder.dynamic().translation((0.0, 60.0, 0.3)).linvel((0.0, -2.0, 0.0)), ColliderBuilder.ball(0.5).density(5.0))
    w = PhysicsWorld(scene, _lib=emul_lib.lib())
    o = oracle_lib.OracleWorld(scene)
    seen_sleep = seen_wake = False
    prev = 0
    for i in range(330):
        w.step(); o.step()
        sw, so = w.sleeping(), o.sleeping()
        assert (sw == so).all(), i
        n = int(sw.sum())
        seen_sleep = seen_sleep or n > 5
        seen_wake = seen_wake or (prev > 5 and n < prev)
        prev = n
        if i % 15 == 14:
            assert is_exact(compare_worlds(w, o)), i
    assert seen_sleep and seen_wake


def test_coulomb_friction_cone_emulated_kernels():
    from test_oracle_kat import _coulomb_params, coulomb_friction_cone
    coulomb_friction_cone(lambda s: PhysicsWorld(s, integration_parameters=_coulomb_params(), _lib=emul_lib.lib()))


def test_ccd_emulated_kernels():
    from test_oracle_kat import ccd_bullet_still_hits_dynamic, ccd_default_tier, ccd_large_dt_no_mid_air_hitch
    mk = lambda s, p: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib())
    ccd_default_tier(mk)
    ccd_large_dt_no_mid_air_hitch(mk)
    ccd_bullet_still_hits_dynamic(mk)


def test_contact_force_events_emulated_kernels():
    from test_oracle_kat import contact_force_event_started_marks_threshold_crossings
    contact_force_event_started_marks_threshold_crossings(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))


def test_event_lists_match_oracle():
    from variant_cases import events_parity_case
    events_parity_case(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), lambda s: oracle_lib.OracleWorld(s))


def test_kinematic_bodies_emulated_kernels():
    from test_oracle_kat import kinematic_bodies, moving_kinematic_wakes_jointed_dynamic
    from variant_cases import kinematic_parity_case
    kinematic_bodies(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))
    moving_kinematic_wakes_jointed_dynamic(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))
    kinematic_parity_case(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), lambda s: oracle_lib.OracleWorld(s))


def test_joint_limits_and_motors_emulated_kernels():
    from test_oracle_kat import angular_limits_are_reached, prismatic_limits_and_position_motor
    from variant_cases import joint_limits_parity_case
    mk = lambda s: PhysicsWorld(s, _lib=emul_lib.lib())
    angular_limits_are_reached(mk, cases=((-45.0, 45.0), (45.0, 315.0)))
    prismatic_limits_and_position_motor(mk)
    joint_limits_parity_case(mk, lambda s, p=None: oracle_lib.OracleWorld(s, params=p))
    joint_limits_parity_case(lambda s, p=None: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib()),
                             lambda s, p=None: oracle_lib.OracleWorld(s, params=p), coulomb=True)


def test_coupled_joint_axes_emulated_kernels():
    from test_oracle_kat import coupled_angular_spring_joint_stays_finite, heavy_cubes_rest_on_spring_jointed_balls, spring_and_rope_joints
    from variant_cases import coupled_axes_parity_case
    mk = lambda s, p=None: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib())
    mo = lambda s, p=None: oracle_lib.OracleWorld(s, params=p)
    spring_and_rope_joints(mk)
    heavy_cubes_rest_on_spring_jointed_balls(mk, num=12)
    coupled_angular_spring_joint_stays_finite(mk)
    coupled_axes_parity_case(mk, mo)
    coupled_axes_parity_case(mk, mo, coulomb=True, warmstart_joints=True, steps=60)


def test_additional_solver_iterations_emulated_kernels():
    from test_oracle_kat import additional_solver_iterations
    from variant_cases import substep_groups_parity_case
    mk = lambda s, p=None: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib())
    mo = lambda s, p=None: oracle_lib.OracleWorld(s, params=p)
    additional_solver_iterations(mk)
    substep_groups_parity_case(mk, mo, steps=40)
    substep_groups_parity_case(mk, mo, steps=30, big=False, coulomb=True, warmstart_joints=True)


def test_sensors_emulated_kernels():
    from test_oracle_kat import sensors
    from variant_cases import sensors_parity_case
    sensors(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))
    sensors_parity_case(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), lambda s: oracle_lib.OracleWorld(s))


def test_compound_bodies_emulated_kernels():
    from parity_util import compare_worlds, is_exact
    from test_oracle_kat import compound_bodies
    from variant_cases import compound_pile
    compound_bodies(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), n=4)
    s = compound_pile()
    w, o = PhysicsWorld(s, _lib=emul_lib.lib()), oracle_lib.OracleWorld(s)
    for i in range(200):
        w.step(); o.step()
        if i % 20 == 19 or i < 2:
            d = compare_worlds(w, o)
            assert is_exact(d), (i, d)


def test_island_structure_emulated_kernels():
    from test_oracle_kat import island_structure
    island_structure(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), lambda w: w.physics_pipeline.label_components())
    from test_oracle_kat import multi_collider_slab_sleeps, sleep_gates_on_displacement
    sleep_gates_on_displacement(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))
    multi_collider_slab_sleeps(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), ni=20, nj=12)


def test_joint_insertion_and_removal_emulated_kernels():
    """ImpulseJointSet::insert / remove after the world has been stepped (rb_world_insert_joints / rb_world_remove_joints).
    persistent_islands.rs joint_links_and_split_after_removal: a rope joint between two distant resting boxes merges their
    islands in the next step, removing it splits them again.  Then a run with joints of every path coming and going -- a
    spherical chain link, a spring, a revolute joint with a limit and contacts disabled between overlapping boxes -- bit-exact
    against the oracle at every checkpoint, warm-start data of everything else untouched."""
    from parity_util import compare_worlds, is_exact
    from rapier_b200.sets import ColliderBuilder, RevoluteJointBuilder, RigidBodyBuilder, RopeJointBuilder, SphericalJointBuilder, SpringJointBuilder
    s = scenes.Scene("joint_islands", gravity=(0.0, -9.81, 0.0))
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(100.0, 0.5, 100.0))
    a = s.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    b = s.insert(RigidBodyBuilder.dynamic().translation((20.0, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    for make in (lambda: PhysicsWorld(s, _lib=emul_lib.lib()), lambda: oracle_lib.OracleWorld(s)):
        w = make()
        island = (lambda: w.physics_pipeline.label_components()) if isinstance(w, PhysicsWorld) else (lambda: w.debug_read("island_of", np.int32))
        if isinstance(w, PhysicsWorld):
            w.reserve_joints(4, generic=True)
        w.step(240)
        assert island()[a] != island()[b]
        rope = RopeJointBuilder(30.0).build_desc(a, b)
        (w.physics_pipeline if isinstance(w, PhysicsWorld) else w).insert_joints([rope])
        w.step(1)
        assert island()[a] == island()[b], "a joint must merge islands"
        (w.physics_pipeline if isinstance(w, PhysicsWorld) else w).remove_joints([0])
        w.step(240)
        assert island()[a] != island()[b], "removing the joint must split them again"

    s = scenes.box_pile(3, 3, 3)
    nb = len(s.bodies)
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w.reserve_joints(8, generic=True)
    o = oracle_lib.OracleWorld(s)
    nj0 = len(s.joints)
    dyn = [i for i, d in enumerate(s.bodies.descs) if d.body_type == 0]
    plan = {
        10: ("insert", SphericalJointBuilder().local_anchor1((0.4, 0.0, 0.0)).local_anchor2((-0.4, 0.0, 0.0)).build_desc(dyn[0], dyn[1])),
        25: ("insert", SpringJointBuilder(0.8, 150.0, 6.0).build_desc(dyn[2], dyn[5])),
        40: ("insert", RevoluteJointBuilder((0.0, 1.0, 0.0)).local_anchor1((0.0, 0.5, 0.0)).local_anchor2((0.0, -0.5, 0.0)).limits(4, -0.4, 0.6).contacts_enabled(False).build_desc(dyn[3], dyn[4])),
        70: ("remove", [nj0]),
        90: ("remove", [nj0 + 2]),
        100: ("insert", RopeJointBuilder(1.5).build_desc(dyn[0], dyn[7])),
    }
    for i in range(140):
        if i in plan:
            kind, arg = plan[i]
            if kind == "insert":
                w.physics_pipeline.insert_joints([arg]); o.insert_joints([arg])
            else:
                w.physics_pipeline.remove_joints(arg); o.remove_joints(arg)
        w.step(); o.step()
        if i % 10 == 9 or i in plan or i - 1 in plan:
            d = compare_worlds(w, o)
            assert is_exact(d), (i, d)
            ji_w, ji_o = w.debug_read("joint_impulses", np.float32), o.debug_read("joint_impulses", np.float32)
            assert (ji_w.view(np.uint32) == ji_o.view(np.uint32)).all(), i
    # capacity and path errors are reported, not silently ignored
    from rapier_b200.world import RapierError
    w2 = PhysicsWorld(s, _lib=emul_lib.lib())
    w2.step(1)
    with pytest.raises(RapierError):
        w2.physics_pipeline.insert_joints([plan[10][1]] * 64)


def test_joint_update_emulated_kernels():
    """rb_world_update_joints = ImpulseJointSet::get_mut(handle, wake_up) + edits.  issue_692_joint_get_mut_wakes_bodies.rs: a
    revolute joint between a kinematic body and a ball that has fallen asleep gets a velocity motor: the ball is awake after the
    next step and starts turning.  Then motor targets and limits of a jointed pile are changed every few steps, bit-exact against
    the oracle (warm-start impulses carried across the updates)."""
    from parity_util import compare_worlds, is_exact
    from rapier_b200.sets import ColliderBuilder, RevoluteJointBuilder, RigidBodyBuilder
    from variant_cases import joint_limits_scene
    s = scenes.Scene("issue_692", gravity=(0.0, -9.81, 0.0))
    kin = s.bodies.insert(RigidBodyBuilder.kinematic_position_based())
    dyn = s.insert(RigidBodyBuilder.dynamic().translation((0.0, -2.0, 0.0)), ColliderBuilder.ball(0.5))
    jb = lambda: RevoluteJointBuilder((1.0, 0.0, 0.0)).local_anchor1((0.0, 0.0, 0.0)).local_anchor2((0.0, 2.0, 0.0))
    s.joints.insert(kin, dyn, jb())
    for oracle in (False, True):
        if oracle:
            w = oracle_lib.OracleWorld(s); api = w
        else:
            w = PhysicsWorld(s, _lib=emul_lib.lib()); w.reserve_joints(0, generic=True); api = w.physics_pipeline
        steps = 0
        while not w.sleeping()[dyn]:
            w.step(); steps += 1
            assert steps < 2000
        api.update_joints([0], [jb().motor_velocity(3, 2.0, 100.0).build_desc(kin, dyn)], wake_up=True)
        w.step()
        assert not w.sleeping()[dyn]
        moved = False
        for _ in range(50):
            w.step()
            moved = moved or float(np.linalg.norm(w.body_states()[1][dyn, 3:])) > 0.1
        assert moved

    s = joint_limits_scene()
    p = A.RbIntegrationParameters.default()
    p.warmstart_joints = 1
    w, o = PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib()), oracle_lib.OracleWorld(s, params=p)
    import copy
    descs = [copy.deepcopy(d) for d in s.joints.descs]
    motorised = [i for i, d in enumerate(descs) if d.motor_axes]
    limited = [i for i, d in enumerate(descs) if d.limit_axes]
    for i in range(120):
        if i % 9 == 4:
            j = motorised[(i // 9) % len(motorised)]
            ax = [a for a in range(6) if descs[j].motor_axes & (1 << a)][0]
            descs[j].motors[ax].target_vel = 1.5 - 0.5 * (i % 7)
            descs[j].motors[ax].target_pos = 0.1 * (i % 5)
            w.physics_pipeline.update_joints([j], [descs[j]]); o.update_joints([j], [descs[j]])
        if i % 14 == 7:
            j = limited[(i // 14) % len(limited)]
            ax = [a for a in range(6) if descs[j].limit_axes & (1 << a)][0]
            descs[j].limits[ax][1] = descs[j].limits[ax][1] + 0.05
            w.physics_pipeline.update_joints([j], [descs[j]], wake_up=False); o.update_joints([j], [descs[j]], wake_up=False)
        w.step(); o.step()
        if i % 10 == 9 or i % 9 == 4:
            d = compare_worlds(w, o)
            assert is_exact(d), (i, d)
            ji_w, ji_o = w.debug_read("joint_impulses", np.float32), o.debug_read("joint_impulses", np.float32)
            assert (ji_w.view(np.uint32) == ji_o.view(np.uint32)).all(), i


def test_physics_world_facade_joint_edits_emulated():
    """PhysicsWorld.insert_impulse_joint / remove_impulse_joint after the first step go through rb_world_insert_joints /
    rb_world_remove_joints (state of everything else untouched); without reserved capacity the insertion is refused loudly."""
    from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder, RopeJointBuilder
    from rapier_b200.world import RapierError
    def world(reserve):
        w = PhysicsWorld(_lib=emul_lib.lib())
        w.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(20.0, 0.5, 20.0))
        a = w.insert(RigidBodyBuilder.dynamic().translation((0.0, 3.0, 0.0)).can_sleep(False), ColliderBuilder.ball(0.3))
        b = w.insert(RigidBodyBuilder.dynamic().translation((1.0, 3.0, 0.0)).can_sleep(False), ColliderBuilder.ball(0.3))
        if reserve:
            w.reserve_joints(2, generic=True)
        w.step(5)
        return w, a, b
    w, a, b = world(True)
    before = w.body_states()[0][a].copy()
    j = w.insert_impulse_joint(a, b, RopeJointBuilder(1.2))
    assert (w.body_states()[0][a].view(np.uint32) == before.view(np.uint32)).all()      # nothing was re-uploaded
    w.set_body_states([b], vel6=[(3.0, 0.0, 0.0, 0.0, 0.0, 0.0)])
    w.step(60)
    pose = w.body_states()[0]
    assert np.linalg.norm(pose[a, :3] - pose[b, :3]) < 1.2 + 0.05                        # the rope holds
    w.remove_impulse_joint(j)
    w.set_body_states([b], vel6=[(4.0, 0.0, 0.0, 0.0, 0.0, 0.0)])
    w.step(60)
    pose = w.body_states()[0]
    assert np.linalg.norm(pose[a, :3] - pose[b, :3]) > 1.5                               # and no longer does once removed
    w, a, b = world(False)
    with pytest.raises(RapierError):
        w.insert_impulse_joint(a, b, RopeJointBuilder(1.2))


def test_dominance_groups_emulated_kernels():
    from test_oracle_kat import dominance_groups
    from variant_cases import dominance_parity_case
    dominance_groups(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))
    dominance_parity_case(lambda s, p=None: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib()),
                          lambda s, p=None: oracle_lib.OracleWorld(s, params=p))


def test_joint_warmstart_emulated_kernels():
    from test_oracle_kat import joint_warmstart
    from variant_cases import joint_limits_parity_case
    mk = lambda s, p=None: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib())
    mo = lambda s, p=None: oracle_lib.OracleWorld(s, params=p)
    joint_warmstart(mk)
    joint_limits_parity_case(mk, mo, warmstart_joints=True)
    joint_limits_parity_case(mk, mo, warmstart_joints=True, coulomb=True, steps=60)
    joint_limits_parity_case(mk, mo, warmstart_joints=True, scene=scenes.joint_grid(6), steps=60)   # locked-only joints on the generic path


def test_convex_polyhedra_emulated_kernels():
    from test_oracle_kat import convex_polyhedra
    convex_polyhedra(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))


def test_capsules_emulated_kernels():
    from test_oracle_kat import capsules_rest
    capsules_rest(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()))


def test_more_joint_known_answers_emulated_kernels():
    from test_oracle_kat import motor_position_with_rotating_base_stays_finite, prismatic_joint_stays_bounded_for_all_axis_rotations
    mk = lambda s, p: PhysicsWorld(s, integration_parameters=p, _lib=emul_lib.lib())
    prismatic_joint_stays_bounded_for_all_axis_rotations(mk)
    motor_position_with_rotating_base_stays_finite(mk)


def test_sleep_wake_scenarios_emulated_kernels():
    from test_oracle_kat import sleep_wake_scenarios
    def mk(s):
        w = PhysicsWorld(s, _lib=emul_lib.lib())
        w.reserve(32, 32)   # (totals: room for the body the impact scenario inserts)
        return w
    sleep_wake_scenarios(mk)


def test_quarantine_emulated_kernels():
    from test_oracle_kat import nan_force_is_quarantined
    nan_force_is_quarantined(lambda s: PhysicsWorld(s, _lib=emul_lib.lib()), expect_error=True)
