"""Island sharding (rapier_b200/sharding.py) against references written here from the definitions.

  * Halo sufficiency.  A scene is run single-process on the emulated kernels.  At every refresh the halo rule
    (sharding.halo_rule) is applied for each rank to the states, exactly as IslandShard applies it; after every step of
    the following window, the exact world AABB of every collider (float64, from body_states() and the collider
    descriptors, widened by prediction / 2 + contact skin as in test_broadphase_reference.py) is computed, and for every
    owned collider whose box overlaps a foreign body's collider box, that foreign body must be in the owner's halo.  A
    foreign body outside the halo is not in the broad phase at all: the two would pass through each other silently.
  * End-to-end runs on two gloo ranks (same harness as test_sharding_gloo.py): a scenario ends bit-identical to the
    single-process run when no contact crosses the shards, and with RB_ERR_SHARD (-6) when one does; which body types
    raise -6; a state edit that breaks the halo's bound is reported at the next refresh (HaloBoundError).
  * Connected components.  label_components() (the concurrent union-find of section_components, rb_collide.cuh) against
    scipy's connected_components over the edges the definition gives, read from the world's own tables: touching pairs
    (pair_keys / pair_nsc, collider -> parent) between two dynamic-or-kinematic bodies, not both kinematic, not involving a
    sensor, whatever their solver groups; and joints between two such bodies.  Each component is labelled with its
    smallest body index, fixed bodies -1.  partition_components must keep components whole, give ranks contiguous blocks
    of them and balance the body count.  Under -m gpu the same comparison runs at sizes where the union-find races.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import emul_lib
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder, SphericalJointBuilder
from rapier_b200.sharding import accel_bound, body_reach, halo_rule, partition_components
from rapier_b200.world import PhysicsWorld, RapierError
from test_broadphase_reference import collider_world_poses, reference_boxes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFRESH = 128
ZERO_G = (0.0, 0.0, 0.0)


# ---- scenarios ------------------------------------------------------------------------------------------------------
# Each returns (scene, owner [nb] or None for the partition, steps, drive(world, step) or None).  Hand-set owners: the
# fixed bodies -1, the rest 0 or 1.
def drop(gravity_scale=1.0, x=0.0):
    """A ball (rank 1) dropped from 4.5 m above a box (rank 0) resting on a fixed ground; gravity_scale < 0 mirrors the
    scene so that the ball falls up onto a box resting under a fixed ceiling.  x: the ball's horizontal offset."""
    s = scenes.Scene("drop", gravity=(0.0, -9.81, 0.0))
    sg = 1.0 if gravity_scale > 0 else -1.0
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5 * sg, 0.0)), ColliderBuilder.cuboid(20.0, 0.5, 20.0))
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.5 * sg, 0.0)).gravity_scale(gravity_scale), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((x, 5.0 * sg, 0.0)).gravity_scale(gravity_scale), ColliderBuilder.ball(0.5))
    return s, np.array([-1, 0, 1], np.int32), 2 * REFRESH, None


CUBE = np.array([[x, y, z] for x in (-2.0, 2.0) for y in (-2.0, 2.0) for z in (-2.0, 2.0)], np.float32)
CUBE_FACES = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
SLOW_SHAPES = {   # shape of the body approached, its extent along x, approach speed, starting surface gap along x
    "capsule_x": (lambda: ColliderBuilder.capsule_x(1.0, 1.0), 2.0, 0.01, 0.05),
    "capsule_y": (lambda: ColliderBuilder.capsule_y(1.0, 1.0), 1.0, 0.01, 0.05),
    "capsule_z": (lambda: ColliderBuilder.capsule_z(1.0, 1.0), 1.0, 0.01, 0.05),
    "sharp_hull": (lambda: ColliderBuilder.convex_mesh(CUBE, CUBE_FACES), 2.0, 0.1, 0.3),
    "round_hull": (lambda: ColliderBuilder.convex_mesh(CUBE, CUBE_FACES, border_radius=0.5), 2.5, 0.1, 0.3),
}


def slow_approach(shape):
    """A ball (rank 1) drifting along -x toward a body of the given shape (rank 0), no gravity.  Neither may sleep: the
    slowest drifts are below the sleep threshold."""
    make, ext, v, gap = SLOW_SHAPES[shape]
    s = scenes.Scene("slow_" + shape, gravity=ZERO_G)
    s.insert(RigidBodyBuilder.dynamic().can_sleep(False), make())
    s.insert(RigidBodyBuilder.dynamic().can_sleep(False).translation((ext + gap + 0.5, 0.0, 0.0)).linvel((-v, 0.0, 0.0)),
             ColliderBuilder.ball(0.5))
    return s, np.array([0, 1], np.int32), 2 * REFRESH, None


def user_force():
    """A ball (rank 1) at rest 4 m from a box (rank 0), pushed toward it by a constant user force of 2 m/s^2: it covers
    the 4 m within the first window (4.55 m in 128 steps), which a margin computed from the speeds at rest does not."""
    s = scenes.Scene("user_force", gravity=ZERO_G)
    s.insert(RigidBodyBuilder.dynamic(), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((5.0, 0.0, 0.0)), ColliderBuilder.ball(0.5))

    def drive(w, k):
        if k == 0:
            m = 1.0 / w.debug_read("body_mprops", np.float32).reshape(-1, 16)[1, 3]
            w.set_body_forces([1], [[-2.0 * m, 0.0, 0.0]])
    return s, np.array([0, 1], np.int32), 2 * REFRESH, drive


def spinning_compound():
    """A compound (rank 1) of a heavy ball 2 m off its origin and a light ball at its origin, so that its centre of mass is
    2 m off the origin, spinning at 3 rad/s about z.  Half a turn later the light ball is 4 m from where the origin was,
    and reaches a box (rank 0) that a sphere about the origin holding both balls never came near."""
    s = scenes.Scene("spinning_compound", gravity=ZERO_G)
    s.insert(RigidBodyBuilder.dynamic().translation((5.0, 0.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    h = s.insert(RigidBodyBuilder.dynamic().angvel((0.0, 0.0, 3.0)), ColliderBuilder.ball(0.5).translation((2.0, 0.0, 0.0)).density(1000.0))
    s.colliders.insert_with_parent(ColliderBuilder.ball(0.5).density(0.001), h)
    return s, np.array([0, 1], np.int32), 2 * REFRESH, None


def kinematic_drive():
    """A position-based kinematic box (rank 0) moved 3 m/s toward a ball at rest (rank 1), a target every step."""
    s = scenes.Scene("kinematic_drive", gravity=ZERO_G)
    s.insert(RigidBodyBuilder.kinematic_position_based().linvel((3.0, 0.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((9.0, 0.0, 0.0)), ColliderBuilder.ball(0.5))

    def drive(w, k):
        w.set_next_kinematic_positions([0], [[3.0 * (k + 1) * w.integration_parameters.dt, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]])
    return s, np.array([0, 1], np.int32), 2 * REFRESH, drive


def near_miss():
    """A ball (rank 1) passing a box (rank 0) at 5 m/s, 0.3 m from it, without touching; no gravity."""
    s = scenes.Scene("near_miss", gravity=ZERO_G)
    s.insert(RigidBodyBuilder.dynamic(), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((8.0, 1.3, 0.0)).linvel((-5.0, 0.0, 0.0)), ColliderBuilder.ball(0.5))
    return s, np.array([0, 1], np.int32), 2 * REFRESH, None


def land_beside():
    """A ball (rank 1) dropped onto the fixed ground 0.3 m beside a box (rank 0) resting there."""
    s, owner, steps, _ = drop(x=1.3)
    return s, owner, steps, None


def kinematic_platform():
    """A box (rank 1) dropped onto a resting position-based kinematic platform (rank 0) after the partition."""
    s = scenes.Scene("kinematic_platform", gravity=(0.0, -9.81, 0.0))
    s.insert(RigidBodyBuilder.kinematic_position_based(), ColliderBuilder.cuboid(2.0, 0.25, 2.0))
    s.insert(RigidBodyBuilder.dynamic().translation((0.3, 3.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    return s, np.array([0, 1], np.int32), 2 * REFRESH, None


HALO_CASES = {
    "drop": lambda: drop(),
    "drop_gravity_scale_2": lambda: drop(2.0),
    "drop_gravity_scale_minus_1": lambda: drop(-1.0),
    **{"slow_" + k: (lambda k=k: slow_approach(k)) for k in SLOW_SHAPES},
    "user_force": user_force,
    "spinning_compound": spinning_compound,
    "kinematic_drive": kinematic_drive,
    "near_miss": near_miss,
    "land_beside": land_beside,
    "kinematic_platform": kinematic_platform,
}


# ---- 1(a): halo sufficiency against the float64 broad-phase boxes ----------------------------------------------------
def collider_table(pipe, n):
    return np.ctypeslib.as_array(pipe._c)[:n]


def run_halo_reference(scene, owner, steps, drive, refresh=REFRESH):
    """Single-process run; returns the (step, rank, owned collider, foreign body) overlaps the halo missed, and the number
    of overlapping (step, rank, owned collider, foreign collider) found."""
    w = PhysicsWorld(scene, _lib=emul_lib.lib())
    w._flush()
    pipe = w.physics_pipeline
    tab = collider_table(pipe, len(scene.colliders))
    hulls = scene.colliders.hulls
    com, reach = (torch.from_numpy(a) for a in body_reach(pipe))
    owner_t = torch.from_numpy(owner.astype(np.int64))
    moving = np.nonzero(owner >= 0)[0]
    inv_mass = w.debug_read("body_mprops", np.float32).reshape(-1, 16)[moving, 3].astype(np.float64)
    gscale = np.array([d.gravity_scale for d in scene.bodies.descs], np.float64)[moving]
    cowner = np.where(tab["parent"] >= 0, owner[np.maximum(tab["parent"], 0)], -1)
    dt = w.integration_parameters.dt
    missed, overlaps = [], 0
    for k in range(steps):
        if drive is not None:
            drive(w, k)
        if k % refresh == 0:
            pose, vel = w.body_states()
            state = torch.from_numpy(np.concatenate([pose, vel], axis=1))
            acc = accel_bound(pipe.gravity, gscale, pipe.user_force[moving], inv_mass)
            halos = [halo_rule(state, com, reach, owner_t, r, refresh * dt, acc).numpy() for r in (0, 1)]
        w.step()
        pose, _ = w.body_states()
        R, t = collider_world_poses(tab, pose)
        lo, hi, _ = reference_boxes(tab, hulls, R, t)
        for r in (0, 1):
            a = np.nonzero(cowner == r)[0]
            b = np.nonzero((cowner >= 0) & (cowner != r))[0]
            ov = ((lo[a, None] <= hi[None, b]) & (lo[None, b] <= hi[a, None])).all(-1)
            overlaps += int(ov.sum())
            for i, j in zip(*np.nonzero(ov)):
                fb = int(tab["parent"][b[j]])
                if not halos[r][fb]:
                    missed.append((k, r, int(a[i]), fb))
    return missed, overlaps


@pytest.mark.parametrize("case", sorted(HALO_CASES))
def test_halo_covers_every_reachable_body(case):
    scene, owner, steps, drive = HALO_CASES[case]()
    missed, overlaps = run_halo_reference(scene, owner, steps, drive)
    assert not missed, f"{case}: foreign bodies within broad-phase reach but not in the halo (step, rank, collider, body): {missed[:6]}"
    if case not in ("near_miss", "land_beside"):   # (these two pass 0.3 m apart by design)
        assert overlaps, f"{case}: the bodies never come within broad-phase reach: the case checks nothing"


def test_reach_uses_the_true_shape_extent():
    """body_reach about the centre of mass: ball r, cuboid |h|, capsule half height + r, hull max |v| + border radius,
    plus the collider's offset from the centre of mass, the contact skin, the prediction distance and the fat skin."""
    s = scenes.Scene("reach", gravity=ZERO_G)
    s.insert(RigidBodyBuilder.dynamic(), ColliderBuilder.ball(1.0))
    s.insert(RigidBodyBuilder.dynamic().translation((10.0, 0.0, 0.0)), ColliderBuilder.cuboid(1.0, 2.0, 2.0))
    for k, mk in enumerate((ColliderBuilder.capsule_x, ColliderBuilder.capsule_y, ColliderBuilder.capsule_z)):
        s.insert(RigidBodyBuilder.dynamic().translation((20.0 + 10 * k, 0.0, 0.0)), mk(1.0, 0.3))
    s.insert(RigidBodyBuilder.dynamic().translation((60.0, 0.0, 0.0)), ColliderBuilder.convex_mesh(CUBE, CUBE_FACES))
    s.insert(RigidBodyBuilder.dynamic().translation((70.0, 0.0, 0.0)), ColliderBuilder.convex_mesh(CUBE, CUBE_FACES, border_radius=0.5))
    h = s.insert(RigidBodyBuilder.dynamic().translation((80.0, 0.0, 0.0)), ColliderBuilder.ball(0.5).translation((2.0, 0.0, 0.0)))
    s.colliders.insert_with_parent(ColliderBuilder.ball(0.5).translation((-2.0, 0.0, 0.0)).density(3.0), h)
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w._flush()
    com, reach = body_reach(w.physics_pipeline)
    pad = 0.02 + 0.04 + s.colliders.descs[0].contact_skin
    expect = [1.0, 3.0, 1.3, 1.3, 1.3, np.sqrt(12.0), np.sqrt(12.0) + 0.5, 3.0 + 0.5]   # compound: com at x = -1
    np.testing.assert_allclose(com[7], [-1.0, 0.0, 0.0], atol=1e-5)
    np.testing.assert_allclose(reach, np.array(expect) + pad, rtol=1e-5)


def test_gravity_term_is_per_axis_and_bench_halo_is_empty():
    """b3d_many_pyramids_80x20 with 2, 4 and 8 replicas splits ranks along z, 13.9 m between pyramid rows, gravity along
    y: applied to the initial states, the halo rule leaves every rank's halo empty (no per-step collective)."""
    for replicas in (2, 4, 8):
        scene = scenes.pyramids(8 * replicas, 10, 20, name="b3d_many_pyramids_80x20")
        w = PhysicsWorld(scene, _lib=emul_lib.lib())
        w._flush()
        pipe = w.physics_pipeline
        owner = partition_components(pipe.label_components(), replicas)
        assert sorted(set(owner.tolist()) - {-1}) == list(range(replicas))
        com, reach = (torch.from_numpy(a) for a in body_reach(pipe))
        pose, vel = pipe.body_states()
        state = torch.from_numpy(np.concatenate([pose, vel], axis=1))
        moving = np.nonzero(owner >= 0)[0]
        inv_mass = pipe.debug_read("body_mprops", np.float32).reshape(-1, 16)[moving, 3].astype(np.float64)
        acc = accel_bound(pipe.gravity, np.ones(len(moving)), pipe.user_force[moving], inv_mass)
        assert acc[0] == 0.0 and acc[2] == 0.0 and acc[1] > 9.0
        owner_t = torch.from_numpy(owner.astype(np.int64))
        for r in range(replicas):
            halo = halo_rule(state, com, reach, owner_t, r, REFRESH * pipe.params.dt, acc)
            assert not halo.any(), f"{replicas} replicas: rank {r} tracks {int(halo.sum())} bodies"


# ---- 1(b), 1(c): two gloo ranks -------------------------------------------------------------------------------------
WORKER = r'''
import os, sys, datetime
sys.path.insert(0, {root!r}); sys.path.insert(0, os.path.join({root!r}, "tests"))
import numpy as np, torch, torch.distributed as dist
import emul_lib
import test_sharding_reference as T
from rapier_b200.world import PhysicsWorld
from rapier_b200.sharding import IslandShard
dist.init_process_group("gloo", timeout=datetime.timedelta(seconds=120))
rank, ws = dist.get_rank(), dist.get_world_size()
scene, owner, steps, drive = T.{make}
w = PhysicsWorld(scene, _lib=emul_lib.lib()); w._flush()
shard = IslandShard(w.physics_pipeline, dist, rank, ws, torch.device("cpu"), refresh_every={refresh!r})
if owner is not None:
    assert (shard.owner == owner).all(), (shard.owner, owner)
err = ""
try:
    for k in range(steps):
        if drive is not None:
            drive(w, k, rank, shard)
        w.step()
        shard.exchange()
    shard.finish()
except Exception as e:
    err = f"{{type(e).__name__}}: {{e}}"
pose, vel = w.body_states()
np.save({out!r} + f"_{{rank}}.npy", np.concatenate([pose, vel], axis=1))
with open({out!r} + f"_{{rank}}.txt", "w") as f:
    f.write(f"{{err}}\n{{shard.halo_steps}}\n")
if not err:
    dist.destroy_process_group()
'''


def _free_port():
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_gloo(tmp_path, make, refresh=REFRESH):
    """Runs `T.<make>` on two gloo ranks; returns per rank (final state [nb, 13], error text, halo steps)."""
    out = str(tmp_path / "state")
    script = tmp_path / "worker.py"
    script.write_text(WORKER.format(root=ROOT, out=out, make=make, refresh=refresh))
    port = str(_free_port())
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=port)
    subprocess.check_call([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
                           "--master-port", port, str(script)], env=env, timeout=600)
    res = []
    for r in range(2):
        err, halo_steps = open(out + f"_{r}.txt").read().split("\n")[:2]
        res.append((np.load(out + f"_{r}.npy"), err, int(halo_steps)))
    return res


def gloo_case(name):
    """HALO_CASES[name] with the partition's owners and a drive(world, step, rank, shard)."""
    scene, owner, steps, drive = HALO_CASES[name]()
    return scene, owner, steps, (None if drive is None else lambda w, k, rank, shard: drive(w, k))


def single_process(name):
    scene, _, steps, drive = HALO_CASES[name]()
    w = PhysicsWorld(scene, _lib=emul_lib.lib())
    for k in range(steps):
        if drive is not None:
            drive(w, k)
        w.step()
    pose, vel = w.body_states()
    return np.concatenate([pose, vel], axis=1)


@pytest.mark.parametrize("name,halo", [("near_miss", True), ("land_beside", True)])
def test_sharded_run_without_cross_shard_contact_is_bit_identical(tmp_path, name, halo):
    """No contact crosses the shards: after finish() both ranks hold the single-process result bit for bit."""
    expect = single_process(name)
    for r, (got, err, halo_steps) in enumerate(run_gloo(tmp_path, f"gloo_case({name!r})")):
        assert not err, f"rank {r}: {err}"
        assert (halo_steps > 0) == halo, (r, halo_steps)
        assert (got.view(np.uint32) == expect.view(np.uint32)).all(), f"rank {r} differs from the single-process run"


@pytest.mark.parametrize("kind", ["emulated", pytest.param("cuda", marks=pytest.mark.gpu)])
@pytest.mark.parametrize("name", ["land_beside", "drop"])
def test_label_components_does_not_change_the_run(request, kind, name):
    """label_components() is a query: a run with a call before the first step (as IslandShard makes) and every 20 steps
    is bit-identical to a run without, and its bodies fall asleep at the same steps."""
    if kind == "cuda":
        request.getfixturevalue("built")

    def run(query):
        scene, _, steps, _ = HALO_CASES[name]()
        w = PhysicsWorld(scene, _lib=emul_lib.lib() if kind == "emulated" else None)
        w._flush()
        asleep = []
        for k in range(steps):
            if query and k % 20 == 0:
                w.physics_pipeline.label_components()
            w.step()
            asleep.append(w.sleeping().copy())
        pose, vel = w.body_states()
        return np.concatenate([pose, vel], axis=1), np.array(asleep)
    a, sa = run(False)
    b, sb = run(True)
    assert sa.any(), "the case should put a body to sleep"
    assert (sa == sb).all(), f"sleep differs from step {int(np.nonzero((sa != sb).any(1))[0][0])} on"
    assert (a.view(np.uint32) == b.view(np.uint32)).all()


def test_sharded_landing_on_another_ranks_kinematic_platform(tmp_path):
    """The box's owner solves the contact against the platform's imported state; the platform's owner forms no pair with
    the box.  Neither rank raises, and both end with the same states, the box at rest on the platform.  The run is not
    bit-identical to the single-process one: there the platform joins the box's island (kinematic bodies are island
    members, DESIGN.md section 6), here it cannot, so sleeping and the solve's grouping differ."""
    res = run_gloo(tmp_path, "gloo_case('kinematic_platform')")
    for r, (got, err, halo_steps) in enumerate(res):
        assert not err, f"rank {r}: {err}"
        assert halo_steps > 0
    assert (res[0][0].view(np.uint32) == res[1][0].view(np.uint32)).all()
    box = res[0][0][1]
    assert abs(box[1] - 0.75) < 0.01 and np.abs(box[7:13]).max() < 0.05, box
    expect = single_process("kinematic_platform")
    assert np.abs(box[:3] - expect[1, :3]).max() < 1e-3


def test_sharded_drop_onto_another_ranks_body_raises(tmp_path):
    """The ball (rank 1) lands on the box (rank 0): the contact with the other rank's dynamic body raises RB_ERR_SHARD
    instead of simulating the two islands apart.  The first rank to raise leaves, so the other one may instead lose its
    peer in the next collective; neither finishes the run."""
    res = run_gloo(tmp_path, "gloo_case('drop')")
    errs = [err for _, err, _ in res]
    assert any("RapierError" in e and "-6" in e for e in errs), errs
    assert all(("RapierError" in e and "-6" in e) or "Connection closed" in e for e in errs), errs
    assert all(halo_steps > 0 for _, _, halo_steps in res)


def violation_case():
    """Two boxes 20 m apart on x, no gravity, one per rank.  At step 48 the owner of box 1 throws it at 75 m/s toward box 0:
    it crosses the 20 m in 16 steps, far beyond what the margin computed at rest bounds, and is inside box 0 (which
    neither rank tracks) at the refresh at step 64."""
    s = scenes.Scene("violation", gravity=ZERO_G)
    s.insert(RigidBodyBuilder.dynamic(), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((20.0, 0.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))

    def drive(w, k, rank, shard):
        if k == 48 and rank == 1:
            w.set_body_states([1], vel6=[[-75.0, 0.0, 0.0, 0.0, 0.0, 0.0]])
    return s, np.array([0, 1], np.int32), 64, drive


def test_bound_broken_by_a_state_edit_is_reported_at_refresh(tmp_path):
    for r, (_, err, halo_steps) in enumerate(run_gloo(tmp_path, "violation_case()", refresh=32)):
        assert err.startswith("HaloBoundError") and "body 1 " in err and "rank 0" in err, f"rank {r}: {err!r}"
        assert halo_steps == 0


def _two_body_world(owned_type, halo_type, gap=0.0):
    """An owned body of type owned_type resting on (touching) a halo body of type halo_type, set up as a rank sees them."""
    make = {"dynamic": RigidBodyBuilder.dynamic, "kinematic": RigidBodyBuilder.kinematic_position_based, "fixed": RigidBodyBuilder.fixed}
    s = scenes.Scene("two_types", gravity=(0.0, -9.81, 0.0))
    s.insert(make[halo_type]().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(2.0, 0.5, 2.0))
    s.insert(make[owned_type]().translation((0.0, 0.5 + gap, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w._flush()
    pipe = w.physics_pipeline
    pipe.set_owned_bodies(np.array([0, 1], np.uint8))
    pipe.set_halo_bodies(np.array([1, 0], np.uint8).ctypes.data)
    return w


@pytest.mark.parametrize("halo_type,raises", [("dynamic", True), ("kinematic", False), ("fixed", False)])
def test_shard_error_by_body_type(halo_type, raises):
    """-6 is raised on the side that owns a dynamic body touching a dynamic halo body, not for a halo kinematic or fixed one
    (their motion does not depend on the contact, so the owner solves it right)."""
    w = _two_body_world("dynamic", halo_type)
    if raises:
        with pytest.raises(RapierError, match="-6"):
            for _ in range(30):
                w.step()
    else:
        for _ in range(30):
            w.step()
        assert w.contact_pairs()["num_contacts"].max() > 0


def test_kinematic_platform_of_another_rank():
    """A dynamic body resting on another rank's kinematic platform (they met after the partition).  The rank owning the
    dynamic body solves the contact against the platform's imported state without error.  The rank owning the platform
    forms no pair at all: the broad phase pairs only colliders of which one belongs to an owned dynamic body, and the
    platform's motion does not depend on the contact.  Both ranks agree: no error, and the result is the single-process
    one (DESIGN.md section 6)."""
    w = _two_body_world("dynamic", "kinematic")
    for _ in range(30):
        w.step()
    assert w.contact_pairs()["num_contacts"].max() > 0
    w = _two_body_world("kinematic", "dynamic")
    for _ in range(30):
        w.step()
    assert len(w.contact_pairs()["num_contacts"]) == 0


# ---- 1(d): connected components against a graph reference ------------------------------------------------------------
def reference_components(w, scene):
    """Labels from scipy over the edges of the module docstring, read from the world's tables after label_components'
    collision pass."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    nb = len(scene.bodies)
    btype = np.array([d.body_type for d in scene.bodies.descs], np.int32)
    solver = np.isin(btype, [A.RB_BODY_DYNAMIC, A.RB_BODY_KINEMATIC_POSITION_BASED, A.RB_BODY_KINEMATIC_VELOCITY_BASED])
    parent = np.array([d.parent for d in scene.colliders.descs], np.int64)
    sensor = np.array([d.sensor for d in scene.colliders.descs], bool)
    keys = w.debug_read("pair_keys", np.uint64)
    nsc = w.debug_read("pair_nsc", np.int32)
    c1, c2 = (keys >> np.uint64(32)).astype(np.int64), (keys & np.uint64(0xffffffff)).astype(np.int64)
    b1, b2 = parent[c1], parent[c2]
    ok = (nsc > 0) & (b1 >= 0) & (b2 >= 0) & ~sensor[c1] & ~sensor[c2]
    ok &= solver[np.maximum(b1, 0)] & solver[np.maximum(b2, 0)]
    ok &= (btype[np.maximum(b1, 0)] == A.RB_BODY_DYNAMIC) | (btype[np.maximum(b2, 0)] == A.RB_BODY_DYNAMIC)
    j = np.array([(d.body1, d.body2) for d in scene.joints.descs], np.int64).reshape(-1, 2)
    j = j[solver[j[:, 0]] & solver[j[:, 1]]] if len(j) else j
    e1 = np.concatenate([b1[ok], j[:, 0]])
    e2 = np.concatenate([b2[ok], j[:, 1]])
    _, lab = connected_components(coo_matrix((np.ones(len(e1)), (e1, e2)), shape=(nb, nb)), directed=False)
    smallest = np.full(lab.max() + 1, nb, np.int64)
    np.minimum.at(smallest, lab, np.arange(nb))
    out = smallest[lab].astype(np.int32)
    out[~solver] = -1
    return out, int(ok.sum()), len(j)


def check_components(w, scene, world_sizes=(2, 3, 4)):
    got = w.physics_pipeline.label_components()
    expect, npairs, njoints = reference_components(w, scene)
    bad = np.nonzero(got != expect)[0]
    assert not len(bad), f"{scene.name}: label_components differs at {len(bad)} bodies, e.g. {[(int(b), int(got[b]), int(expect[b])) for b in bad[:6]]}"
    for ws in world_sizes:
        check_partition(expect, partition_components(got, ws), ws)
    return npairs, njoints


def check_partition(comp, owner, ws):
    assert ((owner == -1) == (comp == -1)).all()
    roots, inv, counts = np.unique(comp[comp >= 0], return_inverse=True, return_counts=True)
    own = owner[comp >= 0]
    first = np.zeros(len(roots), np.int64)
    first[inv] = own
    assert (own == first[inv]).all(), "a component is split across ranks"
    assert (np.diff(first) >= 0).all(), "ranks do not take contiguous blocks of components in root order"
    total, biggest = counts.sum(), counts.max()
    per_rank = np.bincount(own, minlength=ws)
    assert (np.abs(per_rank - total / ws) <= biggest).all(), (per_rank, total / ws, biggest)


def components_scene():
    """Sleeping stacks, a kinematic platform carrying boxes, a joint chain listed in shuffled order, a pair whose solver
    groups fail (still an edge), a pair whose collision groups fail (no pair), a sensor across two boxes (no edge)."""
    s = scenes.Scene("components", gravity=(0.0, -9.81, 0.0))
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(60.0, 0.5, 60.0))
    for x in (-20.0, -16.0):                      # stacks that fall asleep
        for k in range(3):
            s.insert(RigidBodyBuilder.dynamic().translation((x, 0.5 + k, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((-8.0, 1.0, 0.0)), ColliderBuilder.cuboid(2.0, 0.25, 2.0))
    for x in (-9.0, -7.0):                        # carried by the platform
        s.insert(RigidBodyBuilder.dynamic().translation((x, 1.75, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((-8.0, 4.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((-7.0, 4.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    rng = np.random.default_rng(3)
    links = []
    for k in rng.permutation(12):                 # a hanging chain whose links are inserted in shuffled order
        links.append((k, s.insert(RigidBodyBuilder.dynamic().translation((0.0, 10.0 - 0.5 * k, 5.0)), ColliderBuilder.ball(0.2))))
    link = dict(links)
    for k in range(11):
        s.joints.insert(link[k], link[k + 1], SphericalJointBuilder().local_anchor1((0.0, -0.25, 0.0)).local_anchor2((0.0, 0.25, 0.0)))
    s.insert(RigidBodyBuilder.dynamic().translation((8.0, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5).solver_groups(1, 2))
    s.insert(RigidBodyBuilder.dynamic().translation((8.0, 1.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5).solver_groups(1, 2))
    s.insert(RigidBodyBuilder.dynamic().translation((12.0, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5).collision_groups(1, 1))
    s.insert(RigidBodyBuilder.dynamic().translation((12.0, 1.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5).collision_groups(2, 2))
    s.insert(RigidBodyBuilder.dynamic().translation((16.0, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((17.5, 0.5, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.dynamic().translation((16.75, 1.5, 0.0)), ColliderBuilder.cuboid(1.5, 0.5, 0.5).sensor())
    return s


def test_components_match_graph_reference():
    s = components_scene()
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w.step(90)
    assert w.sleeping()[1:4].all(), "the stacks should be asleep"
    npairs, njoints = check_components(w, s)
    assert npairs >= 7 and njoints == 11
    lab = w.physics_pipeline.label_components()
    assert lab[1] == lab[3] and lab[1] != lab[4], "each sleeping stack is one component"


def test_check_partition_rejects_split_and_unbalanced():
    comp = np.array([-1, 1, 1, 3, 3, 3, 6])
    check_partition(comp, partition_components(comp, 2), 2)
    with pytest.raises(AssertionError):
        check_partition(comp, np.array([-1, 0, 1, 1, 1, 1, 1]), 2)
    with pytest.raises(AssertionError):
        check_partition(comp, np.array([-1, 1, 1, 0, 0, 0, 1]), 2)


def box_row(n):
    """n unit boxes along x, each touching the next face to face, inserted in shuffled order; no gravity."""
    s = scenes.Scene(f"box_row_{n}", gravity=ZERO_G)
    for k in np.random.default_rng(1).permutation(n):
        s.insert(RigidBodyBuilder.dynamic().translation((float(k), 0.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    return s


def joint_chain(n):
    """n balls 1 m apart, far from each other's reach, linked in a chain of spherical joints listed in shuffled order."""
    s = scenes.Scene(f"joint_chain_{n}", gravity=ZERO_G)
    rng = np.random.default_rng(2)
    place = rng.permutation(n)
    for k in range(n):
        s.insert(RigidBodyBuilder.dynamic().translation((float(place[k] % 100) * 3.0, 0.0, float(place[k] // 100) * 3.0)), ColliderBuilder.ball(0.5))
    order = np.argsort(place)      # body at chain position p
    for e in rng.permutation(n - 1):
        s.joints.insert(int(order[e]), int(order[e + 1]), SphericalJointBuilder().local_anchor1((1.5, 0.0, 0.0)).local_anchor2((-1.5, 0.0, 0.0)))
    return s


def random_clusters(n, seed=4):
    """n balls in clusters of 1..40 touching neighbours laid along x, clusters 2 m apart on a grid, inserted in random order."""
    rng = np.random.default_rng(seed)
    pos = []
    row, x = 0, 0.0
    while len(pos) < n:
        m = int(min(rng.integers(1, 41), n - len(pos)))
        pos += [(x + k * 1.0, 0.0, row * 3.0) for k in range(m)]
        x += m + 2.0
        if x > 300.0:
            row, x = row + 1, 0.0
    s = scenes.Scene(f"random_clusters_{n}", gravity=ZERO_G)
    for k in rng.permutation(n):
        s.insert(RigidBodyBuilder.dynamic().translation(pos[k]), ColliderBuilder.ball(0.5))
    return s


@pytest.mark.parametrize("make,n", [(box_row, 300), (joint_chain, 300), (random_clusters, 2000)], ids=["box_row", "joint_chain", "random_clusters"])
def test_components_at_small_sizes(make, n):
    s = make(n)
    w = PhysicsWorld(s, _lib=emul_lib.lib())
    w._flush()
    npairs, njoints = check_components(w, s)
    assert npairs + njoints > n // 2


@pytest.mark.gpu
@pytest.mark.parametrize("make,n", [(box_row, 10_000), (joint_chain, 10_000), (random_clusters, 100_000)], ids=["box_row", "joint_chain", "random_clusters"])
def test_components_at_device_sizes(built, make, n):
    s = make(n)
    w = PhysicsWorld(s, device=0)
    w._flush()
    npairs, njoints = check_components(w, s, world_sizes=(2, 8))
    lab = w.physics_pipeline.label_components()
    if make is not random_clusters:
        assert (lab == lab[0]).all() and lab[0] == 0, "one component labelled 0 expected"
    assert npairs + njoints > n // 2
