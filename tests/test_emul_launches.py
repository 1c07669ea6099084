"""The host emulation (tests/emul, -DRB_EMULATE) runs the host's step sequence through the same launcher as the device,
one CTA of one thread per launch: its kernels_launched counts are the ones the device branch of rb_world_step launches."""
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.world import PhysicsWorld

import emul_lib
from variant_cases import substep_groups_scene


def _launches_per_step(scene, params=None, steps=4):
    w = PhysicsWorld(scene, integration_parameters=params, _lib=emul_lib.lib())
    out = []
    for _ in range(steps):
        k0 = w.counters()["kernels_launched"]
        w.step()
        out.append(w.counters()["kernels_launched"] - k0)
    return out


def test_emulated_step_launches_the_device_sequence():
    """k_collide and k_solve_coop per step; a grid-wide island (joint_grid(18): 306 bodies) is solved inside k_collide until
    the host's one-step-old hint shows it, then by k_solve_large; the general path launches k_solve_items_x and
    k_solve_large_x once per substep solve-group."""
    assert _launches_per_step(scenes.pyramids(2, 2, 6)) == [2, 2, 2, 2]
    assert _launches_per_step(scenes.joint_grid(18)) == [2, 2, 3, 3]
    coulomb = A.RbIntegrationParameters.default()
    coulomb.friction_model = 1
    assert _launches_per_step(scenes.pyramids(2, 2, 6), coulomb) == [3, 3, 3, 3]
    s = substep_groups_scene()
    keys = {(d.flags >> A.RB_BODY_EXTRA_ITERS_SHIFT) & 0xFF for d in s.bodies.descs} | {0}
    assert len(keys) == 4
    no_ccd = A.RbIntegrationParameters.default()
    no_ccd.max_ccd_substeps = 0   # (this scene queues CCD clamps: each synchronising call would add a k_ccd_pending)
    assert _launches_per_step(s, no_ccd) == [1 + 2 * len(keys)] * 4
