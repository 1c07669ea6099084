"""Warm start of streamed shared-memory items (constant rows read from the L2 pool, body by body) against the oracle,
in the host emulation of the kernels: an island whose adjacency lists span many staging chunks, with one body that has
more contacts than a chunk holds, warm-started and with warmstart_coefficient = 0 (impulses banked, not applied)."""
import numpy as np
import pytest

import emul_lib
import oracle_lib
from parity_util import compare_worlds, is_exact
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder
from rapier_b200.world import PhysicsWorld

SMEM_FLOATS = 5600   # streams the island below in chunks of 9 slots (see chunk_slots)


def chunk_slots(smem_floats, nb, n):
    """Slots per staging chunk of a streamed item of nb bodies and n constraints (coop_plan in rb_solver.cuh)."""
    body_floats = (nb + 2) * 28            # SB_STRIDE floats per staged body, + world pseudo body + garbage slot
    avail = (smem_floats - body_floats) // 4 - 5 * (n | 1)   # float4 left after the 5 mutable rows per constraint
    rows = avail // 36                     # COOP_ROWS constant float4 rows per constraint
    return (rows // 2 - 1) | 1


def slab_scene():
    """A dynamic slab on the ground carrying a 5 x 5 grid of two-box stacks: the slab touches 26 constraints (25
    boxes + the ground), each of its own colour; the 25 box-on-box contacts share one colour stage."""
    s = scenes.Scene("slab_with_stacks", gravity=(0.0, -9.81, 0.0))
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(20.0, 0.5, 20.0))
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.25, 0.0)), ColliderBuilder.cuboid(3.0, 0.25, 3.0))
    for i in range(5):
        for k in range(5):
            for level in range(2):
                s.insert(RigidBodyBuilder.dynamic().translation((i - 2.0, 0.75 + 0.5 * level, k - 2.0)), ColliderBuilder.cuboid(0.25, 0.25, 0.25))
    return s


@pytest.mark.parametrize("warmstart", [1.0, 0.0], ids=["warm", "bank_only"])
def test_streamed_warm_start_over_many_chunks_matches_oracle(monkeypatch, warmstart):
    monkeypatch.setenv("RB_EMU_COOP_SMEM_FLOATS", str(SMEM_FLOATS))
    scene = slab_scene()
    p = A.RbIntegrationParameters.default()
    p.warmstart_coefficient = warmstart
    w = PhysicsWorld(scene, integration_parameters=p, _lib=emul_lib.lib())
    o = oracle_lib.OracleWorld(scene, params=p)
    for i in range(20):
        w.step()
        o.step()
        d = compare_worlds(w, o)
        assert is_exact(d), f"step {i}: {d}"
    c = w.counters()
    nb, n = 51, 51
    assert c["num_active_manifolds"] == n, "slab-ground, 25 box-slab and 25 box-box contacts"
    assert chunk_slots(SMEM_FLOATS, nb, n) < 26, "the slab must have more contacts than one chunk holds"
    st = w.debug_read("state", np.int32)
    assert st[19] == 1, "the island must have taken the streaming path"
