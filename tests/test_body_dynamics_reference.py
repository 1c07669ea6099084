"""The body phases of the solve (rb_solver.cuh: update_world_mass, body_init, body_increment, body_integrate,
body_writeback) against a float64 restatement, and the linear momentum balance and impulse bounds of the constraint solve,
on the oracle, the emulated kernels and, under -m gpu, the CUDA library (numpy only).

Free-body step (bodies without contacts), restated in float64 from the integration parameters and the body's mass
properties as the library reports them (body_mprops / body_mframe, pinned against geometry by
test_mass_properties_reference.py).  With n = num_solver_iterations + the body's additional_solver_iterations substeps
of h = dt / n, the step runs on the centre-of-mass frame (t_c = t + R lcom):
  * velocity increments, frozen at the start of the step: dv = (F + g m s_g) / m h on free axes, dw = I_w^-1 tau h with
    the world inverse inertia I_w^-1 = R R_f diag(ipi) R_f^T R^T of the pose before the step (zero for non-dynamic bodies);
  * per substep: v += dv, w += dw; the gyroscopic correction (rigid_body.rs:2023-2046) for dynamic bodies with gyroscopic
    forces: w_l = A^T w, L = I w_l, L' = L - (w_l x L) h rescaled to |L|, w = A I^-1 L' (A = R R_f);
  * the caps: |v| <= max_lin_vel, |w| <= pi/4 / dt unless the body allows fast rotation;
  * q <- normalize((w h/2, 1) q), t_c <- t_c + v h: the linearised step, so the angle per substep of a spin about a
    principal axis is 2 atan(|w| h / 2), not |w| h;
  * writeback: v /= 1 + dt d_lin, w /= 1 + dt d_ang, t = t_c - R lcom.
Tolerance: with N the substeps run so far and S the magnitude of the compared quantity plus its rate times the elapsed
time, every component must lie within TOL_FREE * N * u * S (u = 2^-24, TOL_FREE = 16) of the reference.  Largest
ratio seen err / (N u S), oracle and emulated kernels: 3.1.

Linear momentum balance: every contact, friction and joint impulse acts equal and opposite on its two bodies through
their inverse masses (m1 im1 = m2 im2 = 1 up to the float32 reciprocal), so in a world of dynamic bodies only (no
locked translations, no dominance difference), zero gravity, zero damping and caps not engaged, P = sum m v computed
in float64 from body_states() and m = 1 / inv_mass is the same before and after each step.  Each impulse application
rounds the velocities of its two bodies once, an error of at most ~u |m v| per body, so over a step the error of P is
at most c u N sum |m v|, with N the impulse applications on the busiest body: its rows x (substeps x sweeps + 1), the
sweeps being the warm start, the biased and the relaxed passes (1 + pgs + relax) and the + 1 the restitution pass, which
runs once after the substeps (it applies only the normal rows; counting all rows keeps the bound simple); the rows (per manifold its normal rows plus two
tangent rows and a twist row (Coulomb: two tangent rows per point), 6 per joint (12 with limits / motors)).  c = TOL_MOM
= 1, sum |m v| taken as the larger of before and after.  Where a world holds separate clusters (the device piles)
each cluster is checked on its own, with its own N and sum |m v|, so one lost impulse is not hidden by the rest.  Most roundings cancel or are far below the bound: the largest
ratio seen on the oracle and the emulated kernels is 0.002, while an impulse applied with the wrong body's inverse mass
gives 259 and a parallel-axis term of the wrong sign 57 (a wrong inertia turns contact impulses into momentum errors).

Impulse bounds after every step, from the pair tables (pair_data: per manifold point the impulse accumulated over the
step, the last substep's impulse n_k, the twist, the tangent impulse in the world t_w; pair_sc: the point of each solver
contact):
  * every normal impulse >= 0;
  * Coulomb (friction_model = 1): each point's ||t_w|| <= mu n_k (1 + 32 u) (rb_solver.cuh:492, the per-point limit);
  * Simplified: ||t_w|| <= mu sum_k n_k (1 + 32 u), the tangent limit of friction_solve_jac (rb_solver.cuh:507-516,
    :394-398, from contact_with_twist_friction.rs:737-777 of the reference); its twist limit needs the twist distances,
    which no table exposes, and is not checked.
With restitution only the normal bound is checked: the restitution pass runs after the last friction solve and changes
n_k, so the tangent impulse of the last substep need not lie within mu n_k any more.
The 32 u: the clamp's scale and rescaled components (3 roundings), the float32 sum of the limit (up to 4 terms and the
friction product), the rotation into the world through t1, t2 (unit to about 4 u each, two products and a sum),
rounded up; the largest excess seen is 10 u.
"""
import numpy as np
import pytest

from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import (ColliderBuilder, GenericJointBuilder, RevoluteJointBuilder, RigidBodyBuilder, RopeJointBuilder,
                              SphericalJointBuilder, SpringJointBuilder)
from test_mass_properties_reference import build_hull, kind, library, make_world, qmat  # noqa: F401 (kind is a fixture)

U = 2.0 ** -24
TOL_FREE = 16.0
TOL_MOM = 1.0
WORST = {"free": 0.0, "momentum": 0.0}


# ---- float64 restatement of the body phases --------------------------------------------------------------------------------
def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


class FreeBody:
    """float64 state of one body and what the step needs of it."""

    def __init__(self, desc, mp, mf, pose, vel, force, torque, params):
        self.dyn = desc.body_type == A.RB_BODY_DYNAMIC
        self.fl = desc.flags
        self.lcom, self.im, self.ipi, self.qf = mp[:3], mp[3], mp[4:7], mf[:4]
        self.pi = np.array([1.0 / x if x else 0.0 for x in self.ipi])
        self.t, self.q = pose[:3].copy(), pose[3:7].copy()
        self.v, self.w = vel[:3].copy(), vel[3:].copy()
        self.F, self.tau = force, torque
        self.gs, self.ld, self.ad = desc.gravity_scale, desc.linear_damping, desc.angular_damping
        extra = (desc.flags >> A.RB_BODY_EXTRA_ITERS_SHIFT) & 0xFF
        self.nsub = params.num_solver_iterations + extra
        self.dt = params.dt
        self.h = params.dt / self.nsub
        self.max_lin = params.normalized_max_linear_velocity * params.length_unit
        self.max_ang = 0.7853981633974483 / params.dt

    def step(self, g):
        h, R = self.h, qmat(self.q)
        tc = self.t + R @ self.lcom
        if self.dyn:
            A_ = R @ qmat(self.qf)
            Iw = A_ @ np.diag(self.ipi) @ A_.T
            m = 1.0 / self.im if self.im else 0.0
            dv = (self.F + np.asarray(g) * m * self.gs) * self.im * h
            dw = Iw @ self.tau * h
        else:
            dv = dw = np.zeros(3)
        v, w, q = self.v.copy(), self.w.copy(), self.q.copy()
        for _ in range(self.nsub):
            v, w = v + dv, w + dw
            if self.dyn and self.fl & A.RB_BODY_GYROSCOPIC:
                Ax = qmat(qmul(q, self.qf))
                wl = Ax.T @ w
                L = self.pi * wl
                tot = L - np.cross(wl, L) * h
                if tot @ tot:
                    w = Ax @ (self.ipi * (tot * np.sqrt((L @ L) / (tot @ tot))))
            if np.linalg.norm(v) > self.max_lin:
                v = v * (self.max_lin / np.linalg.norm(v))
            if not self.fl & A.RB_BODY_ALLOW_FAST_ROTATION and np.linalg.norm(w) > self.max_ang:
                w = w * (self.max_ang / np.linalg.norm(w))
            q = qmul(np.concatenate([w * h / 2, [1.0]]), q)
            q /= np.linalg.norm(q)
            tc = tc + v * h
        self.v, self.w = v / (1 + self.dt * self.ld), w / (1 + self.dt * self.ad)
        self.q = q
        self.t = tc - qmat(q) @ self.lcom


def read_mass(w):
    return (w.debug_read("body_mprops", np.float32).reshape(-1, 16).astype(np.float64),
            w.debug_read("body_mframe", np.float32).reshape(-1, 7).astype(np.float64))


def free_scene(L):
    """Bodies far apart (no contacts), falling under gravity; returns the scene and per-body user force / torque."""
    s = scenes.Scene("free_bodies", gravity=(0.0, -9.81, 0.0))
    hull = build_hull(L, np.asarray([(0.3, -0.1, 0.05), (-0.15, 0.22, 0.0), (-0.12, -0.2, 0.1), (0.05, 0.02, 0.33),
                                                  (0.1, 0.1, -0.2), (-0.2, -0.05, -0.1)], np.float32))
    FT = []

    def add(bb, cbs, force=(0, 0, 0), torque=(0, 0, 0)):
        h = s.bodies.insert(bb.translation((12.0 * len(s.bodies), 0.0, 0.0)).can_sleep(False))
        for cb in cbs:
            s.colliders.insert_with_parent(cb, h)
        FT.append((np.array(force, np.float64), np.array(torque, np.float64)))
    off_hull = ColliderBuilder.convex_mesh(*hull).translation((0.3, -0.2, 0.1)).rotation((0.3, 0.5, -0.2))
    add(RigidBodyBuilder.dynamic().angvel((2.0, 5.0, -3.0)).linvel((0.5, 1.0, 0.0)).gravity_scale(0.5), [off_hull])
    add(RigidBodyBuilder.dynamic().angvel((2.0, 5.0, -3.0)).gyroscopic_forces_enabled(False), [off_hull])
    compound = [ColliderBuilder.cuboid(0.4, 0.1, 0.2).translation((0.2, 0.1, 0.0)), ColliderBuilder.ball(0.2).translation((-0.3, 0.0, 0.2)).density(3.0)]
    add(RigidBodyBuilder.dynamic().angvel((-4.0, 1.0, 6.0)).linear_damping(0.3).angular_damping(0.7), compound,
        force=(3.0, 1.0, -2.0), torque=(0.2, -0.1, 0.3))
    add(RigidBodyBuilder.dynamic().angvel((3.0, -2.0, 4.0)).additional_solver_iterations(3),
        [ColliderBuilder.cuboid(0.5, 0.2, 0.1).rotation((0.2, 0.1, 0.0))], torque=(0.05, 0.0, 0.02))
    add(RigidBodyBuilder.kinematic_velocity_based().linvel((1.0, 0.5, 0.0)).angvel((0.5, 2.0, -1.0)), [ColliderBuilder.cuboid(0.5, 0.2, 0.1)])
    add(RigidBodyBuilder.dynamic().angvel((80.0, 10.0, 0.0)), [ColliderBuilder.ball(0.3)])                      # angular cap engaged
    fast = RigidBodyBuilder.dynamic().angvel((80.0, 10.0, 0.0))
    fast._flags |= A.RB_BODY_ALLOW_FAST_ROTATION
    add(fast, [ColliderBuilder.ball(0.3)])                                                                       # ... exempt
    add(RigidBodyBuilder.dynamic().linvel((30.0, 0.0, 4.0)), [ColliderBuilder.cuboid(0.2, 0.2, 0.2)])           # linear cap engaged
    add(RigidBodyBuilder.dynamic().angvel((0.0, 40.0, 0.0)).linvel((2.0, 3.0, 0.0)).gravity_scale(-2.0),
        [ColliderBuilder.capsule_z(0.3, 0.1)], force=(0.0, 0.0, 5.0))                                            # caps not engaged
    return s, FT


def free_params(coulomb=False):
    p = A.RbIntegrationParameters.default()
    p.normalized_max_linear_velocity = 20.0 / p.length_unit
    p.friction_model = 1 if coulomb else 0
    return p


def quat_err(a, b):
    return min(np.abs(a - b).max(), np.abs(a + b).max())


@pytest.mark.parametrize("model", ["simplified", "coulomb"])
def test_free_body_step(kind, model):
    s, FT = free_scene(library(kind))
    p = free_params(model == "coulomb")
    w = make_world(kind, s, p)
    idx = np.arange(len(FT))
    w.set_body_forces(idx, np.array([f for f, _ in FT], np.float32), np.array([t for _, t in FT], np.float32))
    pose, vel = (x.astype(np.float64) for x in w.body_states())
    mp, mf = read_mass(w)
    ref = [FreeBody(d, mp[b], mf[b], pose[b], vel[b], *FT[b], p) for b, d in enumerate(s.bodies.descs)]
    for step in range(1, 61):
        w.step()
        for r in ref:
            r.step(s.gravity)
        if step not in (1, 60):
            continue
        pose, vel = (x.astype(np.float64) for x in w.body_states())
        for b, r in enumerate(ref):
            n = r.nsub * step
            T = step * p.dt
            where = f"{kind} {model} body {b} after {step} steps"
            for name, got, want, rate in (("t", pose[b, :3], r.t, r.v), ("v", vel[b, :3], r.v, (r.F + np.asarray(s.gravity)) * r.im),
                                          ("w", vel[b, 3:], r.w, r.w)):
                S = 1.0 + np.abs(want).max() + np.abs(rate).max() * T
                e = np.abs(got - want).max() / (n * U * S)
                WORST["free"] = max(WORST["free"], e)
                assert e <= TOL_FREE, f"{where}: {name} {got} vs {want} ({e:.1f})"
            S = 1.0 + np.abs(r.w).max() * T
            e = quat_err(pose[b, 3:7], r.q) / (n * U * S)
            WORST["free"] = max(WORST["free"], e)
            assert e <= TOL_FREE, f"{where}: q {pose[b, 3:7]} vs {r.q} ({e:.1f})"
    # the caps engaged where they should
    assert np.linalg.norm(vel[5, 3:]) <= 0.7853981633974483 / p.dt * (1 + 1e-6) < np.linalg.norm(vel[6, 3:])
    assert abs(np.linalg.norm(vel[7, :3]) - 20.0) < 1e-4


def test_closed_forms(kind):
    """Constant force: v = v0 + F dt / m every step.  Spin about a principal axis: the angle of each substep is
    2 atan(|w| h / 2) (the linearised quaternion step), so one step turns by n 2 atan(|w| h / 2)."""
    s = scenes.Scene("closed_forms", gravity=(0.0, 0.0, 0.0))
    s.insert(RigidBodyBuilder.dynamic().linvel((0.5, -1.0, 2.0)).can_sleep(False), ColliderBuilder.cuboid(0.3, 0.2, 0.1).density(2.0))
    s.insert(RigidBodyBuilder.dynamic().translation((10.0, 0.0, 0.0)).angvel((0.0, 0.0, 30.0)).can_sleep(False),
             ColliderBuilder.cuboid(0.3, 0.2, 0.1))
    p = A.RbIntegrationParameters.default()
    w = make_world(kind, s, p)
    F = np.array([4.0, -3.0, 1.5])
    w.set_body_forces([0], F[None].astype(np.float32), None)
    m = 1.0 / float(read_mass(w)[0][0, 3])
    v0 = w.body_states()[1][0, :3].astype(np.float64)
    for k in range(1, 11):
        w.step()
        pose, vel = (x.astype(np.float64) for x in w.body_states())
        want = v0 + k * F * p.dt / m
        assert np.abs(vel[0, :3] - want).max() <= 64 * k * U * np.abs(want).max(), f"{kind} constant force step {k}: {vel[0, :3]} vs {want}"
        h = p.dt / p.num_solver_iterations
        ang = k * p.num_solver_iterations * 2.0 * np.arctan(30.0 * h / 2.0)
        want_q = np.array([0.0, 0.0, np.sin(ang / 2), np.cos(ang / 2)])
        assert quat_err(pose[1, 3:7], want_q) <= 64 * k * U * (1 + 30.0 * k * p.dt), f"{kind} spin step {k}: {pose[1, 3:7]} vs {want_q}"
        assert quat_err(pose[1, 3:7], np.array([0.0, 0.0, np.sin(k * 0.5 / 2), np.cos(k * 0.5 / 2)])) > 1e-4   # not |w| h


# ---- momentum balance --------------------------------------------------------------------------------------------------------
def random_part(rng, k, L):
    r = lambda a, b: float(rng.uniform(a, b))
    k %= 8
    if k == 0:
        return [ColliderBuilder.ball(r(0.15, 0.3))]
    if k == 1:
        return [ColliderBuilder.cuboid(r(0.1, 0.3), r(0.1, 0.3), r(0.1, 0.3))]
    if k in (2, 3):
        return [[ColliderBuilder.capsule_x, ColliderBuilder.capsule_y, ColliderBuilder.capsule_z][int(rng.integers(3))](r(0.05, 0.2), r(0.08, 0.15))]
    if k == 4:
        return [ColliderBuilder.convex_mesh(*build_hull(L, rng.uniform(-0.25, 0.25, (8, 3)).astype(np.float32)))]
    if k == 5:
        return [ColliderBuilder.convex_mesh(*build_hull(L, rng.uniform(-0.2, 0.2, (7, 3)).astype(np.float32)), border_radius=0.04)]
    if k == 6:
        return [ColliderBuilder.cuboid(0.25, 0.08, 0.08).translation((0.1, 0.0, 0.0)), ColliderBuilder.ball(0.12).translation((-0.2, 0.05, 0.0)).density(2.0)]
    return [ColliderBuilder.cuboid(0.2, 0.2, 0.2).density(float(rng.choice([0.3, 1.0, 5.0])))]


def cluster(s, rng, n, centre, L, spacing=0.42, vel=1.5, restitution=0.0, sensors=False, extra_iters=0):
    """n dynamic bodies of mixed shapes on a jittered lattice (neighbours touching), velocities pointing inwards; hulls built
    by library L.  Returns the bodies' indices."""
    side = int(np.ceil(n ** (1.0 / 3.0)))
    hs = []
    for i in range(n):
        g = np.array([i % side, (i // side) % side, i // (side * side)], np.float64)
        p = np.asarray(centre) + (g - (side - 1) / 2.0) * spacing + rng.uniform(-0.03, 0.03, 3)
        v = -(p - np.asarray(centre)) / max(np.linalg.norm(p - np.asarray(centre)), 1e-3) * vel + rng.uniform(-0.3, 0.3, 3)
        bb = (RigidBodyBuilder.dynamic().translation(p).rotation(tuple(rng.uniform(-1, 1, 3))).linvel(v).angvel(rng.uniform(-2, 2, 3))
              .can_sleep(False).gyroscopic_forces_enabled(False))
        if extra_iters and i % 7 == 0:
            bb = bb.additional_solver_iterations(extra_iters)
        h = s.bodies.insert(bb)
        for cb in random_part(rng, i, L):
            s.colliders.insert_with_parent(cb.restitution(restitution).friction(0.5), h)
        if sensors and i % 6 == 0:
            s.colliders.insert_with_parent(ColliderBuilder.ball(0.35).density(0.0).sensor(), h)
        hs.append(h)
    return hs


def rows_per_body(s, w, coulomb, njrows):
    """Constraint rows acting on each body in the last step (see the module docstring)."""
    keys = w.debug_read("pair_keys", np.uint64)
    nsc = w.debug_read("pair_nsc", np.int32)
    par = np.array([c.parent for c in s.colliders.descs])
    rows = np.zeros(len(s.bodies))
    for k, n in zip(keys, nsc):
        if n <= 0:
            continue
        for c in (int(k >> np.uint64(32)), int(k & np.uint64(0xffffffff))):
            if par[c] >= 0:
                rows[par[c]] += n + (2 * n if coulomb else 3)
    for j in s.joints.descs:
        for b in (j.body1, j.body2):
            rows[b] += njrows
    return rows


def check_impulse_bounds(w, coulomb, where, mu=0.5, friction=True):
    data = w.debug_read("pair_data", np.float32).reshape(-1, 4, 12).astype(np.float64)
    nsc = w.debug_read("pair_nsc", np.int32)
    cid = w.debug_read("pair_sc", np.int32).reshape(-1, 4, 7)[:, :, 6]   # manifold point of each solver contact
    for i in np.nonzero(nsc > 0)[0]:
        d = data[i, cid[i, :nsc[i]]]
        assert (d[:, 0] >= 0.0).all() and (d[:, 1] >= 0.0).all(), f"{where}: pair {i} negative normal impulse {d[:, :2]}"
        if not friction:
            continue
        t = np.linalg.norm(d[:, 3:6], axis=1)
        if coulomb:
            assert (t <= mu * d[:, 1] * (1 + 32 * U) + 1e-30).all(), f"{where}: pair {i} Coulomb bound: |t| {t} > mu n {mu * d[:, 1]}"
        else:
            assert t.max() <= mu * d[:, 1].sum() * (1 + 32 * U) + 1e-30, f"{where}: pair {i} tangent {t.max()} > mu sum n {mu * d[:, 1].sum()}"


def run_momentum(kind, s, p, steps, where, groups=None, njrows=6, friction_bounds=True):
    """Steps the world, checking the momentum of each group of bodies (no constraint between groups; default: one group
    of every body) and the impulse bounds after every step."""
    w = make_world(kind, s, p)
    coulomb = p.friction_model == 1
    groups = groups or [np.arange(len(s.bodies))]
    extra = np.array([(d.flags >> A.RB_BODY_EXTRA_ITERS_SHIFT) & 0xFF for d in s.bodies.descs])
    sweeps = 1 + p.num_internal_pgs_iterations + p.num_internal_stabilization_iterations
    for k in range(steps):
        mp = read_mass(w)[0]
        dyn = mp[:, 3] > 0.0
        m = np.where(dyn, 1.0 / np.where(dyn, mp[:, 3], 1.0), 0.0)
        v0 = w.body_states()[1][:, :3].astype(np.float64)
        w.step()
        v1 = w.body_states()[1][:, :3].astype(np.float64)
        rows = rows_per_body(s, w, coulomb, njrows)
        for g in groups:
            P0, P1 = (m[g, None] * v0[g]).sum(0), (m[g, None] * v1[g]).sum(0)
            S = max((m[g, None] * np.abs(v0[g])).sum(), (m[g, None] * np.abs(v1[g])).sum())
            # every row on the busiest body, in every sweep of every substep, and its normal rows once more in the
            # restitution pass (counted as all its rows)
            N = max(rows[g].max(), 1.0) * ((p.num_solver_iterations + extra[g].max()) * sweeps + 1)
            r = np.abs(P1 - P0).max() / (U * N * S)
            WORST["momentum"] = max(WORST["momentum"], r)
            assert r <= TOL_MOM, f"{kind} {where} step {k + 1} bodies {g[0]}..: momentum {P0} -> {P1} ({r:.2f} x u N sum|mv|, N = {N})"
        check_impulse_bounds(w, coulomb, f"{kind} {where} step {k + 1}", friction=friction_bounds)
        if kind != "oracle":   # which solve paths ran: State::nlarge_bodies, need_big, coop_streamed, coop_resident
            st = w.debug_read("state", np.int32)
            w.paths = np.maximum(getattr(w, "paths", np.zeros(4, np.int64)), st[[12, 18, 19, 20]])
    c = w.counters()
    assert c["num_active_manifolds"] > 0
    return w


def zero_g(name):
    return scenes.Scene(name, gravity=(0.0, 0.0, 0.0))


CONTACT_CASES = ["streamed", "resident", "coulomb", "restitution", "sensors", "substep_groups"]


@pytest.mark.parametrize("case", CONTACT_CASES)
def test_momentum_balance_contacts(kind, case, monkeypatch):
    rng = np.random.default_rng(1 + CONTACT_CASES.index(case))
    s = zero_g(f"momentum_{case}")
    cluster(s, rng, 45, (0.0, 0.0, 0.0), library(kind), restitution=0.4 if case == "restitution" else 0.0, sensors=case == "sensors",
            extra_iters=2 if case == "substep_groups" else 0)
    p = A.RbIntegrationParameters.default()
    if case == "coulomb":
        p.friction_model = 1
    if case == "streamed" and kind == "emulated":
        monkeypatch.setenv("RB_EMU_COOP_SMEM_FLOATS", "5600")
    w = run_momentum(kind, s, p, 8, case, friction_bounds=case != "restitution")
    if case == "streamed" and kind == "emulated":
        assert w.paths[2] >= 1, "the cluster must have taken the streaming path"
    if case == "resident" and kind != "oracle":
        assert w.paths[3] >= 1, "the cluster must have been solved resident in shared memory"


def test_momentum_balance_grid_wide_item(kind):
    """One zero-g cluster of 343 touching bodies: more than 256, the grid-wide item 0."""
    s = zero_g("momentum_grid_wide")
    cluster(s, np.random.default_rng(5), 343, (0.0, 0.0, 0.0), library(kind), spacing=0.4, vel=0.5)
    w = run_momentum(kind, s, A.RbIntegrationParameters.default(), 3, "grid_wide")
    if kind != "oracle":
        assert w.paths[0] > 256, "the cluster must be the grid-wide item"


@pytest.mark.parametrize("warm", [0, 1], ids=["cold_joints", "warmstart_joints"])
def test_momentum_balance_joints(kind, warm):
    """Chains of dynamic bodies joined by spherical, revolute (with limits and a motor), generic (coupled, limited)
    spring and rope joints, colliding with a free cluster: the general path."""
    rng = np.random.default_rng(13)
    s = zero_g("momentum_joints")
    hs = cluster(s, rng, 27, (0.0, 0.0, 0.0), library(kind))
    chain = []
    for i in range(8):
        chain.append(s.insert(RigidBodyBuilder.dynamic().translation((-1.6 + 0.45 * i, 1.2, 0.0)).linvel((0.0, -1.0, 0.3 * (i % 3)))
                              .angvel((0.0, 0.0, 1.0)).can_sleep(False).gyroscopic_forces_enabled(False), ColliderBuilder.cuboid(0.2, 0.1, 0.1)))
    a1, a2 = (0.225, 0.0, 0.0), (-0.225, 0.0, 0.0)
    s.joints.insert(chain[0], chain[1], SphericalJointBuilder().local_anchor1(a1).local_anchor2(a2))
    s.joints.insert(chain[1], chain[2], RevoluteJointBuilder((0.0, 0.0, 1.0)).local_anchor1(a1).local_anchor2(a2).limits(3, -0.3, 0.4).motor_velocity(3, 2.0, 0.5))
    s.joints.insert(chain[2], chain[3], SpringJointBuilder(0.45, 50.0, 1.0).local_anchor1(a1).local_anchor2(a2))
    s.joints.insert(chain[3], chain[4], RopeJointBuilder(0.5).local_anchor1(a1).local_anchor2(a2))
    s.joints.insert(chain[4], chain[5], GenericJointBuilder(0b000111).coupled_axes(0b110000).limits(4, -0.2, 0.2).local_anchor1(a1).local_anchor2(a2))
    s.joints.insert(chain[5], chain[6], GenericJointBuilder(0b011111).limits(3, -0.5, 0.5).motor_position(3, 0.2, 30.0, 2.0).local_anchor1(a1).local_anchor2(a2))
    s.joints.insert(chain[6], chain[7], GenericJointBuilder(0b111001).limits(1, -0.05, 0.05).motor_velocity(2, 0.5, 1.0).local_anchor1(a1).local_anchor2(a2))
    s.joints.insert(hs[0], chain[7], SphericalJointBuilder().local_anchor2(a1).contacts_enabled(False))
    p = A.RbIntegrationParameters.default()
    p.warmstart_joints = warm
    run_momentum(kind, s, p, 8, f"joints_warm{warm}", njrows=12)


def test_dominance(kind):
    """A body of a higher dominance group hit by lighter ones: its velocity is unchanged bit for bit, and the momentum
    change appears only on the dominated side (their momentum changes, the dominant's does not)."""
    s = zero_g("dominance")
    big = s.insert(RigidBodyBuilder.dynamic().linvel((0.5, 0.0, 0.0)).angvel((0.0, 0.3, 0.0)).dominance_group(5).can_sleep(False)
                   .gyroscopic_forces_enabled(False), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    small = []
    for i, (p, v) in enumerate([((1.3, 0.0, 0.0), (-2.0, 0.0, 0.0)), ((0.0, 1.2, 0.2), (0.0, -1.5, 0.0)), ((-1.1, 0.3, 0.0), (1.0, 0.0, 0.5))]):
        small.append(s.insert(RigidBodyBuilder.dynamic().translation(p).linvel(v).can_sleep(False).gyroscopic_forces_enabled(False),
                              ColliderBuilder.ball(0.3) if i % 2 else ColliderBuilder.cuboid(0.2, 0.2, 0.2)))
    w = make_world(kind, s)
    v_big = w.body_states()[1][big].copy()
    changed = False
    for k in range(20):
        v0 = w.body_states()[1][small].copy()
        w.step()
        vel = w.body_states()[1]
        assert (vel[big].view(np.uint32) == v_big.view(np.uint32)).all(), f"{kind} step {k + 1}: dominant body's velocity changed"
        changed |= bool(np.abs(vel[small] - v0).max() > 0.1)
        check_impulse_bounds(w, False, f"{kind} dominance step {k + 1}")
    assert changed, "the dominated bodies must have been hit"


# ---- device sizes (-m gpu only) ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_momentum_balance_device_sizes(built):
    """Zero-g piles on the device, the momentum checked cluster by cluster (12 m apart, so no constraint joins two):
    * about 20 000 bodies in clusters of 2 to 200.  The first step of a world launches k_solve_coop (the small shape, four
      lanes per constraint); clusters of 60 and more do not fit that shape resident (State::need_big), so the following
      steps launch k_solve_coop_big (one lane per constraint, rb_api.cu: the launch hint host_hint[0]), and the largest
      clusters stream their constraint rows while the small ones stay resident;
    * one 3 000-body cluster: the grid-wide item 0 (k_solve_large)."""
    L = library("cuda")
    rng = np.random.default_rng(17)
    s = zero_g("momentum_device_pile")
    groups, n, k = [], 0, 0
    while n < 20000:
        size = int(rng.choice([2, 3, 5, 8, 13, 30, 60, 120, 200]))
        groups.append(np.array(cluster(s, rng, size, ((k % 40) * 12.0, 0.0, (k // 40) * 12.0), L, vel=1.0)))
        n += size
        k += 1
    w = run_momentum("cuda", s, A.RbIntegrationParameters.default(), 4, "pile_20k", groups=groups)
    assert w.paths[1] == 1, "some item must need the big launch shape (steps 2.. run one lane per constraint)"
    assert w.paths[2] > 0 and w.paths[3] > 0, "items must both stream their rows and stay resident"
    s = zero_g("momentum_device_large")
    cluster(s, rng, 3000, (0.0, 0.0, 0.0), L, spacing=0.4, vel=0.5)
    w = run_momentum("cuda", s, A.RbIntegrationParameters.default(), 3, "cluster_3k")
    assert w.paths[0] > 2000, "the cluster must be the grid-wide item"
