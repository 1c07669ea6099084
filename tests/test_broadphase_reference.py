"""Collider bounds and the broad-phase pair set (rapier_b200/csrc/rb_collide.cuh: refresh_collider, section_build_lists,
section_broad_phase; oracle/oracle_world.cpp: refresh_collider, update_pairs) against references written here from the
definitions (numpy only).

The device broad phase is a different algorithm from the oracle's: z strips as wide as the widest mover (far strips
clamped into the first and last), movers sorted by (strip, quantised min-x), a sweep of the own strip and the next one
reaching back by the widest mover's x extent, an interval search into the statics widened by the widest narrow static,
a short list of wide statics capped at WIDE_CAP = 1024, and grid-wide radix sorts.  Agreement with the oracle on ordinary
scenes leaves most of that idle, so every case here is laid out to reach one part of it, and after every step of every
case, on every backend (the oracle, the emulated kernels, and the CUDA library under -m gpu), three things are checked:

  * Tight box.  `collider_aabb` against the exact world AABB of the shape, computed in float64 from the body pose that
    `body_states()` reports composed with the collider's pose relative to its parent (ball: centre +- r; cuboid: |R| h;
    capsule: the segment's end points +- r; convex hull: the extreme vertices of R v + t, +- the border radius), widened
    by contact_skin + prediction / 2.  Each face may differ from the exact one by at most EPS (eps_box below), outwards
    or inwards: the kernels compute the same formulas in float32, rounding to nearest, so the box is the exact one up to
    rounding and neither contains it nor is contained by it bit for bit.
  * Fat box.  `collider_fat` contains `collider_aabb` (exactly, in float32), and the hysteresis is exact: where the fat
    box before the step contained the new tight box it is unchanged bit for bit, otherwise it is the tight box -+ fat_skin
    (0.04 * length_unit), computed in float32.
  * Pair set.  `pair_keys` is strictly ascending and equals the set of collider pairs c1 < c2 whose fat boxes overlap
    (float32, closed intervals: equal bounds overlap) and that are allowed: neither collider belongs to a removed body,
    different parents, at least one parent strictly dynamic, collision groups passing both ways, no joint with contacts
    disabled between the two bodies.  Up to EXACT_LIMIT colliders the reference is all pairs (every strictly dynamic
    collider against every collider: the only pairs that can be allowed).  Above it: every reported pair overlaps and is
    allowed, and a seeded sample of SAMPLE movers, each against every collider, finds no pair that is missing.

Which state the reads describe: the device refreshes the boxes and runs the broad phase at the start of a step, so after
a step its boxes belong to the poses before it and its pairs to its own fat boxes.  The oracle refreshes the boxes at the
end of a step (and when a body is teleported), so after a step its boxes belong to the poses after it and its pairs to the
fat boxes read before it.

EPS, the tolerance of the tight box (eps_box): with u = 2^-24 (half a float32 ulp, relative), M = the largest magnitude of
the collider's box coordinates and L = the lever arm of the rotation, in the 1-norm: |relative translation|_1 plus the
shape's extent (ball r, cuboid hx + hy + hz, capsule half height + r, hull max |v|_1 + border radius):
  * translation part: at most four roundings at magnitude M (adding the parent's translation to the rotated relative one,
    subtracting / adding the half width, the margin; a hull adds the translation after its border): 4 u M;
  * rotation part (rb_math.cuh: qmul, rotmat, rotate):
      - the composed quaternion q = q_body * q_rel is not renormalised.  Each component is one product and three fused
        multiply-adds, four roundings of terms bounded by |q_body| |q_rel| ~ 1: at most 4 u per component, 8 u in norm.
        The stored float32 quaternions miss unit length by at most about 2.5 u each.  So |q| = 1 +- 13 u, |q|^2 = 1 +- 26 u;
      - rotmat's entries (s^2 R + (1 - s^2) I on the diagonal, s^2 R off it, s = |q|) and rotate (v (w^2 - |b|^2) +
        2 b (v.b) + 2 w (b x v) = s^2 R v) are homogeneous of degree two in q, so the length error scales every rotated
        quantity by 1 +- 26 u: 26 u L;
      - their own roundings (two or three per matrix entry, the fused terms of rotate) and the three-term sums of |R| h
        or R v: at most about 10 u of the same lever arm;
    26 u + 10 u = 36 u, rounded up to 40 u L.
So EPS = u (4 M + 40 L).  At the origin and a 0.5 m shape this is about 1e-6 m; at 1e5 m it is 0.024 m (a float32 ulp
there is 0.0078 m).  The largest deviation seen is in DESIGN.md section 5.
"""
import numpy as np
import pytest

import emul_lib
import oracle_lib
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import ColliderBuilder, FixedJointBuilder, RigidBodyBuilder, SphericalJointBuilder, as_array

F32 = np.float32
U = 2.0 ** -24
FAT_SKIN = F32(0.04)                     # 4.0e-2f * length_unit of the default parameters
HALF_PREDICTION = F32(0.02) / F32(2.0)   # normalized_prediction_distance * length_unit / 2, as the kernels compute it
EXACT_LIMIT = 6000
SAMPLE = 2000
BALL, CUBOID, CAPSULE, CONVEX = A.RB_SHAPE_BALL, A.RB_SHAPE_CUBOID, A.RB_SHAPE_CAPSULE, A.RB_SHAPE_CONVEX
SHAPE_NAMES = {BALL: "ball", CUBOID: "cuboid", CAPSULE: "capsule", CONVEX: "convex"}


def eps_box(mag, reach):
    return U * (4.0 * mag + 40.0 * reach)


# ---- float64 geometry --------------------------------------------------------------------------------------------------
def qmat(q):
    """Rotation matrices of the (normalised) quaternions q = (x, y, z, w), batched over the leading axis."""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    x, y, z, w = (q[..., i] for i in range(4))
    m = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                  2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                  2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)
    return m.reshape(q.shape[:-1] + (3, 3))


def collider_world_poses(tab, body_pose):
    """World rotation [n, 3, 3] and translation [n, 3] of every collider, in float64, from the float32 body states
    (rows: translation, quaternion x y z w) and the colliders' float32 poses relative to their parents."""
    par = tab["parent"]
    R = qmat(tab["pos_wrt_parent_q"])
    t = tab["pos_wrt_parent_t"].astype(np.float64)
    has = par >= 0
    if has.any():
        bp = body_pose[par[has]].astype(np.float64)
        Rb = qmat(bp[:, 3:7])
        R[has] = Rb @ R[has]
        t[has] = np.einsum("nij,nj->ni", Rb, t[has]) + bp[:, :3]
    return R, t


def reference_boxes(tab, hulls, R, t):
    """Exact world AABBs (float64) widened by contact_skin + prediction / 2, and the 1-norm lever arm of each collider (EPS)."""
    n = len(tab)
    shape, he = tab["shape"], tab["half_extents"].astype(np.float64)
    lo, hi = np.zeros((n, 3)), np.zeros((n, 3))
    radius = np.zeros(n)
    for s in (BALL, CUBOID, CAPSULE):
        m = shape == s
        if not m.any():
            continue
        if s == BALL:
            ws = np.repeat(he[m, :1], 3, 1)
            radius[m] = he[m, 0]
        elif s == CUBOID:
            ws = np.einsum("nij,nj->ni", np.abs(R[m]), he[m])
            radius[m] = he[m].sum(1)
        else:
            u = R[m][np.arange(m.sum()), :, he[m, 2].astype(int)]   # the segment's axis in the world
            ws = np.abs(u) * he[m, :1] + he[m, 1:2]
            radius[m] = he[m, 0] + he[m, 1]
        lo[m], hi[m] = t[m] - ws, t[m] + ws
    conv = np.nonzero(shape == CONVEX)[0]
    for hid in np.unique(he[conv, 0].astype(int)):
        sel = conv[he[conv, 0].astype(int) == hid]
        v = np.asarray(hulls[hid - 1][0], np.float64)
        p = np.einsum("nij,vj->nvi", R[sel], v)
        br = he[sel, 1:2]
        lo[sel] = p.min(1) + t[sel] - br
        hi[sel] = p.max(1) + t[sel] + br
        radius[sel] = np.abs(v).sum(1).max() + he[sel, 1]
    margin = tab["contact_skin"].astype(np.float64)[:, None] + float(HALF_PREDICTION)
    reach = radius + np.abs(tab["pos_wrt_parent_t"].astype(np.float64)).sum(1)
    return lo - margin, hi + margin, reach


def overlap(alo, ahi, blo, bhi):
    """Closed float32 boxes overlap on all three axes (broadcast)."""
    return ((alo <= bhi) & (blo <= ahi)).all(-1)


# ---- the model of the world the backends simulate ----------------------------------------------------------------------
class Model:
    """Who may pair with whom, from the descriptors the scene was built from and the bodies removed since."""

    def __init__(self, scene, removed, tab=None):
        self.tab = np.ctypeslib.as_array(as_array(scene.colliders.descs, A.RbColliderDesc)) if tab is None else tab
        btype = np.array([d.body_type for d in scene.bodies.descs], np.int32)
        self.nb = len(btype)
        par = self.tab["parent"]
        gone = np.zeros(self.nb, bool)
        gone[list(removed)] = True
        self.alive = (par < 0) | ~gone[np.maximum(par, 0)]
        self.strict_dyn = (par >= 0) & (btype[np.maximum(par, 0)] == A.RB_BODY_DYNAMIC) & self.alive
        self.parent = par
        self.mem = self.tab["collision_memberships"]
        self.filt = self.tab["collision_filter"]
        self.nocontact = np.array(sorted(min(d.body1, d.body2) * self.nb + max(d.body1, d.body2)
                                         for d in scene.joints.descs if not d.contacts_enabled), np.int64)

    def allowed(self, i, j):
        """Pair filter of the broad phase over index arrays (the overlap is tested separately)."""
        pi, pj = self.parent[i], self.parent[j]
        ok = (i != j) & self.alive[i] & self.alive[j] & (self.strict_dyn[i] | self.strict_dyn[j])
        ok &= ~((pi >= 0) & (pi == pj))
        ok &= ((self.mem[i] & self.filt[j]) != 0) & ((self.mem[j] & self.filt[i]) != 0)
        if len(self.nocontact):
            both = (pi >= 0) & (pj >= 0)
            key = np.minimum(pi, pj).astype(np.int64) * self.nb + np.maximum(pi, pj)
            ok &= ~(both & np.isin(key, self.nocontact))
        return ok


def reference_pairs(model, lo, hi, movers, chunk=256):
    """Sorted keys (c1 << 32 | c2) of every allowed pair with an overlapping collider, over the given movers (all pairs
    when `movers` are all strictly dynamic colliders)."""
    out = []
    for a in range(0, len(movers), chunk):
        m = movers[a:a + chunk]
        ox = (lo[m, None, 0] <= hi[None, :, 0]) & (lo[None, :, 0] <= hi[m, None, 0])
        ii, jj = np.nonzero(ox)
        i, j = m[ii], jj
        keep = overlap(lo[i], hi[i], lo[j], hi[j]) & model.allowed(i, j)
        i, j = i[keep], j[keep]
        out.append((np.minimum(i, j).astype(np.uint64) << np.uint64(32)) | np.maximum(i, j).astype(np.uint64))
    return np.unique(np.concatenate(out)) if out else np.zeros(0, np.uint64)


def check_pairs(model, lo, hi, keys, where, mode="auto", seed=0):
    """The pair-set checks of the module docstring; mode "auto" is exact up to EXACT_LIMIT colliders, else sampled."""
    assert keys.dtype == np.uint64
    assert (keys[1:] > keys[:-1]).all(), f"{where}: pair_keys not strictly ascending"   # (np.diff would wrap around)
    nc = len(lo)
    movers = np.nonzero(model.strict_dyn)[0]
    if mode == "exact" or (mode == "auto" and nc <= EXACT_LIMIT):
        ref = reference_pairs(model, lo, hi, movers)
        missing, extra = np.setdiff1d(ref, keys), np.setdiff1d(keys, ref)
        assert not len(missing) and not len(extra), (
            f"{where}: pair set differs: missing {[(int(k >> 32), int(k & 0xffffffff)) for k in missing[:8]]} "
            f"({len(missing)}), extra {[(int(k >> 32), int(k & 0xffffffff)) for k in extra[:8]]} ({len(extra)})")
        return len(ref)
    c1, c2 = (keys >> np.uint64(32)).astype(np.int64), (keys & np.uint64(0xffffffff)).astype(np.int64)
    assert ((c1 < c2) & (c2 < nc)).all(), f"{where}: malformed pair keys"
    ok = overlap(lo[c1], hi[c1], lo[c2], hi[c2]) & model.allowed(c1, c2)
    assert ok.all(), f"{where}: reported pairs that do not overlap or are not allowed: {list(zip(c1[~ok][:8], c2[~ok][:8]))}"
    rng = np.random.default_rng(seed)
    sample = np.sort(rng.choice(movers, min(SAMPLE, len(movers)), replace=False))
    ref = reference_pairs(model, lo, hi, sample, chunk=64)
    missing = ref[~np.isin(ref, keys)]
    assert not len(missing), f"{where}: pair set misses {[(int(k >> 32), int(k & 0xffffffff)) for k in missing[:8]]} ({len(missing)})"
    return len(ref)


# ---- one world on one backend, checked after every step -----------------------------------------------------------------
class Sim:
    def __init__(self, kind, scene, reserve=None, pair_mode="auto"):
        self.kind, self.scene, self.pair_mode = kind, scene, pair_mode
        self.device = kind != "oracle"
        if kind == "oracle":
            self.w = oracle_lib.OracleWorld(scene)
        else:
            from rapier_b200.world import PhysicsWorld
            self.w = PhysicsWorld(scene, _lib=emul_lib.lib() if kind == "emulated" else None)
            if reserve:
                self.w.reserve(*reserve)
        self.removed = set()
        self.nsteps = 0
        self.worst = {}      # shape -> [largest inward, largest outward deviation of a tight face, in units of EPS]
        self.npairs = []
        self._tab = None

    # public-API changes between steps, mirrored into the scene's descriptor sets
    def insert(self, bodies=(), statics=()):
        s = self.scene
        if self.device:
            for bb, cbs in bodies:
                h = self.w.insert(bb, cbs[0])
                for cb in cbs[1:]:
                    self.w.insert_collider(cb, parent=h)
            for cb in statics:
                self.w.insert_collider(cb)
            return
        nb0, nc0 = len(s.bodies), len(s.colliders)
        for bb, cbs in bodies:
            h = s.bodies.insert(bb)
            for cb in cbs:
                s.colliders.insert_with_parent(cb, h)
        for cb in statics:
            s.colliders.insert(cb)
        self.w.sync_hulls(s.colliders)
        self.w.insert(s.bodies.descs[nb0:], s.colliders.descs[nc0:])

    def remove(self, bodies):
        if self.device:
            for b in bodies:
                self.w.remove(b)
        else:
            self.w.remove_bodies(bodies)
        self.removed.update(bodies)

    def set_body_states(self, idx, pose7=None, vel6=None):
        self.w.set_body_states(idx, pose7, vel6)

    def set_next_kinematic_positions(self, idx, pose7):
        self.w.set_next_kinematic_positions(idx, pose7)

    def body_states(self):
        return self.w.body_states()

    def boxes(self, table):
        b = self.w.debug_read(table, np.float32).reshape(-1, 6)
        return b[:, :3].copy(), b[:, 3:].copy()

    def step(self, n=1):
        for _ in range(n):
            self._step()

    def _step(self):
        pose0 = self.body_states()[0]
        flo0, fhi0 = self.boxes("collider_fat")
        self.w.step()
        self.nsteps += 1
        where = f"{self.kind} {self.scene.name} step {self.nsteps}"
        pose1 = self.body_states()[0]
        alo, ahi = self.boxes("collider_aabb")
        flo, fhi = self.boxes("collider_fat")
        keys = self.w.debug_read("pair_keys", np.uint64)
        if self._tab is None or len(self._tab) != len(self.scene.colliders):
            self._tab = Model(self.scene, ()).tab
        model = Model(self.scene, self.removed, self._tab)
        live = model.alive
        # 1. tight box against the float64 geometry
        R, t = collider_world_poses(model.tab, pose0 if self.device else pose1)
        rlo, rhi, reach = reference_boxes(model.tab, self.scene.colliders.hulls, R, t)
        mag = np.maximum(np.abs(rlo), np.abs(rhi)).max(1)
        eps = eps_box(mag, reach)[:, None]
        out = np.concatenate([rlo - alo, ahi - rhi], 1)[live] / eps[live]   # > 0: looser than exact, < 0: tighter
        bad = np.nonzero((np.abs(out) > 1.0).any(1))[0]
        ids = np.nonzero(live)[0]
        assert not len(bad), (f"{where}: tight box off the float64 box by more than EPS: colliders {ids[bad[:8]].tolist()}, "
                              f"deviation / EPS {out[bad[:4]].tolist()}")
        for s in np.unique(model.tab["shape"][live]):
            m = model.tab["shape"][live] == s
            w = self.worst.setdefault(SHAPE_NAMES[int(s)], [0.0, 0.0])
            w[0], w[1] = max(w[0], float(-out[m].min())), max(w[1], float(out[m].max()))
        # 2. fat box: contains the tight one, exact hysteresis
        cont = ((flo <= alo) & (fhi >= ahi)).all(1)
        assert cont[live].all(), f"{where}: fat box does not contain the tight box: colliders {ids[~cont[live]][:8].tolist()}"
        n0 = len(flo0)
        kept = np.zeros(len(flo), bool)
        kept[:n0] = ((flo0 <= alo[:n0]) & (fhi0 >= ahi[:n0])).all(1)
        same = np.zeros(len(flo), bool)
        same[:n0] = (flo[:n0].view(np.uint32) == flo0.view(np.uint32)).all(1) & (fhi[:n0].view(np.uint32) == fhi0.view(np.uint32)).all(1)
        refat = ((flo.view(np.uint32) == (alo - FAT_SKIN).view(np.uint32)).all(1) &
                 (fhi.view(np.uint32) == (ahi + FAT_SKIN).view(np.uint32)).all(1))
        hyst = np.where(kept, same, refat)
        assert hyst[live].all(), (f"{where}: fat-box hysteresis broken: colliders {ids[~hyst[live]][:8].tolist()} "
                                  f"(kept: {kept[ids[~hyst[live]][:8]].tolist()})")
        # 3. pair set
        plo, phi = (flo, fhi) if self.device else (flo0, fhi0)
        for mode in (("exact", "sampled") if self.pair_mode == "both" else (self.pair_mode,)):
            n = check_pairs(model, plo, phi, keys, f"{where} ({mode})", mode, seed=self.nsteps)
        self.npairs.append(n)


@pytest.fixture(params=["oracle", "emulated", pytest.param("cuda", marks=pytest.mark.gpu)])
def kind(request):
    if request.param == "cuda":
        request.getfixturevalue("built")
    return request.param


# ---- shapes ------------------------------------------------------------------------------------------------------------
TETRA = ([(0.25, -0.1, 0.05), (-0.15, 0.22, 0.0), (-0.12, -0.2, 0.1), (0.05, 0.02, 0.33)],
         [[0, 1, 2], [0, 1, 3], [1, 2, 3], [0, 2, 3]])
OCTA = ([(0.3, 0.05, 0.0), (-0.22, 0.05, 0.0), (0.04, 0.25, 0.0), (0.04, -0.15, 0.0), (0.04, 0.05, 0.2), (0.04, 0.05, -0.28)],
        [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])
PRISM = ([(-0.2, -0.15, -0.2), (0.25, -0.15, -0.2), (0.0, 0.2, -0.2), (-0.2, -0.15, 0.2), (0.25, -0.15, 0.2), (0.0, 0.2, 0.2)],
         [[0, 1, 2], [3, 5, 4], [0, 3, 4, 1], [1, 4, 5, 2], [2, 5, 3, 0]])


def random_collider(rng, k, scale=1.0):
    """Shape k % 7 of balls, cuboids, capsules along each axis and three convex meshes (one round), scaled."""
    r = lambda a, b: float(rng.uniform(a, b)) * scale
    k %= 7
    if k == 0:
        return ColliderBuilder.ball(r(0.08, 0.25))
    if k == 1:
        return ColliderBuilder.cuboid(r(0.05, 0.25), r(0.05, 0.25), r(0.05, 0.25))
    if k in (2, 3, 4):
        return [ColliderBuilder.capsule_x, ColliderBuilder.capsule_y, ColliderBuilder.capsule_z][k - 2](r(0.05, 0.2), r(0.05, 0.12))
    verts, faces = (TETRA, OCTA, PRISM)[k - 5] if k < 7 else PRISM
    pts = np.asarray(verts, np.float32) * F32(scale)
    return ColliderBuilder.convex_mesh(pts, faces, border_radius=0.03 * scale if k == 6 else 0.0)


def rand_rot(rng, amp=np.pi):
    return tuple(float(x) for x in rng.uniform(-amp, amp, 3))


def add_random_movers(s, rng, n, centre, spread, vel=0.5, k0=0, scale=1.0):
    """n dynamic bodies of mixed shapes, randomly posed in a box of half size `spread` around `centre`; some compound,
    some with an offset collider."""
    hs = []
    for i in range(n):
        p = np.asarray(centre, np.float64) + rng.uniform(-1, 1, 3) * np.asarray(spread, np.float64)
        bb = RigidBodyBuilder.dynamic().translation(p).rotation(rand_rot(rng)).linvel(rng.uniform(-vel, vel, 3)).angvel(rng.uniform(-1, 1, 3))
        h = s.bodies.insert(bb)
        cb = random_collider(rng, k0 + i, scale)
        if i % 5 == 3:
            cb = cb.translation(tuple(rng.uniform(-0.2, 0.2, 3) * scale)).rotation(rand_rot(rng))
        s.colliders.insert_with_parent(cb, h)
        if i % 9 == 4 and (k0 + i) % 7 < 5:   # a second part (bodies with a convex mesh have only one collider)
            s.colliders.insert_with_parent(random_collider(rng, (k0 + i) % 5, scale).translation((0.3 * scale, 0.0, 0.0)), h)
        hs.append(h)
    return hs


# ---- exact float32 edges -----------------------------------------------------------------------------------------------
def f32_ord(f):
    i = int(np.float32(f).view(np.int32))
    return i if i >= 0 else -(i & 0x7fffffff) - 1


def f32_of(o):
    return np.int32(o if o >= 0 else -(o + 1) | -0x80000000).view(np.float32)


def f32_solve(fn, target, guess, first=True):
    """Smallest (first=True) float32 x with fn(x) >= target, or the largest with fn(x) <= target, for a nondecreasing fn."""
    lo, hi = f32_ord(guess) - (1 << 24), f32_ord(guess) + (1 << 24)
    if first:
        assert fn(f32_of(lo)) < target <= fn(f32_of(hi))
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (lo, mid) if fn(f32_of(mid)) >= target else (mid, hi)
        return f32_of(hi)
    assert fn(f32_of(lo)) <= target < fn(f32_of(hi))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if fn(f32_of(mid)) <= target else (lo, mid)
    return f32_of(lo)


def fat_lo(t, h):
    """Fat min of an unrotated collider at the origin of an unrotated body at t whose half width along the axis is h
    (cuboid half extent, ball / capsule radius): (t - h) - (skin + prediction / 2) - fat_skin, each rounded to float32."""
    return (F32(t) - F32(h)) - HALF_PREDICTION - FAT_SKIN


def fat_hi(t, h):
    return (F32(t) + F32(h)) + HALF_PREDICTION + FAT_SKIN


def strip_of(minz, wz):
    """The strip index strip_key gives a min-z, before clamping (float32, as the kernel computes it)."""
    return int(np.floor(F32(minz) * (F32(1.0) / F32(wz))))


# ---- layouts -----------------------------------------------------------------------------------------------------------
def layout_control(seed):
    """A dense random pile near the origin on a slab, with some bodies thrown down (motion mostly along y)."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"control_{seed}")
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -0.5, 0.0)), ColliderBuilder.cuboid(4.0, 0.5, 4.0))
    add_random_movers(s, rng, 70, (0.0, 1.2, 0.0), (0.9, 1.0, 0.9), vel=0.5)
    for i in range(6):
        s.insert(RigidBodyBuilder.dynamic().translation((2.5, 0.6 + 0.6 * i, -2.5 + i)).linvel((0.0, -3.0, 0.0)),
                 random_collider(rng, i))
    return s


def layout_strip_edges(seed):
    """Pairs of movers on z-strip boundaries k * wz on both sides of 0, touching across the boundary (equal bounds),
    overlapping it by one float32 ulp, or apart by one ulp; and pairs touching exactly along x and y, mover against
    mover and mover against static.  The widest mover (fat z extent known in float32) sets the strip width."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"strip_edges_{seed}", gravity=(0.0, 0.0, 0.0))
    hw = F32(0.6)
    s.insert(RigidBodyBuilder.dynamic().translation((-20.0, 0.0, 0.0)), ColliderBuilder.cuboid(0.2, 0.2, hw))
    width = fat_hi(0.0, hw) - fat_lo(0.0, hw)
    wz = F32(width * F32(1.01)) + F32(1.0e-3)
    s.strip_width = wz
    s.edges = []
    x = 0.0
    for k in (-3, -1, 0, 1, 4):
        zb = F32(0.0) if k == 0 else f32_solve(lambda z: strip_of(z, wz), k, F32(k * wz))
        # touching, one ulp of overlap, one ulp apart; at 0 no translation lands a fat bound exactly on 0 or one (denormal)
        # ulp from it, so the pairs there overlap the boundary by a few ulps ("over")
        for gap in ((0, 1, -1) if k else ("over",)):
            for kb, hb in ((0, F32(0.15)), (1, F32(0.1))):
                tb = f32_solve(lambda t: fat_lo(t, hb), zb, zb + hb + F32(0.05))
                bz = fat_lo(tb, hb)
                want = f32_of(f32_ord(bz) + (1 if gap == "over" else gap))
                for ha in F32(0.45) + F32(0.001) * np.arange(20, dtype=F32):   # (wider than half a strip) one that lands exactly
                    ta = f32_solve(lambda t: fat_hi(t, ha), want, want - ha - F32(0.05))
                    if fat_hi(ta, ha) == want:
                        break
                assert fat_hi(ta, ha) == want or gap == "over", (k, gap)
                s.insert(RigidBodyBuilder.dynamic().translation((x, 0.0, float(ta))), ColliderBuilder.cuboid(0.2, 0.2, float(ha)))
                a = len(s.colliders) - 1
                cb = ColliderBuilder.ball(float(hb)) if kb == 0 else ColliderBuilder.capsule_x(0.1, float(hb))
                s.insert(RigidBodyBuilder.dynamic().translation((x + 0.05, 0.1, float(tb))), cb)
                s.edges.append((a, len(s.colliders) - 1, k, gap))
                x += 3.0
    # exact touching along each axis, on either side of the mover: against a mover and against a parentless static
    for axis in (0, 1, 2):
        for side in (1, -1):
            for static in (False, True):
                pa = np.array([x, 5.0, 3.0])
                pb = pa.copy()
                if side > 0:
                    pb[axis] = f32_solve(lambda t: fat_lo(t, F32(0.2)), fat_hi(pa[axis], F32(0.25)), F32(pa[axis] + 0.45))
                else:
                    pb[axis] = f32_solve(lambda t: fat_hi(t, F32(0.2)), fat_lo(pa[axis], F32(0.25)), F32(pa[axis] - 0.45))
                s.insert(RigidBodyBuilder.dynamic().translation(pa), ColliderBuilder.cuboid(0.25, 0.25, 0.25))
                if static:
                    s.colliders.insert(ColliderBuilder.cuboid(0.2, 0.2, 0.2).translation(pb))
                else:
                    s.insert(RigidBodyBuilder.dynamic().translation(pb), ColliderBuilder.ball(0.2))
                s.edges.append((len(s.colliders) - 2, len(s.colliders) - 1, None, side))
                x += 3.0
    add_random_movers(s, rng, 40, (60.0, 0.0, 30.0), (3.0, 1.0, 3.0), vel=0.3, scale=0.8)
    return s


def check_strip_edges(sim):
    """The layout does what it claims: collider 0 is the widest mover along z, its fat z extent gives the strip width, and
    the strips of each edge pair."""
    s = sim.scene
    lo, hi = sim.boxes("collider_fat")
    movers = Model(s, ()).strict_dyn
    width = hi[0, 2] - lo[0, 2]
    assert movers[0] and width == (hi[movers, 2] - lo[movers, 2]).max()
    assert F32(width * F32(1.01)) + F32(1.0e-3) == s.strip_width
    for a, b, k, gap in s.edges:
        if k is None:
            ax = [i for i in range(3) if (hi[a, i] == lo[b, i] if gap > 0 else lo[a, i] == hi[b, i])]
            assert len(ax) == 1, (a, b, lo[[a, b]], hi[[a, b]])
            continue
        assert strip_of(lo[b, 2], s.strip_width) == k and strip_of(lo[a, 2], s.strip_width) < k, (a, b, k)
        d = f32_ord(hi[a, 2]) - f32_ord(lo[b, 2])
        assert (d >= 1) if gap == "over" else (d == gap), (a, b, k, gap, d)


def layout_far_field(seed):
    """Clusters of movers out to |z| ~ 1e5 (strips clamped into the first and last) and |x| up to 9e4, where the quantised
    min-x of the sort key (16 m wide at 5e4) ties between every member of a cluster; clusters straddling x = 0."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"far_field_{seed}", gravity=(0.0, 0.0, 0.0))
    centres = [(5.0e4, 1.0e5), (5.0e4 + 3.0, 1.0e5), (-6.0e4, -1.0e5), (9.0e4, -9.9e4), (0.0, 1.0e5), (0.0, -1.0e5),
               (0.0, 0.0), (-3.0e4, 40.0), (3.0e4, -2.0e3), (4.0e4, 8.0e4), (-9.0e4, 9.9e4), (0.5, 5.0e4)]
    k = 0
    for cx, cz in centres:
        n = int(rng.integers(5, 9))
        add_random_movers(s, rng, n, (cx, 0.0, cz), (0.6, 0.5, 0.6), vel=1.5, k0=k)
        k += n
    s.insert(RigidBodyBuilder.fixed().translation((5.0e4, -0.9, 1.0e5)), ColliderBuilder.cuboid(3.0, 0.2, 3.0))
    s.colliders.insert(ColliderBuilder.cuboid(2.0, 0.2, 2.0).translation((-0.5, -0.8, -1.0e5)))
    return s


def layout_reach(seed):
    """A mover much taller in z than the rest (a few wide strips), with small movers beside it along its length up to its
    top end, which lies in the next strip; and a mover much wider in x, in the strip above small movers that touch it
    at its right end: found only by the next-strip search reaching back by the widest mover's x extent."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"reach_{seed}", gravity=(0.0, 0.0, 0.0))
    hh = 10.0
    W = 2 * (hh + 0.2) + 0.1
    wz = W * 1.01 + 1e-3
    zc = 0.45 * wz + hh + 0.25   # min-z at 0.45 wz: the top end lies in the next strip
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.0, zc)), ColliderBuilder.capsule_z(hh, 0.2))
    for i, dz in enumerate((-9.0, -4.0, 0.0, 5.0, 8.5, 9.8)):
        s.insert(RigidBodyBuilder.dynamic().translation((0.35 if i % 2 else -0.35, 0.0, zc + dz)), random_collider(rng, i, 0.4)
                 if i % 3 == 2 else ColliderBuilder.ball(0.1))
    # the wide mover: min-z just above the strip boundary at 0, x from -6.05 to 6.05
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 3.0, 0.17)), ColliderBuilder.cuboid(6.0, 0.1, 0.1))
    for x in (5.95, 5.0, 3.0):
        s.insert(RigidBodyBuilder.dynamic().translation((x, 3.25, 0.0)), ColliderBuilder.ball(0.1))
    s.insert(RigidBodyBuilder.dynamic().translation((-5.9, 2.75, -0.05)), ColliderBuilder.capsule_y(0.05, 0.1))
    add_random_movers(s, rng, 40, (0.0, 8.0, 0.0), (6.0, 1.0, 6.0), vel=0.3)
    return s


def layout_statics(seed):
    """Narrow statics of mixed widths, parentless and on fixed bodies (rotated, one compound); a few long narrow ones
    whose min-x lies metres left of the movers above their right ends (found only through the `wn` widening); and two
    slabs far above four times the mean width (the wide list)."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"statics_{seed}", gravity=(0.0, 0.0, 0.0))
    for i in range(80):
        p = (float(rng.uniform(-12, 12)), float(rng.uniform(-1.0, 0.0)), float(rng.uniform(-12, 12)))
        cb = ColliderBuilder.cuboid(float(rng.uniform(0.2, 0.7)), 0.2, float(rng.uniform(0.1, 0.5)))
        if i % 4 == 0:
            s.insert(RigidBodyBuilder.fixed().translation(p).rotation(rand_rot(rng, 0.5)), cb)
            if i % 8 == 0:
                s.colliders.insert_with_parent(random_collider(rng, i % 5).translation((0.0, 0.4, 0.0)), len(s.bodies) - 1)
        else:
            s.colliders.insert(cb.translation(p).rotation(rand_rot(rng, 0.3) if i % 3 else (0.0, 0.0, 0.0)))
    for i, z in enumerate((-20.0, -17.0, -14.0)):   # long narrow statics (fat width 3.7), a mover over the right end
        s.colliders.insert(ColliderBuilder.cuboid(1.8, 0.1, 0.3).translation((20.0, 0.0, z)))
        s.insert(RigidBodyBuilder.dynamic().translation((21.6, 0.25, z)), random_collider(rng, i, 0.5) if i else ColliderBuilder.ball(0.1))
    s.colliders.insert(ColliderBuilder.cuboid(30.0, 0.2, 3.0).translation((0.0, -3.0, 20.0)))
    s.insert(RigidBodyBuilder.fixed().translation((0.0, -3.0, -30.0)).rotation((0.0, 0.2, 0.0)), ColliderBuilder.cuboid(25.0, 0.2, 4.0))
    add_random_movers(s, rng, 60, (0.0, 0.2, 0.0), (12.0, 0.6, 12.0), vel=1.0)
    add_random_movers(s, rng, 10, (0.0, -2.6, 20.0), (10.0, 0.3, 2.0), vel=0.5, k0=2)
    add_random_movers(s, rng, 10, (0.0, -2.6, -30.0), (10.0, 0.3, 2.0), vel=0.5, k0=4)
    return s


def layout_wide_cap(seed, columns=11, rows=100, narrow=4500):
    """More than WIDE_CAP wide statics: columns x rows plates 10.1 m wide in fat x extent, each under one of `columns`
    long movers, and enough narrow statics (0.2 m) that all plates stay above four times the mean width."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"wide_cap_{seed}", gravity=(0.0, 0.0, 0.0))
    for c in range(columns):
        for r in range(rows):
            s.colliders.insert(ColliderBuilder.cuboid(5.0, 0.05, 0.2).translation((12.0 * c, 0.0, 0.6 * r)))
    side = int(np.ceil(np.sqrt(narrow)))
    for i in range(narrow):
        s.colliders.insert(ColliderBuilder.cuboid(0.05, 0.05, 0.05).translation((200.0 + 0.3 * (i % side), 0.0, 0.3 * (i // side))))
    for c in range(columns):
        s.insert(RigidBodyBuilder.dynamic().translation((12.0 * c + 0.3 * c / columns, 0.2, 29.7)), ColliderBuilder.capsule_z(30.0, 0.1))
    add_random_movers(s, rng, 30, (200.0 + 0.15 * side, 0.3, 0.15 * side), (0.15 * side, 0.1, 0.15 * side), vel=0.3, scale=0.5)
    s.plates = columns * rows
    return s


def layout_filters(seed):
    """Every filter of the pair set on overlapping colliders: compound parts of one body; a kinematic body against a
    fixed one (excluded) and against a dynamic one; asymmetric membership / filter groups; two bodies joined with
    contacts disabled (excluded) and two joined with contacts enabled; sensors."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"filters_{seed}", gravity=(0.0, 0.0, 0.0))
    comp = s.bodies.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.0, 0.0)))
    for dx in (-0.1, 0.1, 0.3):
        s.colliders.insert_with_parent(random_collider(rng, int(dx * 10) + 1).translation((dx, 0.0, 0.0)), comp)
    s.insert(RigidBodyBuilder.dynamic().translation((0.5, 0.0, 0.0)), ColliderBuilder.ball(0.15))
    s.insert(RigidBodyBuilder.fixed().translation((3.0, 0.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5))
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((3.8, 0.0, 0.0)), ColliderBuilder.cuboid(0.4, 0.4, 0.4))
    s.insert(RigidBodyBuilder.kinematic_velocity_based().translation((3.0, 0.9, 0.0)).linvel((0.2, 0.0, 0.0)), ColliderBuilder.ball(0.4))
    s.insert(RigidBodyBuilder.dynamic().translation((4.5, 0.0, 0.0)), ColliderBuilder.capsule_y(0.2, 0.2))
    s.insert(RigidBodyBuilder.kinematic_position_based().translation((3.8, 0.75, 0.0)), ColliderBuilder.ball(0.3))
    groups = [(1, 2), (2, 1), (1, 1), (4, 0xffffffff), (0xffffffff, 4)]
    for i, (m, f) in enumerate(groups):
        s.insert(RigidBodyBuilder.dynamic().translation((6.0 + 0.35 * i, 0.1 * (i % 2), 0.0)), random_collider(rng, i).collision_groups(m, f))
    s.colliders.insert(ColliderBuilder.cuboid(1.0, 0.2, 0.2).translation((6.7, -0.4, 0.0)).collision_groups(2, 2))
    j = []
    for i in range(4):
        j.append(s.insert(RigidBodyBuilder.dynamic().translation((9.0 + 0.3 * i, 0.0, 0.0)), random_collider(rng, i + 2)))
    s.joints.insert(j[0], j[1], FixedJointBuilder().local_anchor1((0.15, 0.0, 0.0)).local_anchor2((-0.15, 0.0, 0.0)).contacts_enabled(False))
    s.joints.insert(j[2], j[3], SphericalJointBuilder().local_anchor1((0.15, 0.0, 0.0)).local_anchor2((-0.15, 0.0, 0.0)))
    s.joints.insert(j[1], j[2], SphericalJointBuilder().local_anchor1((0.15, 0.0, 0.0)).local_anchor2((-0.15, 0.0, 0.0)).contacts_enabled(False))
    s.insert(RigidBodyBuilder.dynamic().translation((12.0, 0.0, 0.0)), ColliderBuilder.ball(0.4).sensor())
    s.insert(RigidBodyBuilder.dynamic().translation((12.5, 0.0, 0.0)), ColliderBuilder.cuboid(0.2, 0.2, 0.2))
    s.colliders.insert(ColliderBuilder.cuboid(0.3, 0.3, 0.3).translation((11.5, 0.0, 0.0)).sensor())
    s.insert(RigidBodyBuilder.fixed().translation((12.0, -0.6, 0.0)), ColliderBuilder.cuboid(1.0, 0.2, 0.3).sensor())
    add_random_movers(s, rng, 20, (6.0, 0.0, 3.0), (6.0, 0.5, 1.0), vel=0.5)
    return s


def layout_sleeping(seed):
    """Bodies at rest beside one another and above statics (fat boxes overlapping, shapes apart) fall asleep and keep their
    pairs; a slow one that cannot sleep passes over them."""
    s = scenes.Scene(f"sleeping_{seed}", gravity=(0.0, 0.0, 0.0))
    shapes = [ColliderBuilder.ball(0.2), ColliderBuilder.cuboid(0.2, 0.2, 0.2), ColliderBuilder.capsule_x(0.1, 0.1),
              ColliderBuilder.convex_mesh(np.asarray(PRISM[0], np.float32) * F32(0.8), PRISM[1])]
    for i in range(12):
        x = 0.48 * i
        s.colliders.insert(ColliderBuilder.cuboid(0.2, 0.1, 0.2).translation((x, -0.35, 0.0)))
        s.insert(RigidBodyBuilder.dynamic().translation((x, 0.0, 0.0)), shapes[i % 4])
    s.insert(RigidBodyBuilder.dynamic().translation((0.0, 0.52, 0.0)).linvel((0.1, 0.0, 0.0)).can_sleep(False), ColliderBuilder.ball(0.2))
    return s


# ---- the tests: one per layout (DESIGN section 5) ----------------------------------------------------------------------
def test_check_pairs_rejects_wrong_tables():
    """The pair checker itself: a table with the right set in the wrong order, with a pair missing, with a pair too many,
    or with a duplicate fails it, in both the exact and the sampled mode (no library involved)."""
    s = scenes.Scene("checker", gravity=(0.0, 0.0, 0.0))
    for x in (0.0, 0.4, 0.8, 1.2):
        s.insert(RigidBodyBuilder.dynamic().translation((x, 0.0, 0.0)), ColliderBuilder.ball(0.25))
    s.colliders.insert(ColliderBuilder.cuboid(2.0, 0.1, 0.5).translation((0.6, -0.5, 0.0)))
    model = Model(s, ())
    centre = np.array([[0.0, 0.0, 0.0], [0.4, 0.0, 0.0], [0.8, 0.0, 0.0], [1.2, 0.0, 0.0], [0.6, -0.5, 0.0]], np.float32)
    half = np.array([[0.3] * 3] * 4 + [[2.05, 0.25, 0.55]], np.float32)
    lo, hi = centre - half, centre + half
    key = lambda a, b: (a << 32) | b
    good = np.array([key(0, 1), key(0, 4), key(1, 2), key(1, 4), key(2, 3), key(2, 4), key(3, 4)], np.uint64)
    for mode in ("exact", "sampled"):
        assert check_pairs(model, lo, hi, good, "good", mode) == len(good)
        swapped = good.copy()
        swapped[[2, 3]] = swapped[[3, 2]]
        wrong = {"not strictly ascending": [swapped, np.concatenate([good[:3], good[2:]])],
                 "differs|misses": [np.delete(good, 4)],
                 "differs|not overlap or are not allowed": [np.sort(np.append(good, np.uint64(key(0, 3))))]}
        for msg, tables in wrong.items():
            for t in tables:
                with pytest.raises(AssertionError, match=msg):
                    check_pairs(model, lo, hi, t, "wrong", mode)


@pytest.mark.parametrize("seed", [0, 1])
def test_control_pile(kind, seed):
    sim = Sim(kind, layout_control(seed))
    sim.step(6)
    assert min(sim.npairs) > 100


def test_strip_edges(kind):
    sim = Sim(kind, layout_strip_edges(3))
    for i in range(4):
        sim.step()
        if i == 0:
            check_strip_edges(sim)


def test_far_field(kind):
    sim = Sim(kind, layout_far_field(5))
    sim.step(5)
    assert min(sim.npairs) > 30


def test_reach_tall_and_wide_movers(kind):
    sim = Sim(kind, layout_reach(7))
    sim.step(4)


def test_narrow_and_wide_statics(kind):
    sim = Sim(kind, layout_statics(11))
    sim.step(6)


def test_wide_cap_overflow(kind):
    s = layout_wide_cap(13)
    sim = Sim(kind, s, pair_mode="both")   # (the sampled checks used above EXACT_LIMIT colliders run here too)
    sim.step(3)
    flo, fhi = sim.boxes("collider_fat")
    widths = fhi[:, 0] - flo[:, 0]
    static = Model(s, ()).parent < 0
    assert (widths[:s.plates] > 4.0 * widths[static].astype(np.float64).mean()).all()
    assert sim.npairs[-1] >= s.plates


def test_filters(kind):
    sim = Sim(kind, layout_filters(17))
    sim.step(5)


def test_sleeping_bodies_keep_pairs(kind):
    sim = Sim(kind, layout_sleeping(19))
    sim.step(45)
    asleep = sim.w.sleeping()
    assert asleep[:12].sum() >= 6 and not asleep[12]


def test_insert_movers_and_parentless_statics(kind):
    rng = np.random.default_rng(23)
    s = layout_control(23)
    sim = Sim(kind, s, reserve=(len(s.bodies) + 40, len(s.colliders) + 80))
    sim.step(2)
    sim.insert(bodies=[(RigidBodyBuilder.dynamic().translation(tuple(rng.uniform(-1, 1, 3) + (0, 1.5, 0))), [random_collider(rng, i)])
                       for i in range(8)])
    sim.step(2)
    sim.insert(statics=[ColliderBuilder.cuboid(0.3, 0.05, 0.3).translation(tuple(rng.uniform(-1, 1, 3) + (0, 1.0, 0))) for _ in range(6)])
    sim.step(2)
    sim.insert(bodies=[(RigidBodyBuilder.dynamic().translation((0.0, 3.0, 0.0)), [ColliderBuilder.ball(0.2), ColliderBuilder.cuboid(0.1, 0.1, 0.1)])],
               statics=[ColliderBuilder.cuboid(3.0, 0.05, 0.2).translation((0.0, 2.7, 0.0))])
    sim.step(2)


def test_remove_bodies(kind):
    s = layout_control(29)
    sim = Sim(kind, s)
    sim.step(2)
    sim.remove([3, 10, 11, 40])
    sim.step(2)
    sim.remove([0])   # the ground slab's body
    sim.step(2)


def test_teleport_fixed_body(kind):
    """A fixed body moved with set_body_states under other movers: the static list is rebuilt from its new place."""
    s = layout_statics(31)
    fixed = [i for i, d in enumerate(s.bodies.descs) if d.body_type == A.RB_BODY_FIXED]
    sim = Sim(kind, s)
    sim.step(2)
    pose = sim.body_states()[0]
    for k, b in enumerate(fixed[:3]):
        p = pose[b].copy()
        p[0] += 5.0 + k
        p[2] -= 3.0
        sim.set_body_states([b], p[None])
        sim.step(2)


def test_kinematic_targets(kind):
    """Position-based kinematic bodies driven across dynamic bodies and statics by set_next_kinematic_positions."""
    s = layout_statics(37)
    kin = [s.insert(RigidBodyBuilder.kinematic_position_based().translation((-8.0 + 4.0 * i, 0.2, -4.0 + 2.0 * i)),
                    random_collider(np.random.default_rng(i), i, 2.0)) for i in range(4)]
    sim = Sim(kind, s)
    for k in range(6):
        pose = sim.body_states()[0][kin].copy()
        pose[:, 0] += 0.3
        pose[:, 2] += 0.1 * (k % 3)
        sim.set_next_kinematic_positions(kin, pose)
        sim.step()


def test_dynamic_teleport_far_and_back(kind):
    """A dynamic body teleported to z = 5e4 and back: its pairs leave the set and rejoin it."""
    s = layout_control(41)
    sim = Sim(kind, s)
    sim.step(2)
    b = 20
    home = sim.body_states()[0][b].copy()
    far = home.copy()
    far[2] += 5.0e4
    sim.set_body_states([b], far[None], np.zeros((1, 6), np.float32))
    sim.step(2)
    sim.set_body_states([b], home[None])
    sim.step(2)


# ---- device sizes (-m gpu only) ----------------------------------------------------------------------------------------
def layout_device_sizes(nx=560, nz=250, seed=43):
    """nx x nz movers in rows along x whose fat boxes overlap their x neighbours, over a floor of 0.5 m static tiles:
    140 000 movers and 253 000 statics, so with 132 CTAs (H100 SXM) every CTA sorts more than 1 024 mover and static
    keys, and bits_for(num colliders) = 19 (three radix passes per key word of the candidate sort)."""
    rng = np.random.default_rng(seed)
    s = scenes.Scene(f"device_sizes_{nx}x{nz}", gravity=(0.0, 0.0, 0.0))
    x0, z0 = -0.225 * nx, -0.5 * nz
    for i in range(int(0.45 * nx / 0.5) + 2):
        for k in range(2 * nz):
            s.colliders.insert(ColliderBuilder.cuboid(0.25, 0.05, 0.25).translation((x0 + 0.5 * i, 0.67, z0 + 0.5 * k)))
    v = rng.uniform(-0.3, 0.3, (nx * nz, 3))
    for k in range(nz):
        for i in range(nx):
            n = k * nx + i
            cb = ColliderBuilder.ball(0.2) if n % 4 != 3 else ColliderBuilder.cuboid(0.15, 0.15, 0.15)
            s.insert(RigidBodyBuilder.dynamic().translation((x0 + 0.45 * i, 1.0, z0 + 1.0 * k)).linvel(v[n]), cb)
    return s


@pytest.mark.gpu
def test_device_sizes(built):
    s = layout_device_sizes()
    assert len(s.colliders) >= 70000
    sim = Sim("cuda", s)
    sim.step(3)


@pytest.mark.gpu
def test_large_world_full_size(built):
    sim = Sim("cuda", scenes.large_world())
    sim.step(3)
