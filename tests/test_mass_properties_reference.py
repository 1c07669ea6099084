"""The convex-hull builder, the polyhedron tables and the bodies' mass properties against float64 references computed here
from geometry (numpy / scipy only), on the oracle, the emulated kernels and, under -m gpu, the CUDA library.

Hull builder (rb_hull.h: convex_hull, reached by every ColliderBuilder::convex_hull / round_convex_hull) against
scipy.spatial.ConvexHull, with EPS = 1e-6 (1 + max |coordinate|), the builder's plane-membership tolerance:
  * repeated points: a point within REPEAT EPS (REPEAT = 4, rb_hull.h REPEAT_EPS) of an earlier kept one in every
    coordinate repeats it and must never be kept; the scipy reference below is the hull of the points that remain;
  * the output vertices are exactly the input points that are hull vertices to EPS: a scipy vertex that lies more than
    2 EPS outside the hull of the other points must be kept, a point within 0.5 EPS of it (or inside) must be dropped,
    unless another point lies within 2 REPEAT EPS of it (two corners that close may both stay: the plane and polygon
    tolerances cannot order them);
  * every face's float64 Newell plane supports the set: every input point lies behind it within (1 + sqrt(3) REPEAT) EPS
    (a dropped repeat lies up to sqrt(3) REPEAT EPS from the point kept for it) and the face's vertices lie on it within
    4 EPS (the face's points are only within EPS of the plane through three of them);
  * coplanar facets are merged: the face count equals the number of scipy facet planes after merging facets whose
    vertices lie within EPS of each other's plane;
  * every face is a convex loop wound counter-clockwise seen from outside;
  * the total face area and the enclosed volume match scipy's to 1e-6 relative;
  * the mesh registers through rb_world_add_hull / orc_world_add_hull.
Collinear and coplanar point sets must be rejected with "the points are coplanar", and sets outside 4..32 points with
"convex_hull takes 4..32 points".

Hull tables (debug table "hull_tables", rb_world_debug_read and orc_world_debug_read; every registered hull in id order,
hull 0 the unit cube; the device has them once a convex collider is uploaded), in 4-byte words per hull:
    nv, nf, ne, nloop (int32) | aabb x y z, radius (float32) | vertices [nv][3] (float32) |
    planes [nf][4]: outward unit normal, offset (float32) | faces [nf][2]: start in the loops, count (int32) |
    loops [nloop] (int32) | edges [ne][4]: v0 < v1, the face running v0 -> v1, the other face (int32)
Checked against the mesh: vertices bit-equal; each loop is the input face, possibly reversed, with the float64 Newell
normal of the input face turned outward (to 4 u per component) and offset = n . (mean of the face's vertices) (to
4 u (1 + size)); the edge list equals the one derived here, in ascending (v0, v1) order; aabb bit-equal to max |x|;
radius within one float32 ulp of the float64 max |v|.

Mass properties (debug tables "body_mprops": local com (3), inverse mass, inverse principal inertia (3), world com (3),
effective world inverse inertia xx xy xz yy yz zz; "body_mframe": principal frame x y z w, effective inverse mass (3)),
against float64 references:
  * ball 2/5 m r^2; cuboid m (b^2 + c^2) / 3; capsule (half height h, radius r, along x, y or z): a cylinder plus two
    half balls, I_axis = m_cyl r^2 / 2 + 2/5 m_ball r^2, I_perp = m_cyl (3 r^2 + 4 h^2) / 12 + m_ball (2/5 r^2 + h^2 + 3/4 h r);
  * sharp hulls: tetrahedra of scipy's facets about scipy's centroid of the vertices, summed in float64, principal axes
    by numpy.linalg.eigh; round hulls (border radius > 0) take the inner hull's properties (what the library does: the
    border is left out of the mass, as MassProperties::from_convex_polyhedron of the inner polyhedron);
  * colliders at an offset and rotated on their body, compounds by the parallel-axis sum in float64;
  * additional mass (RigidBodyAdditionalMassProps::Mass): on a massive body the mass grows by m_add and the inertia scales
    by (m + m_add) / m; on a massless collider the shape's unit-density inertia is scaled to m_add; a colliderless body
    gets the mass alone; a massless compound is rejected.
The inertia is compared as a tensor in the body frame, R_frame diag(1 / ipi) R_frame^T, never frame by frame: the frame
is defined only up to a permutation and sign of its axes (DESIGN deviation 8).  The frame must be a unit quaternion
(a proper rotation).  Tolerance: TOL_MP = 32 u times the magnitude (u = 2^-24): |com - ref| <= TOL_MP (|com| + extent),
|1/inv_mass - m| <= TOL_MP m, |I - I_ref| (max entry) <= TOL_MP |I_ref| (max entry).  The largest ratios seen (error /
(u x magnitude)), oracle and emulated kernels: com 0.18, mass 1.5, tensor 2.9 (DESIGN section 5).

Effective world inertia: after set_body_states with arbitrary rotations and after one step in zero gravity,
b_eii = R_body I_ref^-1 R_body^T with the rows and columns of locked rotation axes zeroed, b_eim = 1/m on free translation
axes and 0 on locked ones; kinematic and fixed bodies all zero.  Tolerance TOL_MP u times the largest entry of the
unlocked tensor; largest ratio seen 13.1 (the float32 rotation of the body and of the frame, composed).
"""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import ConvexHull

import emul_lib
import oracle_lib
from rapier_b200 import _abi as A
from rapier_b200 import scenes
from rapier_b200.sets import ColliderBuilder, RigidBodyBuilder

F32 = np.float32
U = 2.0 ** -24
TOL_MP = 32.0
WORST = {"com": 0.0, "mass": 0.0, "tensor": 0.0, "eii": 0.0}
REPEAT = 4.0   # the builder's repeat radius, in units of its membership tolerance EPS (rb_hull.h: convex_hull)
HULL_ERRORS = ("the points are coplanar", "convex_hull takes 4..32 points", "the hull has more than 32 faces",
               "a face of the hull has more than 8 vertices")


@pytest.fixture(params=["oracle", "emulated", pytest.param("cuda", marks=pytest.mark.gpu)])
def kind(request):
    if request.param == "cuda":
        request.getfixturevalue("built")
    return request.param


def library(kind):
    """The library whose host hull builder a backend uses (the oracle registers hulls built by the library's routine)."""
    if kind == "cuda":
        from rapier_b200._lib import lib
        return lib()
    return emul_lib.lib()


def make_world(kind, scene, params=None):
    if kind == "oracle":
        return oracle_lib.OracleWorld(scene, params=params)
    from rapier_b200.world import PhysicsWorld
    return PhysicsWorld(scene, integration_parameters=params, _lib=None if kind == "cuda" else emul_lib.lib())


# ---- float64 geometry ----------------------------------------------------------------------------------------------------
def qmat(q):
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q)
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def axis_angle_quat(v):
    v = np.asarray(v, np.float64)
    a = np.linalg.norm(v)
    if a == 0.0:
        return np.array([0.0, 0.0, 0.0, 1.0])
    return np.concatenate([v / a * np.sin(a / 2), [np.cos(a / 2)]])


def newell(P):
    """Newell normal (not normalised) of a polygon loop [n, 3] in float64."""
    Q = np.roll(P, -1, 0)
    return np.array([((P[:, 1] - Q[:, 1]) * (P[:, 2] + Q[:, 2])).sum(), ((P[:, 2] - Q[:, 2]) * (P[:, 0] + Q[:, 0])).sum(),
                     ((P[:, 0] - Q[:, 0]) * (P[:, 1] + Q[:, 1])).sum()])


def hull_mass_f64(verts):
    """Unit-density volume, centre of mass and inertia tensor about it of the convex hull of `verts` (float64, scipy)."""
    v = np.asarray(verts, np.float64)
    h = ConvexHull(v)
    c0 = v[h.vertices].mean(0)
    vol, mom, C2 = 0.0, np.zeros(3), np.zeros((3, 3))
    for s in h.simplices:
        a, b, c = v[s] - c0
        det = abs(np.dot(a, np.cross(b, c)))          # scipy's facets are unoriented; about an interior point all are positive
        vol += det / 6.0
        sm = a + b + c
        mom += det * sm / 24.0
        C2 += det / 120.0 * (np.outer(a, a) + np.outer(b, b) + np.outer(c, c) + np.outer(sm, sm))
    com = mom / vol
    C2 -= vol * np.outer(com, com)                    # second moment about the centre of mass
    I = np.trace(C2) * np.eye(3) - C2
    return vol, com + c0, I


def shape_mass_f64(shape, he, density, hulls=None):
    """(mass, com in the collider frame, inertia tensor about it) of one collider at `density`."""
    if shape == A.RB_SHAPE_BALL:
        r = he[0]
        m = density * 4.0 / 3.0 * np.pi * r ** 3
        return m, np.zeros(3), np.eye(3) * 0.4 * m * r * r
    if shape == A.RB_SHAPE_CUBOID:
        a, b, c = he
        m = density * 8.0 * a * b * c
        return m, np.zeros(3), np.diag([b * b + c * c, a * a + c * c, a * a + b * b]) * m / 3.0
    if shape == A.RB_SHAPE_CAPSULE:
        h, r, ax = he[0], he[1], int(he[2])
        mc, ms = density * np.pi * r * r * 2.0 * h, density * 4.0 / 3.0 * np.pi * r ** 3
        perp = mc * (3 * r * r + 4 * h * h) / 12.0 + ms * (0.4 * r * r + h * h + 0.75 * h * r)
        d = np.full(3, perp)
        d[ax] = mc * r * r / 2.0 + 0.4 * ms * r * r
        return mc + ms, np.zeros(3), np.diag(d)
    vol, com, I = hull_mass_f64(hulls[int(he[0]) - 1][0])
    return density * vol, com, density * I


def body_mass_f64(scene, b):
    """float64 (mass, local com, inertia tensor about it in the body frame) of body b from its colliders and additional mass;
    None if the library must reject it."""
    descs = [c for c in scene.colliders.descs if c.parent == b and not (c.sensor and c.density == 0.0)]
    M, S, parts = 0.0, np.zeros(3), []
    for c in descs:
        he = np.array(c.half_extents[:], np.float64)
        m, com, I = shape_mass_f64(c.shape, he, float(c.density), scene.colliders.hulls)
        R = qmat(np.array(c.pos_wrt_parent_q[:], np.float64))
        p = R @ com + np.array(c.pos_wrt_parent_t[:], np.float64)
        parts.append((m, p, R @ I @ R.T))
        M += m
        S += m * p
    add = float(scene.bodies.descs[b].additional_mass)
    if M > 0.0:
        com = S / M
        I = sum(Ii + m * (np.dot(p - com, p - com) * np.eye(3) - np.outer(p - com, p - com)) for m, p, Ii in parts)
        if add > 0.0:
            I = I * (M + add) / M
            M += add
        return M, com, I
    if add <= 0.0:
        return 0.0, np.zeros(3), np.zeros((3, 3))
    if len(descs) == 0:
        return add, np.zeros(3), np.zeros((3, 3))
    if len(descs) > 1 or descs[0].shape == A.RB_SHAPE_CONVEX:
        return None
    c = descs[0]
    m1, com, I1 = shape_mass_f64(c.shape, np.array(c.half_extents[:], np.float64), 1.0)
    R = qmat(np.array(c.pos_wrt_parent_q[:], np.float64))
    return add, R @ com + np.array(c.pos_wrt_parent_t[:], np.float64), R @ I1 @ R.T * (add / m1)


def read_mass(w):
    mp = w.debug_read("body_mprops", np.float32).reshape(-1, 16).astype(np.float64)
    mf = w.debug_read("body_mframe", np.float32).reshape(-1, 7).astype(np.float64)
    return mp, mf


def collider_extent(c, hulls):
    """Largest distance of the shape from its own origin (ball r, cuboid |h|, capsule half height + r, hull max |v| +
    border): the length scale of the centre-of-mass tolerance."""
    he = np.array(c.half_extents[:], np.float64)
    if c.shape == A.RB_SHAPE_BALL:
        return he[0]
    if c.shape == A.RB_SHAPE_CUBOID:
        return float(np.linalg.norm(he))
    if c.shape == A.RB_SHAPE_CAPSULE:
        return he[0] + he[1]
    return float(np.linalg.norm(np.asarray(hulls[int(he[0]) - 1][0], np.float64), axis=1).max()) + he[1]


def check_body_mass(scene, mp, mf, b, where):
    ref = body_mass_f64(scene, b)
    M, com, I = ref
    lcom, im, ipi, q = mp[b, :3], mp[b, 3], mp[b, 4:7], mf[b, :4]
    assert abs(np.dot(q, q) - 1.0) <= 8 * U, f"{where}: principal frame not a unit quaternion: {q}"
    ext = max([collider_extent(c, scene.colliders.hulls) for c in scene.colliders.descs if c.parent == b] + [1.0])
    if M == 0.0:
        assert im == 0.0 and (ipi == 0.0).all(), f"{where}: massless body has inv_mass {im}, ipi {ipi}"
        return
    r = abs(1.0 / im - M) / (U * M)
    WORST["mass"] = max(WORST["mass"], r)
    assert r <= TOL_MP, f"{where}: mass {1.0 / im} vs {M} ({r:.1f} u)"
    scale = np.abs(com).max() + max([np.abs(c.pos_wrt_parent_t[:]).max() for c in scene.colliders.descs if c.parent == b] + [0.0]) + ext
    r = np.abs(lcom - com).max() / (U * scale)
    WORST["com"] = max(WORST["com"], r)
    assert r <= TOL_MP, f"{where}: local com {lcom} vs {com} ({r:.1f} u)"
    if not I.any():
        assert (ipi == 0.0).all(), f"{where}: {ipi}"
        return
    R = qmat(q)
    Ib = R @ np.diag([1.0 / x if x else 0.0 for x in ipi]) @ R.T
    r = np.abs(Ib - I).max() / (U * np.abs(I).max())
    WORST["tensor"] = max(WORST["tensor"], r)
    assert r <= TOL_MP, f"{where}: inertia tensor\n{Ib}\nvs\n{I}\n({r:.1f} u)"


# ---- the hull builder -------------------------------------------------------------------------------------------------------
def build_hull(L, pts):
    """rb_convex_hull: (vertices, faces) or the error message."""
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 3)
    nv, nf = C.c_int32(0), C.c_int32(0)
    verts = np.zeros((32, 3), np.float32)
    sizes = np.zeros(32, np.int32)
    idx = np.zeros(256, np.int32)
    rc = L.rb_convex_hull(len(pts), pts.ctypes.data, C.byref(nv), verts.ctypes.data, C.byref(nf), sizes.ctypes.data, idx.ctypes.data)
    if rc < 0:
        return L.rb_last_error().decode()
    faces, at = [], 0
    for f in range(nf.value):
        faces.append([int(i) for i in idx[at:at + sizes[f]]])
        at += int(sizes[f])
    return verts[:nv.value].copy(), faces


def outside_excess(pts, i):
    """How far point i lies outside the hull of the others (max facet-plane excess; <= 0 inside)."""
    others = np.delete(pts, i, 0)
    try:
        h = ConvexHull(others)
    except Exception:
        return np.inf
    return float((h.equations[:, :3] @ pts[i] + h.equations[:, 3]).max())


def merged_planes(h, pts, eps, widest=False):
    """Number of scipy facet planes once facets whose vertices lie within eps of each other's plane are merged (and the
    most hull vertices on one of them)."""
    n = len(h.simplices)
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a
    eq = h.equations
    for a in range(n):
        for b in range(a + 1, n):
            if eq[a, :3] @ eq[b, :3] < 0.5:
                continue
            if (np.abs(pts[h.simplices[b]] @ eq[a, :3] + eq[a, 3]) <= eps).all() and (np.abs(pts[h.simplices[a]] @ eq[b, :3] + eq[b, 3]) <= eps).all():
                parent[find(a)] = find(b)
    roots = {find(a) for a in range(n)}
    if not widest:
        return len(roots)
    return len(roots), max(len({int(v) for a in range(n) if find(a) == r for v in h.simplices[a]}) for r in roots)


def check_hull(pts, out, where):
    pts64 = np.asarray(pts, np.float32).astype(np.float64)
    size = np.abs(pts64).max()
    eps = 1e-6 * (1.0 + size)
    assert not isinstance(out, str), f"{where}: rejected: {out}"
    verts, faces = out
    v64 = verts.astype(np.float64)
    # a point within REPEAT EPS of an earlier representative in every coordinate repeats it: the builder keeps the earlier
    # one, and the scipy reference is the hull of the representatives
    first = []
    for i in range(len(pts64)):
        if not first or (np.abs(pts64[first] - pts64[i]).max(1) > REPEAT * eps).all():
            first.append(i)
    rep = pts64[first]
    sh = ConvexHull(rep)
    # 1. vertices: exactly the eps-vertices among the representatives, in input order, none twice
    kept = [int(np.nonzero((np.asarray(pts, np.float32) == v).all(1))[0][0]) for v in verts]
    assert kept == sorted(set(kept)), f"{where}: vertices not in input order, or a point kept twice"
    assert set(kept) <= set(first), f"{where}: a repeated point kept as a hull vertex"
    for k, i in enumerate(first):
        ex = outside_excess(rep, k) if k in sh.vertices else -1.0
        if ex > 2 * eps:
            assert i in kept, f"{where}: point {i} ({ex / eps:.2f} EPS outside the others) is not a hull vertex"
        elif ex < 0.5 * eps and (np.abs(np.delete(rep, k, 0) - rep[k]).max(1) > 2 * REPEAT * eps).all():
            assert i not in kept, f"{where}: point {i} ({ex / eps:.2f} EPS outside the others) kept as a hull vertex"
    # 2.-4. supporting planes, convex counter-clockwise loops
    area, vol = 0.0, 0.0
    inner = v64.mean(0)
    for f in faces:
        P = v64[f]
        nn = newell(P)
        ln = np.linalg.norm(nn)
        n = nn / ln
        d = n @ P.mean(0)
        assert (pts64 @ n - d <= (1 + np.sqrt(3) * REPEAT) * eps).all(), f"{where}: face {f} does not support the set ({(pts64 @ n - d).max() / eps:.2f} EPS)"
        assert (np.abs(P @ n - d) <= 4 * eps).all(), f"{where}: face {f} is not planar"
        assert n @ inner - d < 0.0, f"{where}: face {f} wound clockwise seen from outside"
        e = np.roll(P, -1, 0) - P
        turns = np.cross(e, np.roll(e, -1, 0)) @ n
        assert (turns > 0.0).all(), f"{where}: face {f} is not a convex counter-clockwise loop"
        area += ln / 2.0
        vol += d * ln / 2.0 / 3.0
    assert len(faces) == merged_planes(sh, rep, eps), f"{where}: {len(faces)} faces, scipy has {merged_planes(sh, rep, eps)} planes"
    assert abs(area - sh.area) <= 1e-6 * sh.area, f"{where}: area {area} vs {sh.area}"
    assert abs(vol - sh.volume) <= 1e-6 * sh.volume, f"{where}: volume {vol} vs {sh.volume}"


def register_hull(kind, verts, faces):
    sizes = np.array([len(f) for f in faces], np.int32)
    idx = np.array([i for f in faces for i in f], np.int32)
    v = np.ascontiguousarray(verts, np.float32)
    if kind == "oracle":
        o = oracle_lib.OracleWorld(scenes.Scene("hull", gravity=(0.0, 0.0, 0.0)))
        return o.L.orc_world_add_hull(o.h, len(v), v.ctypes.data, len(sizes), sizes.ctypes.data, idx.ctypes.data)
    from rapier_b200.world import PhysicsPipeline
    p = PhysicsPipeline(_lib=library(kind))
    return p.L.rb_world_add_hull(p.h, len(v), v.ctypes.data, len(sizes), sizes.ctypes.data, idx.ctypes.data)


CUBE = np.array([(x, y, z) for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float64) * 0.5
PRISM = np.array([(0.0, 0.0, -0.4), (0.6, 0.0, -0.4), (0.2, 0.5, -0.4), (0.0, 0.0, 0.4), (0.6, 0.0, 0.4), (0.2, 0.5, 0.4)])
BIPYR = np.array([(np.cos(a), np.sin(a), 0.0) for a in np.arange(5) * 2 * np.pi / 5] + [(0, 0, 0.8), (0, 0, -0.7)]) * 0.4


def point_sets():
    """(name, points, expected error or None)."""
    rng = np.random.default_rng(7)
    out = []
    for k in range(6):
        out.append((f"box_{k}", rng.uniform(-0.5, 0.5, (int(rng.integers(6, 13)), 3)) * (1.0, 0.6, 1.4), None))
        s = rng.normal(size=(int(rng.integers(8, 15)), 3))
        out.append((f"sphere_{k}", 0.7 * s / np.linalg.norm(s, axis=1, keepdims=True), None))
    for name, P in (("cube", CUBE), ("prism", PRISM), ("bipyramid", BIPYR)):
        out.append((name, P, None))
        # extra points on faces: the centre of a face and a point on an edge (both coplanar, never vertices)
        f_pts = P[np.abs(P[:, 2] - P[:, 2].max()) < 1e-9]
        c = f_pts.mean(0)
        e = 0.5 * (f_pts[0] + f_pts[1]) if len(f_pts) > 1 else None
        if len(f_pts) > 2:
            out.append((f"{name}+face_points", np.vstack([P, c, e]), None))
            eps = 1e-6 * (1.0 + np.abs(P).max())
            for k in (0.3, 3.0, 30.0):
                out.append((f"{name}+face_centre_{k}eps", np.vstack([P, c + (0, 0, k * eps)]), None))
    out.append(("bipyramid_apex_offset", np.vstack([BIPYR, BIPYR.mean(0) + (0.001, 0.0, 0.0)]), None))
    out.append(("duplicates", np.vstack([CUBE, CUBE[:5], PRISM[:1] * 0.1]), None))
    # a corner repeated a fraction of EPS to a few EPS away (0.05 EPS is one float32 ulp here), before or after the corner
    eps = 1e-6 * 1.5
    for d in ((1, 0, 0), (1, 1, 0), (1, 1, 1), (-1, 0, 0), (0.3, 1, -0.7)):
        for k in (0.05, 0.3, 0.6, 1.0, 2.5, 3.9):
            moved = CUBE[7] + k * eps * np.array(d, np.float64)
            out.append((f"corner_repeat_{k}eps_{'_'.join(str(x) for x in d)}", np.vstack([CUBE, moved] if k < 1 else [moved, CUBE]), None))
    out.append(("tetrahedron", np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1)], np.float64) * 0.6 - 0.1, None))
    out.append(("32_points_box", rng.uniform(-1, 1, (32, 3)), "limits"))
    out.append(("32_points_cube_grid", np.array([(x, y, z) for x in (-1, 1) for y in (-1, 1) for z in (-1, 0.5, 1)] +
                                                [(x, y, 0.0) for x in (-1, -0.5, 0.0, 0.5, 1) for y in (-1, 1)] +
                                                [(0.3, 0.2, 1.0), (-0.4, 0.1, -1.0), (1.0, 0.3, 0.2), (0.0, -1.0, 0.7)] +
                                                [(x, y, z) for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (0.0,)] + [(0.0, 0.0, 0.0)] * 2, np.float64) * 0.4, None))
    ring = [(np.cos(a), np.sin(a), h) for h in (-0.5, 0.5) for a in np.arange(10) * 2 * np.pi / 10]
    out.append(("decagonal_prism", np.array(ring) * 0.5, "limits"))
    out.append(("collinear", np.outer(np.linspace(-1, 1, 7), (0.3, 0.5, -0.2)), "the points are coplanar"))
    plane = rng.uniform(-1, 1, (12, 2))
    out.append(("coplanar", np.c_[plane, 0.2 * plane[:, 0] - 0.1 * plane[:, 1] + 0.3], "the points are coplanar"))
    out.append(("coplanar_square", CUBE[CUBE[:, 2] > 0], "the points are coplanar"))
    out.append(("3_points", CUBE[:3], "convex_hull takes 4..32 points"))
    out.append(("33_points", rng.uniform(-1, 1, (33, 3)), "convex_hull takes 4..32 points"))
    return out


POINT_SETS = point_sets()


@pytest.mark.parametrize("name", [n for n, _, _ in POINT_SETS])
def test_hull_builder_against_scipy(kind, name):
    _, P, err = next(s for s in POINT_SETS if s[0] == name)
    pts = np.asarray(P, np.float32)
    out = build_hull(library(kind), pts)
    where = f"{kind} {name}"
    if err == "limits":   # the builder's documented limits: at most 32 faces of at most 8 vertices (scipy decides which applies)
        pts64 = pts.astype(np.float64)
        if isinstance(out, str):
            nplanes, widest = merged_planes(ConvexHull(pts64), pts64, 1e-6 * (1.0 + np.abs(pts64).max()), True)
            assert out.endswith(HULL_ERRORS[2]) and nplanes > 32 or out.endswith(HULL_ERRORS[3]) and widest > 8, \
                f"{where}: {out!r}, scipy: {nplanes} planes, up to {widest} vertices on one"
            return
    elif err is not None:
        assert isinstance(out, str) and out.endswith(err) and any(out.endswith(e) for e in HULL_ERRORS), f"{where}: {out!r}"
        return
    check_hull(pts, out, where)
    assert register_hull(kind, *out) >= 1, f"{where}: the hull does not register"


# ---- hull tables ------------------------------------------------------------------------------------------------------------
def parse_hull_tables(raw):
    words = raw.view(np.uint32)
    fl = raw.view(np.float32)
    out, at = [], 0
    while at < len(words):
        nv, nf, ne, nl = (int(x) for x in words[at:at + 4])
        at += 4
        h = dict(aabb=fl[at:at + 3].copy(), radius=float(fl[at + 3]))
        at += 4
        h["verts"] = fl[at:at + 3 * nv].reshape(nv, 3).copy(); at += 3 * nv
        h["planes"] = fl[at:at + 4 * nf].reshape(nf, 4).copy(); at += 4 * nf
        h["faces"] = words[at:at + 2 * nf].reshape(nf, 2).astype(np.int64); at += 2 * nf
        h["loops"] = words[at:at + nl].astype(np.int64); at += nl
        h["edges"] = words[at:at + 4 * ne].reshape(ne, 4).astype(np.int64); at += 4 * ne
        out.append(h)
    assert at == len(words)
    return out


def check_hull_table(h, verts, faces, where):
    v = np.asarray(verts, np.float32)
    assert (h["verts"].view(np.uint32) == v.view(np.uint32)).all(), f"{where}: vertices differ"
    v64 = v.astype(np.float64)
    size = np.abs(v64).max()
    centroid = v64.mean(0)
    assert len(h["faces"]) == len(faces)
    directed = {}
    for f, face in enumerate(faces):
        s, n = h["faces"][f]
        loop = [int(x) for x in h["loops"][s:s + n]]
        nn = newell(v64[face])
        nrm = nn / np.linalg.norm(nn)
        d = nrm @ v64[face].mean(0)
        if nrm @ centroid - d > 0.0:
            nrm, d, face = -nrm, -d, face[::-1]
        k = loop.index(face[0]) if face[0] in loop else -1
        assert k >= 0 and loop[k:] + loop[:k] == list(face), f"{where}: loop {loop} is not face {face} wound outward"
        assert np.abs(h["planes"][f, :3] - nrm).max() <= 4 * U, f"{where}: plane normal {h['planes'][f, :3]} vs {nrm}"
        assert abs(h["planes"][f, 3] - d) <= 4 * U * (1 + size), f"{where}: plane offset {h['planes'][f, 3]} vs {d}"
        for a, b in zip(loop, loop[1:] + loop[:1]):
            directed[(a, b)] = f
    edges = sorted((a, b, f, directed[(b, a)]) for (a, b), f in directed.items() if a < b)
    assert [tuple(int(x) for x in e) for e in h["edges"]] == edges, f"{where}: edge list differs"
    assert (h["aabb"] == np.abs(v).max(0)).all(), f"{where}: aabb {h['aabb']} vs {np.abs(v).max(0)}"
    r = np.sqrt((v64 ** 2).sum(1)).max()
    assert abs(h["radius"] - r) <= np.spacing(F32(r)), f"{where}: radius {h['radius']} vs {r}"


def test_hull_tables(kind):
    L = library(kind)
    s = scenes.Scene("hull_tables", gravity=(0.0, 0.0, 0.0))
    meshes = []
    for k, (name, P, err) in enumerate(POINT_SETS):
        if err is None and k % 3 == 0:
            out = build_hull(L, np.asarray(P, np.float32))
            meshes.append(out)
            s.insert(RigidBodyBuilder.dynamic().translation((3.0 * k, 0.0, 0.0)), ColliderBuilder.convex_mesh(*out))
    w = make_world(kind, s)
    w.step()
    tabs = parse_hull_tables(w.debug_read("hull_tables", np.uint8))
    assert len(tabs) == len(s.colliders.hulls) + 1
    cube = np.array([-1, -1, -1, 1, -1, -1, 1, 1, -1, -1, 1, -1, -1, -1, 1, 1, -1, 1, 1, 1, 1, -1, 1, 1], np.float32).reshape(8, 3)
    cube_faces = [[0, 3, 2, 1], [4, 5, 6, 7], [0, 1, 5, 4], [2, 3, 7, 6], [1, 2, 6, 5], [0, 4, 7, 3]]
    check_hull_table(tabs[0], cube, cube_faces, f"{kind} unit cube")
    for i, (verts, faces) in enumerate(s.colliders.hulls):
        check_hull_table(tabs[i + 1], verts, faces, f"{kind} hull {i + 1}")


# ---- mass properties ---------------------------------------------------------------------------------------------------------
def hull_points(k):
    return [P for n, P, e in POINT_SETS if e is None][k]


def mass_scene(L):
    """One body per case (hulls built by library L); returns the scene and the case names by body."""
    s = scenes.Scene("mass_properties", gravity=(0.0, 0.0, 0.0))
    names = []
    hull = lambda k: build_hull(L, np.asarray(hull_points(k), np.float32))

    def body(name, parts, add=0.0, x=None):
        bb = RigidBodyBuilder.dynamic().translation((4.0 * len(names), 0.0, 0.0))
        if add:
            bb = bb.additional_mass(add)
        h = s.bodies.insert(bb)
        for p in parts:
            s.colliders.insert_with_parent(p, h)
        names.append(name)
    for dens in (0.0, 1e-3, 1.0, 1e3):
        body(f"ball_d{dens}", [ColliderBuilder.ball(0.37).density(dens)])
        body(f"cuboid_d{dens}", [ColliderBuilder.cuboid(0.5, 0.2, 0.11).density(dens)])
        for ax, cap in enumerate((ColliderBuilder.capsule_x, ColliderBuilder.capsule_y, ColliderBuilder.capsule_z)):
            body(f"capsule{'xyz'[ax]}_d{dens}", [cap(0.45, 0.18).density(dens)])
        body(f"hull_d{dens}", [ColliderBuilder.convex_mesh(*hull(0)).density(dens)])
    for k in range(8):
        body(f"hull_{k}", [ColliderBuilder.convex_mesh(*hull(k))])
        body(f"round_hull_{k}", [ColliderBuilder.convex_mesh(*hull(k), border_radius=0.07)])
        body(f"hull_{k}_posed", [ColliderBuilder.convex_mesh(*hull(k)).translation((0.3, -0.2, 0.45)).rotation((0.4, -1.1, 0.7))])
    body("ball_offset", [ColliderBuilder.ball(0.3).translation((0.2, 0.1, -0.3))])
    body("cuboid_posed", [ColliderBuilder.cuboid(0.4, 0.1, 0.25).translation((0.1, 0.3, 0.0)).rotation((0.3, 0.9, -0.2))])
    body("capsule_posed", [ColliderBuilder.capsule_y(0.3, 0.1).translation((-0.2, 0.0, 0.1)).rotation((1.2, 0.0, 0.4))])
    # compounds: "simple" path (axis-aligned, offsets along one axis), rotated parts, off-axis offsets (Jacobi path)
    body("compound_simple_x", [ColliderBuilder.cuboid(0.3, 0.2, 0.1).translation((-0.4, 0.0, 0.0)), ColliderBuilder.ball(0.25).translation((0.5, 0.0, 0.0)).density(2.0)])
    body("compound_simple_y", [ColliderBuilder.capsule_z(0.2, 0.1).translation((0.0, 0.6, 0.0)), ColliderBuilder.cuboid(0.2, 0.2, 0.2).translation((0.0, -0.3, 0.0))])
    body("compound_rotated", [ColliderBuilder.cuboid(0.5, 0.1, 0.1).rotation((0.0, 0.0, 0.6)), ColliderBuilder.cuboid(0.1, 0.4, 0.1).rotation((0.5, 0.0, 0.0))])
    body("compound_off_axis", [ColliderBuilder.cuboid(0.3, 0.1, 0.2).translation((0.4, 0.3, 0.0)), ColliderBuilder.ball(0.2).translation((-0.3, 0.0, 0.2)).density(3.0),
                               ColliderBuilder.capsule_x(0.2, 0.08).translation((0.0, -0.4, -0.1))])
    body("compound_two_axes", [ColliderBuilder.cuboid(0.3, 0.1, 0.2).translation((0.5, 0.4, 0.0)), ColliderBuilder.cuboid(0.3, 0.1, 0.2).translation((-0.5, -0.4, 0.0))])
    body("compound_mixed", [ColliderBuilder.cuboid(0.2, 0.3, 0.1).translation((0.1, 0.2, 0.3)).rotation((0.2, 0.3, 0.1)).density(1e3),
                            ColliderBuilder.capsule_z(0.3, 0.05).translation((-0.2, 0.1, 0.0)).rotation((0.0, 0.7, 0.0)).density(1e-3)])
    body("compound_sensor", [ColliderBuilder.cuboid(0.3, 0.2, 0.1).translation((0.2, 0.0, 0.0)), ColliderBuilder.ball(0.6).translation((1.0, 1.0, 0.0)).density(0.0).sensor()])
    body("compound_massless_part", [ColliderBuilder.ball(0.3).translation((0.2, 0.0, 0.0)), ColliderBuilder.cuboid(0.5, 0.5, 0.5).translation((0.0, 0.7, 0.4)).density(0.0)])
    body("sensor_only", [ColliderBuilder.ball(0.3).density(0.0).sensor()], add=2.5)
    # additional mass
    body("add_massive", [ColliderBuilder.cuboid(0.3, 0.2, 0.4).translation((0.1, 0.0, 0.0))], add=7.0)
    body("add_compound", [ColliderBuilder.cuboid(0.3, 0.2, 0.1).translation((0.4, 0.3, 0.0)), ColliderBuilder.ball(0.2).translation((-0.3, 0.0, 0.0))], add=3.0)
    body("add_hull", [ColliderBuilder.convex_mesh(*hull(2)).translation((0.1, 0.0, 0.2))], add=0.5)
    body("add_massless_ball", [ColliderBuilder.ball(0.3).density(0.0).translation((0.0, 0.2, 0.0))], add=4.0)
    body("add_massless_capsule", [ColliderBuilder.capsule_x(0.4, 0.1).density(0.0).rotation((0.0, 0.0, 0.5))], add=1.5)
    body("add_massless_cuboid", [ColliderBuilder.cuboid(0.3, 0.2, 0.1).density(0.0).translation((0.1, 0.1, 0.1))], add=100.0)
    body("add_colliderless", [], add=3.0)
    body("colliderless", [])
    return s, names


def test_mass_properties(kind):
    s, names = mass_scene(library(kind))
    w = make_world(kind, s)
    w.step()
    mp, mf = read_mass(w)
    for b, name in enumerate(names):
        check_body_mass(s, mp, mf, b, f"{kind} {name}")


@pytest.mark.parametrize("case", ["massless_compound", "massless_hull"])
def test_additional_mass_rejected(kind, case):
    s = scenes.Scene(case, gravity=(0.0, 0.0, 0.0))
    h = s.bodies.insert(RigidBodyBuilder.dynamic().additional_mass(2.0))
    if case == "massless_compound":
        s.colliders.insert_with_parent(ColliderBuilder.ball(0.3).density(0.0), h)
        s.colliders.insert_with_parent(ColliderBuilder.cuboid(0.2, 0.2, 0.2).density(0.0).translation((0.5, 0.0, 0.0)), h)
    else:
        s.colliders.insert_with_parent(ColliderBuilder.convex_mesh(*build_hull(library(kind), np.asarray(CUBE, np.float32))).density(0.0), h)
    assert body_mass_f64(s, h) is None
    if kind == "oracle":   # orc_world_set_scene returns RB_ERR_INVALID
        with pytest.raises(RuntimeError, match=r"^orc_world_set_scene failed: -3$"):
            make_world(kind, s)
        return
    from rapier_b200.world import RapierError
    why = "multi-collider body" if case == "massless_compound" else "convex polyhedron"
    with pytest.raises(RapierError, match=f"status -3: additional mass on a massless {why} is not supported"):
        make_world(kind, s).step()


# ---- effective world inertia ---------------------------------------------------------------------------------------------------
LOCKS = [A.RB_BODY_LOCK_TX, A.RB_BODY_LOCK_TY, A.RB_BODY_LOCK_TZ, A.RB_BODY_LOCK_RX, A.RB_BODY_LOCK_RY, A.RB_BODY_LOCK_RZ]


def test_effective_world_inertia(kind):
    rng = np.random.default_rng(11)
    s = scenes.Scene("eff_inertia", gravity=(0.0, 0.0, 0.0))
    L = library(kind)
    shapes = [ColliderBuilder.cuboid(0.4, 0.15, 0.25).translation((0.1, 0.0, 0.05)).rotation((0.3, 0.2, 0.9)),
              ColliderBuilder.convex_mesh(*build_hull(L, np.asarray(hull_points(1), np.float32))),
              ColliderBuilder.capsule_z(0.3, 0.1).rotation((0.5, 0.4, 0.0))]
    bodies, locks = [], []
    for mask in range(64):
        bits = sum(LOCKS[k] for k in range(6) if mask >> k & 1)
        h = s.bodies.insert(RigidBodyBuilder.dynamic().translation((3.0 * mask, 0.0, 0.0)).locked_axes(bits).gyroscopic_forces_enabled(False))
        s.colliders.insert_with_parent(shapes[mask % 3], h)
        bodies.append(h)
        locks.append(mask)
    for t, bt in enumerate((A.RB_BODY_FIXED, A.RB_BODY_KINEMATIC_POSITION_BASED, A.RB_BODY_KINEMATIC_VELOCITY_BASED)):
        h = s.bodies.insert(RigidBodyBuilder(bt).translation((0.0, 5.0 + 3 * t, 0.0)))
        s.colliders.insert_with_parent(shapes[t], h)
        bodies.append(h)
        locks.append(None)
    w = make_world(kind, s)
    pose, _ = w.body_states()
    pose = pose.copy()
    for i in range(len(bodies)):
        pose[i, 3:7] = axis_angle_quat(rng.uniform(-np.pi, np.pi, 3))
    w.set_body_states(np.arange(len(bodies)), pose, np.zeros((len(bodies), 6), np.float32))
    for stage in ("set_body_states", "step"):
        if stage == "step":
            w.step()
        pose = w.body_states()[0].astype(np.float64)
        mp, mf = read_mass(w)
        for i, (b, mask) in enumerate(zip(bodies, locks)):
            where = f"{kind} {stage} body {b} locks {mask}"
            eii = mp[b, 10:16]
            E = np.array([[eii[0], eii[1], eii[2]], [eii[1], eii[3], eii[4]], [eii[2], eii[4], eii[5]]])
            if mask is None:
                assert not E.any() and not mf[b, 4:7].any(), f"{where}: non-dynamic body has effective masses"
                continue
            M, _, I = body_mass_f64(s, b)
            Rb = qmat(pose[b, 3:7])
            ref = Rb @ np.linalg.inv(I) @ Rb.T
            eim = np.full(3, 1.0 / M)
            for k in range(3):
                if mask >> (3 + k) & 1:
                    ref[k, :] = 0.0
                    ref[:, k] = 0.0
                if mask >> k & 1:
                    eim[k] = 0.0
            r = np.abs(E - ref).max() / (U * np.abs(Rb @ np.linalg.inv(I) @ Rb.T).max())
            WORST["eii"] = max(WORST["eii"], r)
            assert r <= TOL_MP, f"{where}: effective world inverse inertia\n{E}\nvs\n{ref}\n({r:.1f} u)"
            for k in range(3):
                if mask >> (3 + k) & 1:
                    assert not E[k].any() and not E[:, k].any(), f"{where}: locked rotation axis {k} not zeroed exactly"
            assert np.abs(mf[b, 4:7] - eim).max() <= TOL_MP * U / M and ((mf[b, 4:7] == 0.0) == (eim == 0.0)).all(), \
                f"{where}: effective inverse mass {mf[b, 4:7]} vs {eim}"
