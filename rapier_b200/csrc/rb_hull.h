// rb_hull.h -- host side of convex polyhedra: validation of a convex mesh, derived tables (planes, edges), mass
// properties, and a small convex-hull builder.  Host code only (compiled into the library and into the emulation build).
//
// Replaces parry3d 0.30.2 `ConvexPolyhedron::from_convex_hull / from_convex_mesh`, `MassProperties::from_convex_polyhedron`
// and `transformation::convex_hull` as reached from ColliderBuilder::{convex_hull, convex_mesh, round_convex_hull}
// (src/geometry/collider.rs:1039-1090); parry is not in the tree, so these are first-principles restatements:
// signed-tetrahedron integration for volume / centre of mass / inertia tensor, a cyclic Jacobi diagonalisation for the
// principal axes, and a brute-force supporting-plane search for the hull of at most 32 points.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <vector>

namespace rbhull {

constexpr int MAX_VERTS = 32, MAX_FACES = 32, MAX_FACE_VERTS = 8, MAX_EDGES = 64;
constexpr double REPEAT_EPS = 4.0;   // convex_hull: repeat radius of the input points, in units of its plane tolerance

struct Hull {
    std::vector<float> verts;                 // 3 * nv
    std::vector<int> face_start, face_count;  // into loops
    std::vector<int> loops;
    std::vector<float> planes;                // 4 * nf: outward unit normal, offset
    std::vector<int> edges;                   // 4 * ne: v0, v1, face running v0 -> v1, the other face
    // mass properties at unit density (about the centre of mass, in the hull's frame)
    float volume, com[3], principal_inertia[3], principal_frame[4];
    float aabb[3], radius;                    // max |coordinate| per axis, max |v| (both about the origin)
    int nv() const { return (int)verts.size() / 3; }
    int nf() const { return (int)face_count.size(); }
    int ne() const { return (int)edges.size() / 4; }
};

inline void cross3d(const double a[3], const double b[3], double o[3]) {
    o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
inline double dot3d(const double a[3], const double b[3]) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// Cyclic Jacobi diagonalisation of a symmetric 3x3 matrix: a = v diag(w) v^T (columns of v = eigenvectors).
inline void jacobi3(double a[3][3], double v[3][3], double w[3]) {
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) v[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 32; ++sweep) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        const double diag = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
        if (off <= 1.0e-30 * diag || off == 0.0) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (a[p][q] == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
                const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {   // a <- a J
                    const double akp = a[k][p], akq = a[k][q];
                    a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {   // a <- J^T a
                    const double apk = a[p][k], aqk = a[q][k];
                    a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const double vkp = v[k][p], vkq = v[k][q];
                    v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq;
                }
            }
    }
    for (int i = 0; i < 3; ++i) w[i] = a[i][i];
}

// Rotation matrix (columns = axes, right-handed) to a unit quaternion (x, y, z, w).
inline void mat_to_quat(const double m[3][3], float q[4]) {
    const double tr = m[0][0] + m[1][1] + m[2][2];
    double x, y, z, w;
    if (tr > 0.0) {
        const double s = std::sqrt(tr + 1.0) * 2.0;
        w = 0.25 * s; x = (m[2][1] - m[1][2]) / s; y = (m[0][2] - m[2][0]) / s; z = (m[1][0] - m[0][1]) / s;
    } else if (m[0][0] > m[1][1] && m[0][0] > m[2][2]) {
        const double s = std::sqrt(1.0 + m[0][0] - m[1][1] - m[2][2]) * 2.0;
        w = (m[2][1] - m[1][2]) / s; x = 0.25 * s; y = (m[0][1] + m[1][0]) / s; z = (m[0][2] + m[2][0]) / s;
    } else if (m[1][1] > m[2][2]) {
        const double s = std::sqrt(1.0 + m[1][1] - m[0][0] - m[2][2]) * 2.0;
        w = (m[0][2] - m[2][0]) / s; x = (m[0][1] + m[1][0]) / s; y = 0.25 * s; z = (m[1][2] + m[2][1]) / s;
    } else {
        const double s = std::sqrt(1.0 + m[2][2] - m[0][0] - m[1][1]) * 2.0;
        w = (m[1][0] - m[0][1]) / s; x = (m[0][2] + m[2][0]) / s; y = (m[1][2] + m[2][1]) / s; z = 0.25 * s;
    }
    const double n = std::sqrt(x * x + y * y + z * z + w * w);
    q[0] = (float)(x / n); q[1] = (float)(y / n); q[2] = (float)(z / n); q[3] = (float)(w / n);
}

// Volume, centre of mass and principal inertia of the polyhedron at unit density.
inline bool mass_properties(Hull& h) {
    double vol = 0.0, com[3] = {0, 0, 0}, C[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};   // C = integral of x x^T
    for (int f = 0; f < h.nf(); ++f) {
        const int s = h.face_start[f], n = h.face_count[f];
        double a[3];
        for (int k = 0; k < 3; ++k) a[k] = h.verts[3 * h.loops[s] + k];
        for (int i = 1; i + 1 < n; ++i) {
            double b[3], c[3], bc[3];
            for (int k = 0; k < 3; ++k) { b[k] = h.verts[3 * h.loops[s + i] + k]; c[k] = h.verts[3 * h.loops[s + i + 1] + k]; }
            cross3d(b, c, bc);
            const double det = dot3d(a, bc);   // 6 x the signed volume of (origin, a, b, c)
            vol += det / 6.0;
            double sum[3];
            for (int k = 0; k < 3; ++k) { sum[k] = a[k] + b[k] + c[k]; com[k] += det * sum[k] / 24.0; }
            for (int r = 0; r < 3; ++r)
                for (int t = 0; t < 3; ++t) C[r][t] += det / 120.0 * (a[r] * a[t] + b[r] * b[t] + c[r] * c[t] + sum[r] * sum[t]);
        }
    }
    if (!(vol > 1.0e-12)) return false;
    for (int k = 0; k < 3; ++k) com[k] /= vol;
    double I[3][3];
    const double trc = C[0][0] + C[1][1] + C[2][2], c2 = dot3d(com, com);
    for (int r = 0; r < 3; ++r)
        for (int t = 0; t < 3; ++t) I[r][t] = (r == t ? trc : 0.0) - C[r][t] - vol * ((r == t ? c2 : 0.0) - com[r] * com[t]);
    double v[3][3], w[3];
    jacobi3(I, v, w);
    // right-handed frame
    double x0[3] = {v[0][0], v[1][0], v[2][0]}, x1[3] = {v[0][1], v[1][1], v[2][1]}, x2[3] = {v[0][2], v[1][2], v[2][2]}, cr[3];
    cross3d(x0, x1, cr);
    if (dot3d(cr, x2) < 0.0) for (int k = 0; k < 3; ++k) v[k][2] = -v[k][2];
    h.volume = (float)vol;
    for (int k = 0; k < 3; ++k) { h.com[k] = (float)com[k]; h.principal_inertia[k] = (float)(w[k] > 0.0 ? w[k] : 0.0); }
    mat_to_quat(v, h.principal_frame);
    return true;
}

// Derives planes, edges, bounds and mass properties of a closed convex mesh; checks its limits, winding and convexity.
// Returns nullptr on success, else what is wrong.
inline const char* from_mesh(int nv, const float* verts, int nf, const int32_t* face_sizes, const int32_t* face_indices, Hull& h) {
    if (nv < 4 || nv > MAX_VERTS) return "a convex polyhedron needs 4..32 vertices";
    if (nf < 4 || nf > MAX_FACES) return "a convex polyhedron needs 4..32 faces";
    h = Hull();
    h.verts.assign(verts, verts + 3 * nv);
    for (int i = 0; i < 3 * nv; ++i) if (!std::isfinite(verts[i])) return "non-finite vertex";
    double centroid[3] = {0, 0, 0};
    for (int i = 0; i < nv; ++i) for (int k = 0; k < 3; ++k) centroid[k] += verts[3 * i + k] / nv;
    int at = 0;
    for (int f = 0; f < nf; ++f) {
        const int n = face_sizes[f];
        if (n < 3 || n > MAX_FACE_VERTS) return "faces need 3..8 vertices";
        std::vector<int> loop(face_indices + at, face_indices + at + n);
        at += n;
        for (int k = 0; k < n; ++k) if (loop[k] < 0 || loop[k] >= nv) return "face index out of range";
        // Newell normal
        double nn[3] = {0, 0, 0}, mid[3] = {0, 0, 0};
        for (int k = 0; k < n; ++k) {
            const float* p = verts + 3 * loop[k];
            const float* q = verts + 3 * loop[(k + 1) % n];
            nn[0] += ((double)p[1] - q[1]) * ((double)p[2] + q[2]);
            nn[1] += ((double)p[2] - q[2]) * ((double)p[0] + q[0]);
            nn[2] += ((double)p[0] - q[0]) * ((double)p[1] + q[1]);
            for (int c = 0; c < 3; ++c) mid[c] += (double)p[c] / n;
        }
        const double len = std::sqrt(dot3d(nn, nn));
        if (!(len > 1.0e-12)) return "degenerate face";
        for (int c = 0; c < 3; ++c) nn[c] /= len;
        double d = dot3d(nn, mid);
        if (dot3d(nn, centroid) - d > 0.0) {   // wound clockwise: turn it round
            std::reverse(loop.begin(), loop.end());
            for (int c = 0; c < 3; ++c) nn[c] = -nn[c];
            d = -d;
        }
        h.face_start.push_back((int)h.loops.size());
        h.face_count.push_back(n);
        h.loops.insert(h.loops.end(), loop.begin(), loop.end());
        for (int c = 0; c < 3; ++c) h.planes.push_back((float)nn[c]);
        h.planes.push_back((float)d);
    }
    // convexity: every vertex behind every face (to a tolerance relative to the size)
    double size = 0.0;
    for (int i = 0; i < 3 * nv; ++i) size = std::max(size, (double)std::fabs(verts[i]));
    for (int f = 0; f < nf; ++f)
        for (int i = 0; i < nv; ++i) {
            const double s = (double)h.planes[4 * f] * verts[3 * i] + (double)h.planes[4 * f + 1] * verts[3 * i + 1] + (double)h.planes[4 * f + 2] * verts[3 * i + 2] - h.planes[4 * f + 3];
            if (s > 1.0e-4 * (1.0 + size)) return "the mesh is not convex";
        }
    // edges: every directed edge of a loop pairs with the reversed edge of exactly one other face
    std::map<std::pair<int, int>, int> directed;
    for (int f = 0; f < nf; ++f)
        for (int k = 0; k < h.face_count[f]; ++k) {
            const int a = h.loops[h.face_start[f] + k], b = h.loops[h.face_start[f] + (k + 1) % h.face_count[f]];
            if (a == b || directed.count({a, b})) return "the mesh is not a closed 2-manifold";
            directed[{a, b}] = f;
        }
    for (const auto& kv : directed) {
        const int a = kv.first.first, b = kv.first.second;
        auto opp = directed.find({b, a});
        if (opp == directed.end()) return "the mesh is not closed";
        if (a < b) { h.edges.push_back(a); h.edges.push_back(b); h.edges.push_back(kv.second); h.edges.push_back(opp->second); }
    }
    if (h.ne() > MAX_EDGES) return "a convex polyhedron may have at most 64 edges";
    h.aabb[0] = h.aabb[1] = h.aabb[2] = h.radius = 0.0f;
    for (int i = 0; i < nv; ++i) {
        const float* p = verts + 3 * i;
        for (int k = 0; k < 3; ++k) h.aabb[k] = std::max(h.aabb[k], std::fabs(p[k]));
        h.radius = std::max(h.radius, std::sqrt(std::fma(p[2], p[2], std::fma(p[1], p[1], p[0] * p[0]))));
    }
    if (!mass_properties(h)) return "the polyhedron has no volume";
    return nullptr;
}

inline void unit_cube(Hull& h) {
    const float v[24] = {-1, -1, -1, 1, -1, -1, 1, 1, -1, -1, 1, -1, -1, -1, 1, 1, -1, 1, 1, 1, 1, -1, 1, 1};
    const int32_t sizes[6] = {4, 4, 4, 4, 4, 4};
    const int32_t idx[24] = {0, 3, 2, 1, 4, 5, 6, 7, 0, 1, 5, 4, 2, 3, 7, 6, 1, 2, 6, 5, 0, 4, 7, 3};
    from_mesh(8, v, 6, sizes, idx, h);
}

// Convex hull of at most 32 points by supporting-plane search: every plane through three points that leaves all the
// others on one side carries a face; the points on it (to a tolerance) are ordered into a convex polygon.
inline const char* convex_hull(int np, const float* pts, std::vector<float>& out_verts, std::vector<int32_t>& sizes, std::vector<int32_t>& indices) {
    if (np < 4 || np > MAX_VERTS) return "convex_hull takes 4..32 points";
    double size = 0.0;
    for (int i = 0; i < 3 * np; ++i) { if (!std::isfinite(pts[i])) return "non-finite point"; size = std::max(size, (double)std::fabs(pts[i])); }
    const double eps = 1.0e-6 * (1.0 + size);
    auto P = [&](int i, double o[3]) { for (int k = 0; k < 3; ++k) o[k] = pts[3 * i + k]; };
    // A repeated point -- within REPEAT_EPS * eps of an earlier kept one in every coordinate -- takes no part (the earlier
    // one stands for it).  Two such copies of one corner are both on or near every plane through it, and the faces around
    // that corner would not all keep the same copy, leaving the mesh open; up to a few eps apart the tolerances of the plane
    // membership and of the polygon turns still disagree about them.
    const double rep = REPEAT_EPS * eps;
    std::vector<char> dup(np, 0);
    for (int i = 0; i < np; ++i)
        for (int j = 0; j < i && !dup[i]; ++j)
            dup[i] = !dup[j] && std::fabs((double)pts[3 * i] - pts[3 * j]) <= rep && std::fabs((double)pts[3 * i + 1] - pts[3 * j + 1]) <= rep &&
                     std::fabs((double)pts[3 * i + 2] - pts[3 * j + 2]) <= rep;
    std::vector<uint32_t> seen;            // vertex masks of the faces found
    std::vector<std::vector<int>> faces;
    for (int i = 0; i < np; ++i)
        for (int j = i + 1; j < np; ++j)
            for (int k = j + 1; k < np; ++k) {
                if (dup[i] || dup[j] || dup[k]) continue;
                double a[3], b[3], c[3], ab[3], ac[3], n[3];
                P(i, a); P(j, b); P(k, c);
                for (int t = 0; t < 3; ++t) { ab[t] = b[t] - a[t]; ac[t] = c[t] - a[t]; }
                cross3d(ab, ac, n);
                const double len = std::sqrt(dot3d(n, n));
                if (!(len > 1.0e-9 * (1.0 + size * size))) continue;
                for (int t = 0; t < 3; ++t) n[t] /= len;
                const double d = dot3d(n, a);
                int pos = 0, neg = 0;
                uint32_t mask = 0;
                for (int m = 0; m < np; ++m) {
                    if (dup[m]) continue;
                    double q[3];
                    P(m, q);
                    const double s = dot3d(n, q) - d;
                    if (s > eps) pos++; else if (s < -eps) neg++; else mask |= 1u << m;
                }
                if (pos && neg) continue;
                if (std::find(seen.begin(), seen.end(), mask) != seen.end()) continue;
                seen.push_back(mask);
                if (pos) for (int t = 0; t < 3; ++t) n[t] = -n[t];   // outward: all the other points behind
                // order the coplanar points: 2-D hull (monotone chain) in a basis of the plane
                double u[3] = {ab[0], ab[1], ab[2]}, w[3];
                const double ul = std::sqrt(dot3d(u, u));
                for (int t = 0; t < 3; ++t) u[t] /= ul;
                cross3d(n, u, w);
                std::vector<std::pair<std::pair<double, double>, int>> p2;
                for (int m = 0; m < np; ++m)
                    if (mask >> m & 1) { double q[3]; P(m, q); p2.push_back({{dot3d(q, u), dot3d(q, w)}, m}); }
                std::sort(p2.begin(), p2.end());
                auto turn = [&](int o, int x, int y) {
                    return (p2[x].first.first - p2[o].first.first) * (p2[y].first.second - p2[o].first.second) -
                           (p2[x].first.second - p2[o].first.second) * (p2[y].first.first - p2[o].first.first);
                };
                std::vector<int> hull;
                const int m2 = (int)p2.size();
                for (int pass = 0; pass < 2; ++pass) {
                    const size_t base = hull.size();
                    for (int x = 0; x < m2; ++x) {
                        const int idx = pass == 0 ? x : m2 - 1 - x;
                        while (hull.size() >= base + 2 && turn(hull[hull.size() - 2], hull[hull.size() - 1], idx) <= eps * (1.0 + size)) hull.pop_back();
                        hull.push_back(idx);
                    }
                    hull.pop_back();
                }
                if (hull.size() < 3) continue;
                std::vector<int> loop;
                for (int x : hull) loop.push_back(p2[x].second);   // counter-clockwise about n (u x w = n)
                faces.push_back(loop);
            }
    if (faces.size() < 4) return "the points are coplanar";
    // keep the points that are a corner of some face, renumbered in input order
    std::vector<int> remap(np, -1);
    for (const auto& f : faces) for (int v : f) remap[v] = 0;
    int nv = 0;
    out_verts.clear();
    for (int i = 0; i < np; ++i)
        if (remap[i] == 0) { remap[i] = nv++; for (int k = 0; k < 3; ++k) out_verts.push_back(pts[3 * i + k]); }
    sizes.clear(); indices.clear();
    for (const auto& f : faces) {
        if ((int)f.size() > MAX_FACE_VERTS) return "a face of the hull has more than 8 vertices";
        sizes.push_back((int32_t)f.size());
        for (int v : f) indices.push_back(remap[v]);
    }
    if ((int)faces.size() > MAX_FACES) return "the hull has more than 32 faces";
    return nullptr;
}

}  // namespace rbhull
