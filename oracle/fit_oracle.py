"""Numpy restatement of the grid-fitting kernels (meshdiffusion_b200/csrc/fit.cu): space carving (`mdb_carve_vertices`),
closest points on a triangle mesh (`mdb_closest_points`) and nearest points of a point set (`mdb_nearest_vertex`).

In float32 every product, sum and quotient is a numpy operation rounded on its own, in the kernels' order, so the results
match the kernels bit for bit. `closest_points(..., dtype=np.float64)` is the same algorithm in float64, the accuracy
yardstick. Pure numpy: also runs without a GPU.
"""
import numpy as np

F32 = np.float32


def mvp_rows(m, p):
    """clip [..., 4] = m [4, 4] (row-major) times [p, 1]: per row ((m0 x + m1 y) + m2 z) + m3."""
    m = np.asarray(m, F32).reshape(4, 4)
    p = np.asarray(p, F32)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return np.stack([((m[i, 0] * x + m[i, 1] * y) + m[i, 2] * z) + m[i, 3] for i in range(4)], -1).astype(F32)


def carve(pts, mvps, depth, face_id, window):
    """One mesh: pts [N, 3], mvps [V, 4, 4], depth / face_id [V, res, res] -> outside bool [N] (a view sees the vertex)."""
    pts = np.asarray(pts, F32)
    V, res = depth.shape[0], depth.shape[-1]
    fres = F32(res)
    outside = np.zeros(pts.shape[0], bool)
    for v in range(V):
        h = mvp_rows(mvps[v], pts)
        w = h[:, 3]
        with np.errstate(all="ignore"):
            X = ((h[:, 0] / w) * F32(0.5) + F32(0.5)) * fres
            Y = ((h[:, 1] / w) * F32(0.5) + F32(0.5)) * fres
            z = h[:, 2] / w
        ok = (w > 0) & (X >= 0) & (X < fres) & (Y >= 0) & (Y < fres) & ~outside
        for i in np.nonzero(ok)[0]:
            c, r = int(X[i]), int(Y[i])
            sl = (v, slice(max(r - window, 0), min(r + window, res - 1) + 1), slice(max(c - window, 0), min(c + window, res - 1) + 1))
            outside[i] = bool(((face_id[sl] < 0) | (depth[sl] > z[i])).all())
    return outside


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _axpy(a, s, d):
    return a + s[..., None] * d


def _segment(p, a, b):
    ab = b - a
    den = _dot(ab, ab)
    with np.errstate(all="ignore"):
        t = np.where(den > 0, _dot(p - a, ab) / np.where(den > 0, den, 1), 0).astype(p.dtype)
    t = np.fmin(np.fmax(t, 0), 1).astype(p.dtype)
    return _axpy(a, t, ab)


def closest_on_triangles(p, a, b, c):
    """Closest points [..., 3] of p on triangles abc (broadcasting), in p's dtype, in the kernel's order of operations."""
    dt = p.dtype
    with np.errstate(all="ignore"):
        ab, ac, ap = b - a, c - a, p - a
        d1, d2 = _dot(ab, ap), _dot(ac, ap)
        bp = p - b
        d3, d4 = _dot(ab, bp), _dot(ac, bp)
        vc = d1 * d4 - d3 * d2
        cp = p - c
        d5, d6 = _dot(ab, cp), _dot(ac, cp)
        vb = d5 * d2 - d1 * d6
        va = d3 * d6 - d5 * d4
        e43, e56 = d4 - d3, d5 - d6
        den = (va + vb) + vc
        shape = np.broadcast_shapes(a.shape, p.shape)
        cases = [
            (d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0),
            (d6 >= 0) & (d5 <= d6), (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0),
        ]
        values = [
            lambda: np.broadcast_to(a, shape), lambda: np.broadcast_to(b, shape), lambda: _axpy(a, d1 / (d1 - d3), ab),
            lambda: np.broadcast_to(c, shape), lambda: _axpy(a, d2 / (d2 - d6), ac), lambda: _axpy(b, e43 / (e43 + e56), c - b),
            lambda: np.where((den > 0)[..., None], _axpy(_axpy(a, vb / den, ab), vc / den, ac), np.nan),
        ]
        r = np.full(shape, np.nan, dt)
        case =np.full(shape[:-1], len(cases), np.int8)  # the region that applies first, in the kernel's order
        for k in reversed(range(len(cases))):
            case = np.where(cases[k], k, case)
        for k, val in enumerate(values):
            if (case == k).any():
                r = np.where((case == k)[..., None], np.asarray(val(), dt), r)
        # the vertex regions (0, 1, 3) return the vertex itself; the others fall back to the edges unless finite
        bad = ~np.isfinite(r).all(-1) & (case != 0) & (case != 1) & (case != 3)
        if bad.any():
            s0, s1, s2 = _segment(p, a, b), _segment(p, b, c), _segment(p, c, a)
            q0, q1, q2 = _dot(p - s0, p - s0), _dot(p - s1, p - s1), _dot(p - s2, p - s2)
            fb = np.where((q1 < q0)[..., None], s1, s0)
            q = np.where(q1 < q0, q1, q0)
            fb = np.where((q2 < q)[..., None], s2, fb)
            r = np.where(bad[..., None], fb, r)
    return r.astype(dt)


def closest_points(queries, verts, faces, dtype=F32, chunk=1 << 21):
    """One mesh: queries [Q, 3] -> (dist2 [Q], face int64 [Q], closest [Q, 3]) as mdb_closest_points computes them (dtype
    float32) or the same algorithm in float64."""
    q = np.asarray(queries, dtype)
    v = np.asarray(verts, dtype)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    Q, F = q.shape[0], f.shape[0]
    best = np.full(Q, np.inf, dtype)
    best_f = np.full(Q, -1, np.int64)
    best_c = np.full((Q, 3), np.nan, dtype)
    step = max(1, chunk // max(1, Q))
    for s in range(0, F, step):
        ff = f[s:s + step]
        a, b, c = v[ff[:, 0]][:, None], v[ff[:, 1]][:, None], v[ff[:, 2]][:, None]  # [f, 1, 3]
        cp = closest_on_triangles(q[None], a, b, c)                                 # [f, Q, 3]
        d = _dot(q[None] - cp, q[None] - cp)
        d = np.where(np.isnan(d), np.inf, d)
        k = np.argmin(d, 0)                                                          # first minimum: the lower face
        dk = d[k, np.arange(Q)]
        better = dk < best
        best = np.where(better, dk, best)
        best_f = np.where(better, s + k, best_f)
        best_c = np.where(better[:, None], cp[k, np.arange(Q)], best_c)
    return best.astype(dtype), best_f, best_c.astype(dtype)


def nearest_vertex(queries, points):
    """One point set: queries [Q, 3] -> (dist2 fp32 [Q], index int64 [Q]) as mdb_nearest_vertex computes them."""
    q = np.asarray(queries, F32)
    p = np.asarray(points, F32)
    if p.shape[0] == 0:
        return np.full(q.shape[0], np.inf, F32), np.full(q.shape[0], -1, np.int64)
    d = q[:, None] - p[None]
    d2 = _dot(d, d)
    d2 = np.where(np.isnan(d2), np.inf, d2)
    k = np.argmin(d2, 1)  # the first minimum: the lower index
    best = d2[np.arange(q.shape[0]), k].astype(F32)
    return best, np.where(best < np.inf, k, -1).astype(np.int64)


# ---- analytic test shapes: (verts fp32 [V, 3], faces int64 [F, 3]) and the signed distance they approximate (> 0 inside)

def icosphere(radius=0.45, subdiv=4, centre=(0.0, 0.0, 0.0)):
    t = (1.0 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7],
         [9, 8, 1]]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdiv):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return (np.stack(v) * radius + np.asarray(centre)).astype(F32), np.asarray(f, np.int64)


def sphere_sdf(p, radius=0.45, centre=(0.0, 0.0, 0.0)):
    return radius - np.linalg.norm(np.asarray(p, np.float64) - np.asarray(centre), axis=-1)


def torus(major=0.32, minor=0.13, n_major=96, n_minor=48):
    """Around the y axis."""
    u, w = np.meshgrid(np.arange(n_major) * 2 * np.pi / n_major, np.arange(n_minor) * 2 * np.pi / n_minor, indexing="ij")
    rho = major + minor * np.cos(w)
    v = np.stack([rho * np.cos(u), minor * np.sin(w), rho * np.sin(u)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n_major), np.arange(n_minor), indexing="ij")
    a = i * n_minor + j
    b = ((i + 1) % n_major) * n_minor + j
    c = ((i + 1) % n_major) * n_minor + (j + 1) % n_minor
    d = i * n_minor + (j + 1) % n_minor
    f = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)])
    return v.astype(F32), f.astype(np.int64)


def torus_sdf(p, major=0.32, minor=0.13):
    p = np.asarray(p, np.float64)
    rho = np.hypot(p[..., 0], p[..., 2])
    return minor - np.hypot(rho - major, p[..., 1])


def box(half=0.4, open_top=False):
    """Axis-aligned cube [-half, half]^3, two triangles a side, outward winding; open_top drops the +y side."""
    v = np.array([[x, y, z] for x in (-half, half) for y in (-half, half) for z in (-half, half)], F32)
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]  # -x +x -y +y -z +z
    if open_top:
        quads.pop(3)
    f = [[q[0], q[1], q[2]] for q in quads] + [[q[0], q[2], q[3]] for q in quads]
    return v, np.asarray(f, np.int64)


def box_sdf(p, half=0.4):
    return half - np.abs(np.asarray(p, np.float64)).max(-1)
