"""Float32 numpy restatement of the depth-map kernels (meshdiffusion_b200/csrc/depth_partial.cu): back-projection of a
camera depth map (`mdb_depth_unproject`) and the closest point on the observed surface in an image-space window
(`mdb_depth_closest_points`).

Every product, sum and quotient is a float32 numpy operation rounded on its own, in the kernels' order, so the buffers,
flags, distances and points match the kernels bit for bit. `triangulation` is the whole observed surface as a mesh,
for a brute-force search (fit_oracle.closest_points), the yardstick of the window rule. Pure numpy: also runs without a
GPU.
"""
import numpy as np

from oracle.fit_oracle import _dot, closest_on_triangles, mvp_rows

F32 = np.float32
EMPTY_DEPTH = F32(100.0)
MAX_HALF = 31


def _observed(d):
    return np.isfinite(d) & (d > 0)


def unproject(depth, proj, inv_mv, max_jump):
    """One observation: depth fp32 [res, res], proj / inv_mv [4, 4] -> (zbuf fp32, valid int32, points fp32 [res, res, 3],
    edge uint8), as mdb_depth_unproject writes them."""
    d = np.asarray(depth, F32)
    res = d.shape[0]
    P = np.asarray(proj, F32).reshape(4, 4)
    ok = _observed(d)
    ds = np.where(ok, d, F32(1))
    fres = F32(res)
    idx = np.arange(res, dtype=F32)
    xn = ((idx + F32(0.5)) / fres) * F32(2) - F32(1)
    xn, yn = np.broadcast_to(xn[None, :], d.shape), np.broadcast_to(xn[:, None], d.shape)
    xc = (ds * (xn + P[0, 2])) / P[0, 0]
    yc = (ds * (yn + P[1, 2])) / P[1, 1]
    cam = np.stack([xc, yc, -ds], -1).astype(F32)
    world = mvp_rows(inv_mv, cam)[..., :3]
    points = np.where(ok[..., None], world, F32(0)).astype(F32)
    zbuf = np.where(ok, (P[2, 3] - P[2, 2] * ds) / ds, EMPTY_DEPTH).astype(F32)
    valid = np.where(ok, 0, -1).astype(np.int32)
    jump = F32(max_jump)
    edge = np.zeros(d.shape, bool)
    pad = np.pad(d, 1, constant_values=np.nan)
    for dr, dc in ((0, -1), (0, 1), (-1, 0), (1, 0)):
        n = pad[1 + dr:1 + dr + res, 1 + dc:1 + dc + res]
        with np.errstate(invalid="ignore"):
            edge |= _observed(n) & (np.abs(d - n) > jump)
    return zbuf, valid, points, (edge & ok).astype(np.uint8)


def usable(valid, edge):
    return (np.asarray(valid) == 0) & (np.asarray(edge) == 0)


def _block_triangles(points, use, r0, r1, c0, c1):
    """Triangles of the usable blocks of rows r0..r1, columns c0..c1 in the kernel's order -> a, b, c [n, 3]."""
    rr, cc = np.meshgrid(np.arange(r0, r1 + 1), np.arange(c0, c1 + 1), indexing="ij")
    rr, cc = rr.reshape(-1), cc.reshape(-1)
    ok = use[rr, cc] & use[rr, cc + 1] & use[rr + 1, cc] & use[rr + 1, cc + 1]
    rr, cc = rr[ok], cc[ok]
    p00, p01, p10, p11 = points[rr, cc], points[rr, cc + 1], points[rr + 1, cc], points[rr + 1, cc + 1]
    a = np.stack([p00, p00], 1).reshape(-1, 3)
    b = np.stack([p01, p11], 1).reshape(-1, 3)
    c = np.stack([p11, p10], 1).reshape(-1, 3)
    return a, b, c


def _nearest(q, a, b, c):
    if a.shape[0] == 0:
        return np.inf, np.full(3, np.nan, F32), False
    cp = closest_on_triangles(q[None], a, b, c)
    d = _dot(q[None] - cp, q[None] - cp)
    d = np.where(np.isnan(d), np.inf, d)
    k = int(np.argmin(d))  # the first minimum: the lower pixel, then the first triangle
    if not d[k] < np.inf:
        return np.inf, np.full(3, np.nan, F32), False
    return d[k], cp[k], True


def window(q, mvp, proj, res, radius):
    """(r0, r1, c0, c1) of the query's block window, or None when the kernel skips the query."""
    h = mvp_rows(mvp, np.asarray(q, F32)[None])[0]
    w = h[3]
    if not w > 0:
        return None
    P = np.asarray(proj, F32).reshape(4, 4)
    fres = F32(res)
    X = ((h[0] / w) * F32(0.5) + F32(0.5)) * fres
    Y = ((h[1] / w) * F32(0.5) + F32(0.5)) * fres
    scale = (np.maximum(np.abs(P[0, 0]), np.abs(P[1, 1])) * F32(0.5)) * fres
    hp = (F32(radius) * scale) / w
    if not (X > -64 and X < fres + 64 and Y > -64 and Y < fres + 64):
        return None
    half = MAX_HALF if hp >= MAX_HALF else int(np.ceil(hp))
    cq, rq = int(np.floor(X - F32(0.5))), int(np.floor(Y - F32(0.5)))
    return max(rq - half, 0), min(rq + half, res - 2), max(cq - half, 0), min(cq + half, res - 2)


def closest_points(queries, mvp, proj, radius, points, valid, edge):
    """One observation: queries [Q, 3] -> (dist2 fp32 [Q], closest fp32 [Q, 3], found bool [Q]) as
    mdb_depth_closest_points computes them."""
    q = np.asarray(queries, F32).reshape(-1, 3)
    points = np.asarray(points, F32)
    res = points.shape[0]
    use = usable(valid, edge)
    d2 = np.full(q.shape[0], np.inf, F32)
    cp = np.full((q.shape[0], 3), np.nan, F32)
    found = np.zeros(q.shape[0], bool)
    with np.errstate(all="ignore"):
        for i in range(q.shape[0]):
            win = window(q[i], mvp, proj, res, radius)
            if win is None or win[0] > win[1] or win[2] > win[3]:
                continue
            d2[i], cp[i], found[i] = _nearest(q[i], *_block_triangles(points, use, *win))
    return d2, cp, found


def triangulation(points, valid, edge):
    """The observed surface as a mesh (verts [res * res, 3], faces [F, 3]) in the kernel's triangle order."""
    points = np.asarray(points, F32)
    res = points.shape[0]
    use = usable(valid, edge)
    rr, cc = np.meshgrid(np.arange(res - 1), np.arange(res - 1), indexing="ij")
    rr, cc = rr.reshape(-1), cc.reshape(-1)
    ok = use[rr, cc] & use[rr, cc + 1] & use[rr + 1, cc] & use[rr + 1, cc + 1]
    k00 = (rr * res + cc)[ok]
    k01, k10, k11 = k00 + 1, k00 + res, k00 + res + 1
    faces = np.stack([np.stack([k00, k01, k11], 1), np.stack([k00, k11, k10], 1)], 1).reshape(-1, 3)
    return points.reshape(-1, 3), faces.astype(np.int64)
