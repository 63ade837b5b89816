"""Float32 numpy restatement of the single-view visibility kernels (meshdiffusion_b200/csrc/raster.cu): the first-layer
depth / face-id rasterizer (`mdb_raster_depth`) and the visible-tet test (`mdb_visible_tets`).

Every product, sum and quotient is a float32 numpy operation, rounded on its own, in the kernels' order, so the buffers
and flags match the kernels bit for bit. Pure numpy: also runs without a GPU.
"""
import numpy as np

F32 = np.float32
EMPTY_DEPTH = F32(100.0)
WINDOW = 7


def mvp_rows(m, p):
    """clip [..., 4] = m [4, 4] (row-major) times [p, 1] for p [..., 3]: per row ((m0 x + m1 y) + m2 z) + m3."""
    m = np.asarray(m, F32).reshape(4, 4)
    p = np.asarray(p, F32)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    return np.stack([((m[i, 0] * x + m[i, 1] * y) + m[i, 2] * z) + m[i, 3] for i in range(4)], -1).astype(F32)


def edge_fn(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def setup(verts, faces, mvp, res):
    """Per face: screen x, y [F, 3], z / w [F, 3], area [F], drawn [F], behind [F] (a vertex with w <= 0)."""
    clip = mvp_rows(mvp, np.asarray(verts, F32)[np.asarray(faces, np.int64)])  # [F, 3, 4]
    w = clip[..., 3]
    behind = ~(w > 0).all(axis=1)
    with np.errstate(all="ignore"):
        x = ((clip[..., 0] / w) * F32(0.5) + F32(0.5)) * F32(res)
        y = ((clip[..., 1] / w) * F32(0.5) + F32(0.5)) * F32(res)
        z = clip[..., 2] / w
        finite = np.isfinite(x).all(1) & np.isfinite(y).all(1) & np.isfinite(z).all(1)
        area = edge_fn(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2])
    drawn = ~behind & finite & np.isfinite(area) & (area != 0)
    return x, y, z, area, drawn, behind


def fragment(x, y, z, area, px, py):
    """(covered, depth) of faces (x, y, z [..., 3], area [...]) at pixel centres (px, py), broadcasting."""
    with np.errstate(all="ignore"):
        inbox = (px >= x.min(-1)) & (px <= x.max(-1)) & (py >= y.min(-1)) & (py <= y.max(-1))
        e0 = edge_fn(x[..., 1], y[..., 1], x[..., 2], y[..., 2], px, py)
        e1 = edge_fn(x[..., 2], y[..., 2], x[..., 0], y[..., 0], px, py)
        e2 = edge_fn(x[..., 0], y[..., 0], x[..., 1], y[..., 1], px, py)
        pos = (e0 >= 0) & (e1 >= 0) & (e2 >= 0)
        neg = (e0 <= 0) & (e1 <= 0) & (e2 <= 0)
        inside = np.where(area > 0, pos, neg)
        depth = ((e0 * z[..., 0] + e1 * z[..., 1]) + e2 * z[..., 2]) / area
    return inbox & inside & (depth >= -1) & (depth <= 1), depth.astype(F32)


def depth_key(d):
    u = np.asarray(d, F32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint64)


def rasterize(verts, faces, mvp, res):
    """One (mesh, view) job -> (depth fp32 [res, res], face_id int32 [res, res], n_behind)."""
    x, y, z, area, drawn, behind = setup(verts, faces, mvp, res)
    best = np.full((res, res), np.iinfo(np.uint64).max, np.uint64)
    for f in np.nonzero(drawn)[0]:
        c0 = int(max(np.floor(x[f].min()) - 1, 0)); c1 = int(min(np.ceil(x[f].max()), res - 1))
        r0 = int(max(np.floor(y[f].min()) - 1, 0)); r1 = int(min(np.ceil(y[f].max()), res - 1))
        if c0 > c1 or r0 > r1:
            continue
        py, px = np.meshgrid(np.arange(r0, r1 + 1, dtype=F32) + F32(0.5), np.arange(c0, c1 + 1, dtype=F32) + F32(0.5), indexing="ij")
        cov, d = fragment(x[f], y[f], z[f], area[f], px, py)
        key = (depth_key(d) << np.uint64(32)) | np.uint64(f)
        win = best[r0:r1 + 1, c0:c1 + 1]
        np.minimum(win, np.where(cov, key, np.iinfo(np.uint64).max), out=win)
    return resolve(best) + (int(behind.sum()),)


def resolve(best):
    empty = best == np.iinfo(np.uint64).max
    k = (best >> np.uint64(32)).astype(np.uint32)
    u = np.where(k & np.uint32(0x80000000), k & np.uint32(0x7fffffff), ~k).astype(np.uint32)
    depth = np.where(empty, EMPTY_DEPTH, u.view(F32)).astype(F32)
    face = np.where(empty, -1, (best & np.uint64(0xffffffff)).astype(np.int64)).astype(np.int32)
    return depth, face


def rasterize_pixels(verts, faces, mvp, res, rows, cols, chunk=1 << 22):
    """Brute force over every face at the given pixels only -> (depth [n], face_id [n])."""
    x, y, z, area, drawn, _ = setup(verts, faces, mvp, res)
    ids = np.nonzero(drawn)[0]
    py = np.asarray(rows, F32) + F32(0.5)
    px = np.asarray(cols, F32) + F32(0.5)
    best = np.full(py.shape[0], np.iinfo(np.uint64).max, np.uint64)
    step = max(1, chunk // max(1, py.shape[0]))
    for s in range(0, ids.size, step):
        f = ids[s:s + step]
        cov, d = fragment(x[f, None], y[f, None], z[f, None], area[f, None], px[None], py[None])
        key = (depth_key(d) << np.uint64(32)) | f.astype(np.uint64)[:, None]
        best = np.minimum(best, np.where(cov, key, np.iinfo(np.uint64).max).min(0))
    return resolve(best)


def tet_centres(pos, tets):
    p = np.asarray(pos, F32)[np.asarray(tets, np.int64)]  # [T, 4, 3]
    return (((p[:, 0] + p[:, 1]) + p[:, 2]) + p[:, 3]) * F32(0.25)


def centre_pixels(pos, tets, mvp, res):
    """(ndc [T, 3], q [T, 3] rounded half to even, in_view [T]) of the tet centres."""
    h = mvp_rows(mvp, tet_centres(pos, tets))
    with np.errstate(all="ignore"):
        n = h[:, :3] / h[:, 3:4]
        q = np.rint((n * F32(0.5) + F32(0.5)) * F32(res - 1))
    in_view = ((q >= 0) & (q <= res - 1)).all(1)
    return n, q, in_view


def window_min(img, r=WINDOW):
    """Minimum over the (2r+1)^2 window clipped to the image, per pixel."""
    out = img.copy()
    for axis in (0, 1):
        src = out.copy()
        n = src.shape[axis]
        for s in range(1, r + 1):
            a = [slice(None)] * 2
            b = [slice(None)] * 2
            a[axis], b[axis] = slice(0, n - s), slice(s, n)
            out[tuple(a)] = np.minimum(out[tuple(a)], src[tuple(b)])
            out[tuple(b)] = np.minimum(out[tuple(b)], src[tuple(a)])
    return out


def visible_tets(pos, tets, f2t, mvp, depth, face_id):
    """One job -> (visible bool [T], rast bool [T]) as mdb_visible_tets computes them."""
    res = depth.shape[0]
    n, q, in_view = centre_pixels(pos, tets, mvp, res)
    dmin = window_min(np.asarray(depth, F32))
    all_empty = window_min((np.asarray(face_id) < 0).astype(np.int8)) == 1
    vis = np.zeros(in_view.shape[0], bool)
    k = np.nonzero(in_view)[0]
    row, col = q[k, 1].astype(np.int64), q[k, 0].astype(np.int64)
    vis[k] = (dmin[row, col] >= n[k, 2]) | all_empty[row, col]
    rast = np.zeros(in_view.shape[0], bool)
    ids = np.asarray(face_id)[np.asarray(face_id) >= 0]
    rast[np.asarray(f2t, np.int64)[ids]] = True
    return vis, rast
