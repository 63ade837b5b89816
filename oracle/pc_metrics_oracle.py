"""ORACLE (test infrastructure only): numpy restatement of surface sampling, the Chamfer distance and the MMD / COV / 1-NNA
generation metrics of geometry/pointcloud.py and diffusion/gen_metrics.py.

No third-party implementation (kaolin, pytorch3d, PointFlow) is available to pin these against, so they rest on their
definitions: the brute-force Chamfer distance is checked against the k-d tree one, and the metrics against cases whose
answers are known by construction (tests/test_pc_metrics_cpu.py).
"""
import numpy as np
from scipy.spatial import cKDTree


def face_areas(verts, faces):
    """0.5 |(b - a) x (c - a)| in fp64 from fp32 corners, with the kernel's operation order."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    return 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)


def sample_points(verts, faces, uniforms):
    """One mesh, uniforms [N, 3] = (u, r1, r2) -> (points fp64 [N, 3], face index [N]); None if the mesh is empty."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if f.shape[0] == 0:
        return None
    cdf = np.cumsum(face_areas(verts, f))
    total = cdf[-1]
    if not total > 0:
        return None
    u = np.asarray(uniforms, np.float32).astype(np.float64)
    face = np.searchsorted(cdf, u[:, 0] * total, side="right")  # smallest k with cdf[k] > u * total
    v = np.asarray(verts, np.float32).astype(np.float64)
    s = np.sqrt(u[:, 1:2])
    r2 = u[:, 2:3]
    p = (1 - s) * v[f[face, 0]] + s * (1 - r2) * v[f[face, 1]] + s * r2 * v[f[face, 2]]
    return p, face


def chamfer_brute(x, y):
    """CD(X, Y) = mean_x min_y |x-y|^2 + mean_y min_x |x-y|^2 in fp64, all pairs."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    d = ((x[:, None, :] - y[None, :, :]) ** 2).sum(-1)
    return float(d.min(axis=1).mean() + d.min(axis=0).mean())


def chamfer_kdtree(x, y):
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    dxy, _ = cKDTree(y).query(x)
    dyx, _ = cKDTree(x).query(y)
    return float((dxy ** 2).mean() + (dyx ** 2).mean())


def chamfer(x, y):
    return chamfer_brute(x, y) if len(x) * len(y) <= 1 << 22 else chamfer_kdtree(x, y)


def chamfer_matrix(A, B=None):
    B = A if B is None else B
    return np.array([[chamfer(a, b) for b in B] for a in A], np.float64)


def metrics(d_gr, d_gg, d_rr):
    """MMD / COV / 1-NNA from the three CD matrices, written out loop by loop with the lowest-index tie rule."""
    d_gr, d_gg, d_rr = (np.asarray(d, np.float64) for d in (d_gr, d_gg, d_rr))
    ng, nr = d_gr.shape

    def first_argmin(row):
        best = 0
        for k in range(1, len(row)):
            if row[k] < row[best]:
                best = k
        return best

    mmd = sum(min(d_gr[g, r] for g in range(ng)) for r in range(nr)) / nr
    cov = len({first_argmin(d_gr[g]) for g in range(ng)}) / nr

    def dist(p, q):  # concatenated order [G..., R...]
        if p < ng and q < ng:
            return d_gg[p, q]
        if p >= ng and q >= ng:
            return d_rr[p - ng, q - ng]
        return d_gr[p, q - ng] if p < ng else d_gr[q, p - ng]

    n = ng + nr
    same = []
    for p in range(n):
        row = [np.inf if q == p else dist(p, q) for q in range(n)]
        same.append((first_argmin(row) < ng) == (p < ng))
    same = np.array(same)
    return {"mmd_cd": mmd, "cov_cd": cov, "1nna_cd": float(same.mean()),
            "1nna_cd_gen": float(same[:ng].mean()), "1nna_cd_ref": float(same[ng:].mean())}
