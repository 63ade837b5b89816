"""Numpy restatement of the light field distance (meshdiffusion_b200/geometry/lfd.py, csrc/lfd.cu), and the generator of
the camera-set rotation table.

* `icosahedral_group` -- the 60 rotations of the dodecahedron, by closure of two generators in fp64;
* `generate_rotations` -- the table R_0 .. R_9 (`python -m oracle.lfd_oracle` prints it as geometry/lfd.py holds it);
* `mvps` -- the 100 orthographic cameras of a mesh, fp64 rounded to fp32 once;
* `descriptor` / `mesh_descriptors` -- one silhouette's 48 bytes, float32 / fp64 operation by operation in the kernel's order, with the same
  thread assignment (pixel p to lane p mod 256, in pixel order) and the same reduction tree;
* `lfd` / `lfd_matrix` -- the integer distance.
Pure numpy: also runs without a GPU.
"""
import math

import numpy as np

from . import raster_oracle as ro

F32 = np.float32
PHI = (1 + math.sqrt(5)) / 2
VERTS = np.array([(1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1), (0, 1 / PHI, PHI), (0, 1 / PHI, -PHI),
                  (1 / PHI, PHI, 0), (1 / PHI, -PHI, 0), (PHI, 0, 1 / PHI), (PHI, 0, -1 / PHI)], np.float64)
LANES = 256
RAYS = 64
FOURIER = 10
ZERNIKE = [(n, m) for n in range(1, 11) for m in range(n % 2, n + 1, 2)]


# ---- cameras --------------------------------------------------------------------------------------------------------

def _axis_angle(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * k + (1 - math.cos(angle)) * (k @ k)


def icosahedral_group():
    """[60, 3, 3] fp64: closure of a 5-fold rotation about the face axis (0, phi, 1) and the 3-fold cyclic permutation of
    the axes; the identity first."""
    gens = [_axis_angle((0, PHI, 1), 2 * math.pi / 5), np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], np.float64)]
    group = [np.eye(3)]
    frontier = [np.eye(3)]
    while frontier:
        nxt = []
        for a in frontier:
            for g in gens:
                c = g @ a
                if not any(np.abs(c - b).max() < 1e-9 for b in group):
                    group.append(c)
                    nxt.append(c)
        frontier = nxt
    return np.stack(group)


def permutations(group):
    """int8 [60, 10]: pi_g(i) = j where g v_i = +-v_j."""
    out = np.zeros((len(group), 10), np.int8)
    for k, g in enumerate(group):
        img = VERTS @ g.T
        for i in range(10):
            hit = [j for j in range(10) if min(np.abs(img[i] - VERTS[j]).max(), np.abs(img[i] + VERTS[j]).max()) < 1e-9]
            assert len(hit) == 1
            out[k, i] = hit[0]
    return out


def _quat_matrix(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rotation_distance(a, cands, group):
    """Least rotation angle of a^-1 c g over the group, for every candidate c [n, 3, 3] -> [n]."""
    rel = np.einsum("ji,njk,gkl->ngil", a, cands, group)
    tr = np.trace(rel, axis1=2, axis2=3)
    return np.arccos(np.clip((tr - 1) / 2, -1, 1)).min(axis=1)


def generate_rotations(n=10, n_candidates=4096, seed=2003):
    """R_0 = identity, then greedy farthest points among random rotations (unit quaternions of normal draws from
    default_rng(seed)), distance as `rotation_distance`, ties to the lower candidate index -> [n, 3, 3] fp64."""
    q = np.random.default_rng(seed).standard_normal((n_candidates, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    cands = np.stack([_quat_matrix(x) for x in q])
    group = icosahedral_group()
    out = [np.eye(3)]
    dmin = rotation_distance(out[0], cands, group)
    for _ in range(n - 1):
        k = int(np.argmax(dmin))
        out.append(cands[k])
        dmin = np.minimum(dmin, rotation_distance(cands[k], cands, group))
    return np.stack(out)


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def centre_scale(verts):
    """Bounding-box midpoint c and 1 / max |v - c| of fp32 vertices, in fp64."""
    v = np.asarray(verts, F32).astype(np.float64)
    c = (v.min(0) + v.max(0)) * 0.5
    d = v - c
    r = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]).max()
    return c, (1.0 / r if r > 0 else 1.0)


def mvps(rotations, c, s):
    """[100, 4, 4] fp32: light field k major, view i minor; view direction d = R_k v_i / sqrt(3)."""
    out = np.zeros((10, 10, 4, 4), np.float64)
    for k in range(10):
        R = rotations[k]
        for i in range(10):
            v = VERTS[i]
            d = np.array([_dot(R[j], v) for j in range(3)]) / math.sqrt(3)
            h = np.array([1.0, 0.0, 0.0]) if abs(d[1]) > 0.9 else np.array([0.0, 1.0, 0.0])
            e0 = _cross(h, d)
            e0 = e0 / math.sqrt(_dot(e0, e0))
            e1 = _cross(d, e0)
            for row, (a, e) in enumerate(((0.9 * s, e0), (0.9 * s, e1), (0.5 * s, d))):
                out[k, i, row, :3] = a * e
                out[k, i, row, 3] = -(a * _dot(e, c))
            out[k, i, 3, 3] = 1.0
    return out.reshape(100, 4, 4).astype(F32)


def fourier_tables():
    """(ray (cos, sin) fp32 [64, 2], DFT (cos, sin) fp64 [11, 64, 2])."""
    k = np.arange(RAYS)
    th = 2 * np.pi * k / RAYS
    ray = np.stack([np.cos(th), np.sin(th)], -1).astype(F32)
    a = 2 * np.pi * ((np.arange(FOURIER + 1)[:, None] * k[None]) % RAYS) / RAYS
    return ray, np.stack([np.cos(a), np.sin(a)], -1)


# ---- descriptor -----------------------------------------------------------------------------------------------------

def _radial(n, m):
    """Coefficients c_j of s^j in P_nm(s) = R_n^m(rho) / rho^m."""
    d = (n - m) // 2
    c = [0] * (d + 1)
    for k in range(d + 1):
        c[d - k] = (-1) ** k * math.factorial(n - k) // (math.factorial(k) * math.factorial((n + m) // 2 - k)
                                                          * math.factorial((n - m) // 2 - k))
    return c


def descriptor(mask):
    """bool [res, res] silhouette -> (uint8 [48], number of inside pixels)."""
    mask = np.asarray(mask, bool)
    res = mask.shape[0]
    P = res * res
    flat = mask.reshape(-1)
    n = int(flat.sum())
    if n == 0:
        return np.zeros(48, np.uint8), 0
    p = np.nonzero(flat)[0]
    r_, c_ = p // res, p % res
    sx, sy = int((2 * c_ + 1).sum()), int((2 * r_ + 1).sum())
    cx, cy = F32(np.float64(sx) / np.float64(2 * n)), F32(np.float64(sy) / np.float64(2 * n))
    # per-pixel values on a [passes, lanes] layout: pixel p is lane p % 256 of pass p // 256
    passes = -(-P // LANES)
    allp = np.arange(passes * LANES)
    ins = np.zeros(passes * LANES, bool)
    ins[:P] = flat
    dx = ((allp % res).astype(F32) + F32(0.5)) - cx
    dy = ((allp // res).astype(F32) + F32(0.5)) - cy
    rho2 = dx * dx + dy * dy
    rad = F32(np.sqrt(rho2[ins].max(), dtype=F32)) + F32(0.5)
    u, w = dx / rad, dy / rad
    s = u * u + w * w
    zr, zi = [np.ones_like(u)], [np.zeros_like(u)]
    for _ in range(10):
        zr.append(zr[-1] * u - zi[-1] * (-w))
        zi.append(zr[-2] * (-w) + zi[-1] * u)
    vals = []
    for n_, m in ZERNIKE:
        c = _radial(n_, m)
        poly = np.full_like(s, F32(c[-1]))
        for cj in c[-2::-1]:
            poly = poly * s + F32(cj)
        vals += [poly * zr[m], poly * zi[m]]
    v = np.stack(vals).astype(np.float64)  # [70, passes * lanes]
    v[:, ~ins] = 0.0  # an outside pixel adds nothing (x + 0 == x for every accumulator value reached)
    v = v.reshape(70, passes, LANES)
    acc = np.zeros((70, LANES))
    for i in range(passes):
        acc = acc + v[:, i]
    st = LANES // 2
    while st:
        acc[:, :st] = acc[:, :st] + acc[:, st:2 * st]
        st //= 2
    tot = acc[:, 0]
    out = np.zeros(48, np.uint8)
    for k, (n_, _) in enumerate(ZERNIKE):
        re, im = tot[2 * k], tot[2 * k + 1]
        a = ((n_ + 1) * np.sqrt(re * re + im * im)) / ((np.pi * np.float64(rad)) * np.float64(rad))
        out[k] = min(255.0, np.floor(a * 256.0 + 0.5))
    # radial signature
    ray, dft = fourier_tables()
    j = np.arange(4 * res + 8)
    h = F32(0.5) * j.astype(F32)
    rk = np.zeros(RAYS)
    for k in range(RAYS):
        x = cx + h * ray[k, 0]
        y = cy + h * ray[k, 1]
        inb = (x >= 0) & (x < res) & (y >= 0) & (y < res)
        stop = int(np.argmin(inb)) if not inb.all() else inb.size
        assert not inb[stop:].any()
        xi, yi = np.floor(x[:stop]).astype(np.int64), np.floor(y[:stop]).astype(np.int64)
        hit = np.nonzero(mask[yi, xi])[0]
        last = int(j[hit].max()) if hit.size else -1
        rk[k] = 0.5 * last if last > 0 else 0.0
    re = np.zeros(FOURIER + 1)
    im = np.zeros(FOURIER + 1)
    for k in range(RAYS):
        re = re + rk[k] * dft[:, k, 0]
        im = im - rk[k] * dft[:, k, 1]
    mag = np.sqrt(re * re + im * im)
    if mag[0] > 0:
        out[35:45] = np.minimum(255.0, np.floor((mag[1:] / mag[0]) * 512.0 + 0.5))
    return out, n


def mesh_descriptors(verts, faces, rotations, res=256):
    """One mesh -> (uint8 [10, 10, 48], empty views): rasterized by the float32 rasterizer restatement from `mvps`."""
    c, s = centre_scale(verts)
    out, empty = np.zeros((100, 48), np.uint8), 0
    for j, m in enumerate(mvps(rotations, c, s)):
        _, face_id, _ = ro.rasterize(verts, faces, m, res)
        out[j], n = descriptor(face_id >= 0)
        empty += n == 0
    return out.reshape(10, 10, 48), empty


# ---- distance -------------------------------------------------------------------------------------------------------

def lfd(a, b, perms):
    """a, b uint8 [10, 10, 48] -> min over s, t, g of sum_i d(a[s][i], b[t][pi_g(i)]) (int)."""
    a = np.asarray(a, np.int64).reshape(10, 10, 48)
    b = np.asarray(b, np.int64).reshape(10, 10, 48)
    d = np.abs(a[:, :, None, None, :] - b[None, None]).sum(-1)  # [s, i, t, j]
    perms = np.asarray(perms, np.int64)
    i = np.arange(10)
    sums = d[:, i[None, :], :, perms].sum(1)  # [g, s, t]... fancy indexing puts the broadcast axes first
    return int(sums.min())


def lfd_matrix(A, B=None, perms=None):
    """int64 [nA, nB] of `lfd`; B None: the self matrix."""
    B = A if B is None else B
    return np.array([[lfd(x, y, perms) for y in B] for x in A], np.int64).reshape(len(A), len(B))


if __name__ == "__main__":
    np.set_printoptions(precision=17, floatmode="unique")
    for R in generate_rotations():
        print("    (" + ", ".join("(" + ", ".join(repr(float(x)) for x in row) + ")" for row in R) + "),")
