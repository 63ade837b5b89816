"""Point clouds of generated shapes and the Chamfer and Earth Mover's distances between them, on the sm_90a kernels
(`mdb_mesh_sample_points`, `mdb_chamfer_matrix`, `mdb_emd_matrix`). No reference counterpart: the reference's fitting code
calls kaolin's `sample_points` / `chamfer_distance` (nvdiffrec/lib/geometry/dmtet.py:455-457) and ships no evaluation code.

Chamfer convention: CD(X, Y) = mean_x min_y |x - y|^2 + mean_y min_x |x - y|^2 (squared distances, sum of the two means),
as kaolin's `chamfer_distance` and the PointFlow evaluation code compute it.
EMD convention: EMD(X, Y) = min over bijections pi of (1/N) sum_i |x_i - y_pi(i)| (Euclidean distances), the quantity
PointFlow's `emd_approx` approximates; here it is solved to within a stated eps and certified by a dual bound.
"""
import numpy as np
import torch

from .. import _native
from . import dmtet

CD_CONVENTION = "mean_x min_y |x-y|^2 + mean_y min_x |x-y|^2 (squared Euclidean, sum of the two means)"
EMD_CONVENTION = "min over bijections pi of mean_x |x-pi(x)| (Euclidean, not squared; clouds of equal size)"


def _offsets(off, n, name):
    o = np.asarray(off.cpu() if torch.is_tensor(off) else off, dtype=np.int64).reshape(-1)
    if o.shape[0] != n + 1 or o[0] != 0 or np.any(np.diff(o) < 0):
        raise ValueError(f"{name} must be {n + 1} non-decreasing offsets starting at 0")
    return o


def sample_surface_points(verts, faces, vert_off, face_off, n_points, seed, first_id=0, uniforms=None):
    """Area-weighted surface points of B meshes packed like `MarchingTets._extract_raw`'s output.

    verts fp32 [V,3] and faces int64 [F,3] (indices local to their mesh) on the CUDA device; vert_off / face_off: B + 1
    offsets (host sequence or tensor), mesh b owning verts[vert_off[b]:vert_off[b+1]] and faces[face_off[b]:face_off[b+1]].
    uniforms: optional fp32 [B, n_points, 3] in [0, 1); None draws them from Philox(seed) keyed by mesh id first_id + b and
    point index, so a mesh's points do not depend on the batch it is sampled in.
    Returns (points fp32 [B, n_points, 3], empty bool [B]); rows of empty meshes (no faces or zero area) stay NaN."""
    L = _native.lib()
    verts = verts.float().contiguous()
    faces = faces.long().contiguous()
    if not verts.is_cuda:
        raise _native.NativeError("surface sampling runs on the CUDA device only")
    vo = _offsets(vert_off, len(vert_off) - 1, "vert_off")
    B = vo.shape[0] - 1
    fo = _offsets(face_off, B, "face_off")
    if vo[-1] != verts.shape[0] or fo[-1] != faces.shape[0]:
        raise ValueError("offsets do not cover verts / faces")
    if n_points < 1:
        raise ValueError("n_points must be at least 1")
    dev = verts.device
    if faces.shape[0]:
        nv = torch.from_numpy(np.repeat(np.diff(vo), np.diff(fo))).to(dev)
        if bool(((faces < 0) | (faces >= nv[:, None])).any()):
            raise ValueError("face index out of range for its mesh")
    if uniforms is not None:
        uniforms = uniforms.float().contiguous()
        if tuple(uniforms.shape) != (B, n_points, 3) or uniforms.device != dev:
            raise ValueError(f"uniforms must be [{B}, {n_points}, 3] on {dev}")
    points = torch.full((B, n_points, 3), float("nan"), device=dev, dtype=torch.float32)
    written = torch.empty(B, device=dev, dtype=torch.int32)
    cdf = torch.empty(max(faces.shape[0], 1), device=dev, dtype=torch.float64)
    vo_d = torch.from_numpy(vo[:-1].copy()).to(dev)
    fo_d = torch.from_numpy(fo).to(dev)
    _native.check(L.mdb_mesh_sample_points(_native.ptr(verts), _native.ptr(faces), _native.ptr(vo_d), _native.ptr(fo_d), B,
                                           int(n_points), _native.ptr(uniforms), int(seed) & (2 ** 64 - 1), int(first_id),
                                           _native.ptr(cdf), _native.ptr(points), _native.ptr(written),
                                           _native.current_stream()))
    return points, written == 0


def chamfer_matrix(A, B=None):
    """A fp32 [nA, N, 3], B fp32 [nB, M, 3] (CUDA) -> CD(A_i, B_j) float64 [nA, nB]. B None: the self matrix of A
    (symmetric, diagonal exactly 0). Bitwise reproducible; entry (i, j) does not depend on the other clouds."""
    L = _native.lib()
    A = A.float().contiguous()
    if A.dim() != 3 or A.shape[2] != 3 or not A.is_cuda:
        raise ValueError("A must be a CUDA tensor [nA, N, 3]")
    if B is not None:
        B = B.float().contiguous()
        if B.dim() != 3 or B.shape[2] != 3 or B.device != A.device:
            raise ValueError("B must be a tensor [nB, M, 3] on the device of A")
    nB, M = (A.shape[0], A.shape[1]) if B is None else (B.shape[0], B.shape[1])
    out = torch.empty(A.shape[0], nB, device=A.device, dtype=torch.float64)
    _native.check(L.mdb_chamfer_matrix(_native.ptr(A), A.shape[0], A.shape[1], _native.ptr(B), nB, M, _native.ptr(out),
                                       _native.current_stream()))
    return out


def chamfer_pairs(clouds, pairs):
    """clouds fp32 [n, N, 3] (CUDA), pairs: P index pairs (a, b) with a != b -> (cd float64 [P], mean_ab float64 [P],
    max_ab float32 [P]) from one `mdb_chamfer_pairs` launch. cd[p] = CD(clouds[a], clouds[b]), bitwise the
    `chamfer_matrix` entry of the same two clouds; mean_ab[p] and max_ab[p] are the mean and the max over x in a of
    min over y in b of |x - y|^2 (sqrt(max_ab) is the one-sided Hausdorff distance a -> b). An entry does not depend on
    the other pairs. The list is checked on the host: a == b or an index out of range raises ValueError."""
    L = _native.lib()
    clouds = clouds.float().contiguous()
    if clouds.dim() != 3 or clouds.shape[2] != 3 or not clouds.is_cuda:
        raise ValueError("clouds must be a CUDA tensor [n, N, 3]")
    n, N = clouds.shape[0], clouds.shape[1]
    p = np.asarray(pairs.cpu() if torch.is_tensor(pairs) else pairs, dtype=np.int64).reshape(-1, 2)
    if p.size and (p.min() < 0 or p.max() >= n):
        raise ValueError(f"chamfer_pairs: a cloud index is outside [0, {n})")
    if np.any(p[:, 0] == p[:, 1]):
        raise ValueError("chamfer_pairs: a pair (a, a) compares a cloud with itself")
    P = p.shape[0]
    cd = torch.empty(P, device=clouds.device, dtype=torch.float64)
    mean_ab = torch.empty_like(cd)
    max_ab = torch.empty(P, device=clouds.device, dtype=torch.float32)
    if P == 0:
        return cd, mean_ab, max_ab
    pd = torch.from_numpy(p.astype(np.int32)).to(clouds.device)
    _native.check(L.mdb_chamfer_pairs(_native.ptr(clouds), n, N, _native.ptr(pd), P, _native.ptr(cd), _native.ptr(mean_ab),
                                      _native.ptr(max_ab), _native.current_stream()))
    return cd, mean_ab, max_ab


# the auction's fp32 limit (csrc/emd.cu kFloor): eps must be at least this share of the pair's bounding-box diagonal
EMD_EPS_FLOOR = 2.0 ** -18


def emd_matrix(A, B=None, eps=1e-5):
    """A fp32 [nA, N, 3], B fp32 [nB, N, 3] (CUDA) -> (EMD(A_i, B_j), certified gap), both float64 [nA, nB].

    EMD is EMD_CONVENTION, solved by an auction to within eps of the optimum: every entry is the mean cost of a true
    bijection, and gap = entry - a dual lower bound, so 0 <= entry - optimum <= gap <= eps (over the fp32 point distances).
    B None: the self matrix of A (symmetric, diagonal exactly 0). Bitwise reproducible; entry (i, j) does not depend on
    the other clouds. Clouds of different sizes, non-finite coordinates and an eps below what fp32 prices resolve at the
    clouds' scale (EMD_EPS_FLOOR x the bounding-box diagonal of a pair) raise ValueError."""
    L = _native.lib()
    A = A.float().contiguous()
    if A.dim() != 3 or A.shape[2] != 3 or not A.is_cuda:
        raise ValueError("A must be a CUDA tensor [nA, N, 3]")
    if B is not None:
        B = B.float().contiguous()
        if B.dim() != 3 or B.shape[2] != 3 or B.device != A.device:
            raise ValueError("B must be a tensor [nB, N, 3] on the device of A")
        if B.shape[1] != A.shape[1]:
            raise ValueError(f"EMD needs clouds of equal size, got N = {A.shape[1]} and M = {B.shape[1]}")
    if A.shape[1] < 1:
        raise ValueError("clouds need at least one point")
    eps = float(eps)
    if not (eps > 0 and np.isfinite(eps)):
        raise ValueError("eps must be positive and finite")
    nB = A.shape[0] if B is None else B.shape[0]
    out = torch.zeros(A.shape[0], nB, device=A.device, dtype=torch.float64)
    gap = torch.zeros_like(out)
    if A.shape[0] == 0 or nB == 0:
        return out, gap
    Bs = A if B is None else B
    if not (bool(torch.isfinite(A).all()) and bool(torch.isfinite(Bs).all())):
        raise ValueError("point coordinates must be finite")
    # the largest pair diagonal: the auction cannot resolve an eps below the floor at that scale
    lo_a, hi_a, lo_b, hi_b = A.amin(1), A.amax(1), Bs.amin(1), Bs.amax(1)
    ext = torch.maximum(hi_a[:, None], hi_b[None]) - torch.minimum(lo_a[:, None], lo_b[None])
    cmax = float(ext.square().sum(-1).sqrt().max())
    if np.float32(eps) < np.float32(cmax) * np.float32(EMD_EPS_FLOOR):
        raise ValueError(f"eps = {eps:.3g} is below what fp32 prices resolve at these clouds' scale: the floor is "
                         f"{EMD_EPS_FLOOR:.3g} x the bounding-box diagonal {cmax:.3g} = {cmax * EMD_EPS_FLOOR:.3g}")
    _native.check(L.mdb_emd_matrix(_native.ptr(A), A.shape[0], _native.ptr(B), nB, A.shape[1], np.float32(eps).item(),
                                   _native.ptr(out), _native.ptr(gap), _native.current_stream()))
    bad = torch.isnan(out)
    if bool(bad.any()):
        capped = int((bad & torch.isinf(gap)).sum())
        raise _native.NativeError(f"emd_matrix: {int(bad.sum())} entries did not converge ({capped} hit the auction's round "
                                  f"limit; the others have an eps below the fp32 floor of their pair)")
    return out, gap


_TETS = {}


def _tet_grid(resolution, device):
    key = (int(resolution), str(device))
    if key not in _TETS:
        verts, idx = dmtet.load_tet_grid(resolution)
        v = torch.tensor(verts, device=device)
        coords = dmtet.grid_coords_of_tet_vertices(v.cpu()).to(device)
        _TETS[key] = (v, coords, idx, {})
    return _TETS[key]


def grids_to_meshes(grids, resolution, mesh_scale=1.1, deform_scale=3.0):
    """grids [B,4,R,R,R] (CUDA) -> (verts fp32 [V,3], faces int64 [F,3], vert_off, face_off host int64 [B + 1]): tet-vertex
    gather and marching tets, meshes packed in batch order. The scale defaults are tools/npy_to_obj.py's (nvdiffrec
    configs/res64.json), so every set meshed through here shares one frame."""
    v, coords, idx, engines = _tet_grid(resolution, grids.device)
    B = grids.shape[0]
    if B not in engines:
        engines[B] = dmtet.MarchingTets(idx, v.shape[0], max_batch=B)
    sdf, pos = dmtet.grid_to_tet_inputs(grids.float(), coords, v, resolution, mesh_scale, deform_scale)
    mverts, mfaces, _, _, _, off = engines[B]._extract_raw(pos, sdf)
    return mverts, mfaces, off[:, 0], off[:, 1]


def grids_to_point_clouds(grids, resolution, n_points, seed, first_id=0, mesh_scale=1.1, deform_scale=3.0):
    """grids [B,4,R,R,R] (CUDA) -> (points fp32 [B, n_points, 3], empty bool [B]): `grids_to_meshes` and surface sampling,
    mesh b keyed by id first_id + b."""
    mverts, mfaces, vert_off, face_off = grids_to_meshes(grids, resolution, mesh_scale, deform_scale)
    return sample_surface_points(mverts, mfaces, vert_off, face_off, n_points, seed, first_id=first_id)
