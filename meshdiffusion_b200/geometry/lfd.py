"""Light field distance (LFD) between meshes, for `--mode=eval_metrics` (`eval.metric_lfd`), on the sm_90a kernels
`mdb_raster_depth` (csrc/raster.cu) and `mdb_lfd_descriptors` / `mdb_lfd_matrix` (csrc/lfd.cu).

The structure is Chen et al., "On Visual Similarity Based 3D Model Retrieval" (Eurographics 2003): 10 light fields per
shape, each 10 orthographic silhouettes seen from one vertex of each antipodal pair of a regular dodecahedron; per
silhouette 35 Zernike magnitudes and 10 Fourier magnitudes quantized to 8 bits; two light fields compared under each of
the dodecahedron's 60 rotations, two shapes over all 10 x 10 light-field pairs. The camera-set rotations, the quantization
scales and the ray-based Fourier signature are this project's own, so the values are not interchangeable with those of
the 3DRetrieval binary (LFD_CONVENTION). Every step is rounded on its own; oracle/lfd_oracle.py restates it in numpy.
"""
import math

import numpy as np
import torch

from .. import _native
from . import singleview
from .pointcloud import _offsets

LFD_CONVENTION = ("Chen et al. 2003 structure (10 light fields x 10 dodecahedron views, 35 Zernike + 10 Fourier "
                  "magnitudes per 256^2 silhouette, 8-bit, L1 per view, min over 10 x 10 light-field pairs and the 60 "
                  "rotations); this project's camera rotations, quantization and ray signature, not the 3DRetrieval "
                  "binary's values")
LFD_RES = 256
N_FIELDS, N_VIEWS, DESC_BYTES = 10, 10, 48
COEFS = 45  # 35 Zernike + 10 Fourier bytes; the last 3 of the 48 are zero
RAYS, FOURIER = 64, 10
MAX_VIEWS_PER_CALL = 1024

PHI = (1 + math.sqrt(5)) / 2
# one vertex of each antipodal pair of the dodecahedron (|v| = sqrt(3))
DODECAHEDRON = np.array([(1, 1, 1), (1, 1, -1), (1, -1, 1), (1, -1, -1), (0, 1 / PHI, PHI), (0, 1 / PHI, -PHI),
                         (1 / PHI, PHI, 0), (1 / PHI, -PHI, 0), (PHI, 0, 1 / PHI), (PHI, 0, -1 / PHI)], np.float64)
# R_0 .. R_9, the rotations of the 10 camera sets: the identity, then greedy farthest points (modulo the dodecahedron's
# rotations) among 4096 random rotations; `python -m oracle.lfd_oracle` regenerates the table
ROTATIONS = np.array([
    ((1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)),
    ((-0.4759600749708959, 0.8153836796584514, -0.32956253121424883), (-0.3049891708033575, -0.504505875917471, -0.8077471305163674), (-0.8248900609938147, -0.283942381675207, 0.4888078468705589)),
    ((-0.8274836540840367, 0.3196523049650829, -0.46162019686560446), (-0.5405372196341373, -0.231009089162179, 0.808983507195701), (0.1519549815370535, 0.9189435263687153, 0.3639402134020143)),
    ((-0.4926298198632888, -0.8129545527787965, -0.3105169169267444), (0.7986694853239358, -0.5640604364741832, 0.2096732629997289), (-0.34560514144593274, -0.14470908444455385, 0.9271549854718767)),
    ((0.03268769534150617, -0.8579893822319835, 0.5126263108253806), (0.9879442609826938, 0.10539065215402776, 0.11339729992335443), (-0.15131970051721397, 0.5027395254162215, 0.8510906636896289)),
    ((-0.5011304138353267, 0.016076346897367977, 0.865222433481512), (0.8591130364341908, -0.11078918347672695, 0.49965042525087955), (0.10388984049491412, 0.9937138963982517, 0.04170843016640302)),
    ((0.8077219888074014, -0.4740478939074063, -0.35051930485918836), (-0.36117115550382606, 0.07205185505959932, -0.9297117438295064), (0.46598346025266524, 0.877546081105957, -0.11301455794069093)),
    ((-0.9029656083841564, -0.1037629865700987, -0.41699682575948294), (0.13913804009882205, -0.9887299558831131, -0.05526011343489046), (-0.40656329872836483, -0.10791810301071778, 0.9072265247277984)),
    ((0.22117677240506095, 0.9752315944778731, -0.002042665079029282), (-0.8948974184834284, 0.20212408881790034, -0.3978749340071941), (-0.3876073344767555, 0.08982866943063733, 0.9174373899117835)),
    ((0.1073008040945509, 0.6258077879041928, 0.7725614215317277), (-0.17251239356450718, 0.7769799608590073, -0.6054268035775919), (-0.9791455517476998, -0.06831363715976713, 0.19133017396818586)),
], np.float64)


def _axis_angle(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * k + (1 - math.cos(angle)) * (k @ k)


def _rotation_group():
    """The 60 rotations of the dodecahedron [60, 3, 3]: closure of the 5-fold rotation about the face axis (0, phi, 1)
    and the 3-fold cyclic permutation of the axes, the identity first."""
    gens = (_axis_angle((0, PHI, 1), 2 * math.pi / 5), np.array([[0, 0, 1], [1, 0, 0], [0, 1, 0]], np.float64))
    group, frontier = [np.eye(3)], [np.eye(3)]
    while frontier:
        new = []
        for a in frontier:
            for g in gens:
                c = g @ a
                if min(np.abs(c - b).max() for b in group) > 1e-9:
                    group.append(c)
                    new.append(c)
        frontier = new
    return np.stack(group)


def _view_permutations(group):
    """int8 [60, 10]: pi_g(i) = j where g v_i = +-v_j."""
    img = np.einsum("gij,vj->gvi", group, DODECAHEDRON)  # [g, v, 3]
    diff = np.minimum(np.abs(img[:, :, None] - DODECAHEDRON[None, None]).max(-1),
                      np.abs(img[:, :, None] + DODECAHEDRON[None, None]).max(-1))  # [g, v, j]
    if not ((diff < 1e-9).sum(-1) == 1).all():
        raise AssertionError("the rotation group does not permute the dodecahedron's views")
    return diff.argmin(-1).astype(np.int8)


GROUP = _rotation_group()
PERMUTATIONS = _view_permutations(GROUP)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _view_frames():
    """fp64 [100, 3, 3]: rows e0, e1, d of view i of light field k at 10 k + i. d = R_k v_i / sqrt(3); h = (0, 1, 0), or
    (1, 0, 0) when |d_y| > 0.9; e0 = normalize(h x d); e1 = d x e0."""
    v = DODECAHEDRON
    d = np.stack([_dot(ROTATIONS[:, None, j, :], v[None]) for j in range(3)], -1) / math.sqrt(3)  # [k, i, 3]
    h = np.where((np.abs(d[..., 1]) > 0.9)[..., None], np.array([1.0, 0.0, 0.0]), np.array([0.0, 1.0, 0.0]))
    e0 = _cross(h, d)
    e0 = e0 / np.sqrt(_dot(e0, e0))[..., None]
    e1 = _cross(d, e0)
    return np.stack([e0, e1, d], -2).reshape(N_FIELDS * N_VIEWS, 3, 3)


FRAMES = _view_frames()


def camera_mvps(centre, scale):
    """centre fp64 [M, 3], scale fp64 [M] -> fp32 [M, 100, 4, 4], the row-major orthographic mvps of every light-field view:
    rows (0.9 s e0, -0.9 s e0.c), (0.9 s e1, -0.9 s e1.c), (0.5 s d, -0.5 s d.c), (0, 0, 0, 1), in fp64, rounded once."""
    c = np.asarray(centre, np.float64).reshape(-1, 1, 1, 3)
    a = np.asarray(scale, np.float64).reshape(-1, 1, 1) * np.array([0.9, 0.9, 0.5])[None, None]  # [M, 1, 3]
    out = np.zeros((c.shape[0], FRAMES.shape[0], 4, 4), np.float64)
    out[:, :, :3, :3] = a[..., None] * FRAMES[None]
    out[:, :, :3, 3] = -(a * _dot(FRAMES[None], c))
    out[:, :, 3, 3] = 1.0
    return out.astype(np.float32)


def normalization(verts, vert_off):
    """Per mesh of the packed fp32 verts: (bounding-box midpoint c fp64 [M, 3], s = 1 / max |v - c| fp64 [M]), with
    |x| = sqrt((x0^2 + x1^2) + x2^2) in fp64; s = 1 for a mesh without extent."""
    vo = _offsets(vert_off, len(vert_off) - 1, "vert_off")
    M = vo.shape[0] - 1
    dev = verts.device
    counts = torch.from_numpy(np.diff(vo)).to(dev)
    idx = torch.repeat_interleave(torch.arange(M, device=dev), counts)
    v = verts.double()
    lo = torch.full((M, 3), math.inf, device=dev, dtype=torch.float64).scatter_reduce(0, idx[:, None].expand(-1, 3), v, "amin")
    hi = torch.full((M, 3), -math.inf, device=dev, dtype=torch.float64).scatter_reduce(0, idx[:, None].expand(-1, 3), v, "amax")
    c = torch.where((counts > 0)[:, None], (lo + hi) * 0.5, torch.zeros_like(lo))
    d = v - c[idx]
    r = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    rmax = torch.zeros(M, device=dev, dtype=torch.float64).scatter_reduce(0, idx, r, "amax").cpu().numpy()
    scale = np.ones(M)
    np.divide(1.0, rmax, out=scale, where=rmax > 0)
    return c.cpu().numpy(), scale


_TABLES = {}


def fourier_tables(device):
    """(ray directions (cos, sin) fp32 [64, 2], DFT table (cos, sin) of 2 pi m k / 64 fp64 [11, 64, 2]) on the device,
    both computed in fp64 on the host."""
    key = str(device)
    if key not in _TABLES:
        k = np.arange(RAYS)
        th = 2 * np.pi * k / RAYS
        ray = np.stack([np.cos(th), np.sin(th)], -1).astype(np.float32)
        a = 2 * np.pi * ((np.arange(FOURIER + 1)[:, None] * k[None]) % RAYS) / RAYS
        dft = np.stack([np.cos(a), np.sin(a)], -1)
        _TABLES[key] = (torch.from_numpy(ray).to(device), torch.from_numpy(dft).to(device),
                        torch.from_numpy(PERMUTATIONS.copy()).to(device))
    return _TABLES[key]


def silhouette_descriptors(face_id):
    """face_id int32 [n, res, res] (CUDA; res <= 256) -> (descriptors uint8 [n, 48], inside-pixel counts int32 [n]) of the
    silhouettes face_id >= 0. An empty silhouette gives zeros."""
    face_id = face_id.to(torch.int32).contiguous()
    if face_id.dim() != 3 or face_id.shape[1] != face_id.shape[2] or not face_id.is_cuda:
        raise ValueError("face_id must be a CUDA tensor [n, res, res]")
    n, res = face_id.shape[0], face_id.shape[1]
    ray, dft, _ = fourier_tables(face_id.device)
    desc = torch.empty(n, DESC_BYTES, device=face_id.device, dtype=torch.uint8)
    n_inside = torch.empty(n, device=face_id.device, dtype=torch.int32)
    _native.check(_native.lib().mdb_lfd_descriptors(_native.ptr(face_id), n, res, _native.ptr(ray), _native.ptr(dft),
                                                    _native.ptr(desc), _native.ptr(n_inside), _native.current_stream()))
    return desc, n_inside


def lfd_descriptors(verts, faces, vert_off, face_off, res=LFD_RES):
    """Light-field descriptors of B meshes packed like `MarchingTets._extract_raw`'s output (verts fp32 [V, 3], faces int64
    [F, 3] local to their mesh, B + 1 offsets each) -> (uint8 [B, 10, 10, 48] on the device, empty views int64 [B]).

    Each mesh is centred on its bounding box and scaled to unit radius (`normalization`), rasterized from the 100 views of
    `camera_mvps` at res x res, at most MAX_VIEWS_PER_CALL views per rasterizer call, and every silhouette is described
    by `silhouette_descriptors`."""
    verts = verts.float().contiguous()
    faces = faces.long().contiguous()
    if not verts.is_cuda:
        raise ValueError("light field descriptors run on the CUDA device only")
    vo = _offsets(vert_off, len(vert_off) - 1, "vert_off")
    B = vo.shape[0] - 1
    fo = _offsets(face_off, B, "face_off")
    if vo[-1] != verts.shape[0] or fo[-1] != faces.shape[0]:
        raise ValueError("offsets do not cover verts / faces")
    dev = verts.device
    V = N_FIELDS * N_VIEWS
    desc = torch.empty(B * V, DESC_BYTES, device=dev, dtype=torch.uint8)
    n_inside = torch.empty(B * V, device=dev, dtype=torch.int32)
    if B == 0:
        return desc.view(0, N_FIELDS, N_VIEWS, DESC_BYTES), np.zeros(0, np.int64)
    centre, scale = normalization(verts, vo)
    mvp = torch.from_numpy(camera_mvps(centre, scale).reshape(B * V, 16)).to(dev)
    job_mesh = torch.arange(B, dtype=torch.int32, device=dev).repeat_interleave(V)
    vo_d = torch.from_numpy(vo[:-1].copy()).to(dev)
    fo_d = torch.from_numpy(fo).to(dev)
    step = max(1, min(MAX_VIEWS_PER_CALL, singleview._MAX_JOB_PIXELS // (res * res)))
    for j0 in range(0, B * V, step):
        _, face_id = singleview._raster_packed(verts, faces, vo_d, fo_d, job_mesh[j0:j0 + step].contiguous(),
                                               mvp[j0:j0 + step].contiguous(), res)
        desc[j0:j0 + step], n_inside[j0:j0 + step] = silhouette_descriptors(face_id)
    empty = (n_inside == 0).view(B, V).sum(1).cpu().numpy().astype(np.int64)
    return desc.view(B, N_FIELDS, N_VIEWS, DESC_BYTES), empty


def lfd_matrix(A, B=None):
    """A uint8 [nA, 10, 10, 48], B uint8 [nB, 10, 10, 48] (CUDA) -> LFD(A_i, B_j) int32 [nA, nB] on the device: min over
    light fields s of A, t of B and the 60 rotations g of sum_i L1(A[s][i], B[t][pi_g(i)]). Exact integers, symmetric,
    batch-invariant. B None: the self matrix of A (diagonal 0)."""
    shape = (N_FIELDS, N_VIEWS, DESC_BYTES)
    A = A.to(torch.uint8).contiguous()
    if A.dim() != 4 or tuple(A.shape[1:]) != shape or not A.is_cuda:
        raise ValueError("A must be a CUDA uint8 tensor [nA, 10, 10, 48]")
    if B is not None:
        B = B.to(torch.uint8).contiguous()
        if B.dim() != 4 or tuple(B.shape[1:]) != shape or B.device != A.device:
            raise ValueError("B must be a uint8 tensor [nB, 10, 10, 48] on the device of A")
    nB = A.shape[0] if B is None else B.shape[0]
    out = torch.empty(A.shape[0], nB, device=A.device, dtype=torch.int32)
    _, _, perms = fourier_tables(A.device)
    _native.check(_native.lib().mdb_lfd_matrix(_native.ptr(A), A.shape[0], _native.ptr(B), nB, _native.ptr(perms),
                                               _native.ptr(out), _native.current_stream()))
    return out
