"""DMTet training grids fitted to triangle meshes, geometry only (`--mode=fit_grids`).

The reference makes its training grids with nvdiffrec/fit_dmtets.py: a rendering fit (materials, lights, 2 x 5000 render
iterations per shape). Here the grid comes from the mesh's geometry alone, on the library's kernels (csrc/fit.cu):

* `carve_signs` -- the sign: the mesh is rasterized from `camera_mvps` (`mdb_raster_depth`) and a tet vertex is outside
  when one view sees it (`mdb_carve_vertices`). Carving needs no consistent orientation or closed surface (the rasterizer
  draws both windings) and fills cavities no view reaches, as a render-based fit does.
* `closest_points` / `nearest_vertex` -- brute-force point-to-mesh and point-to-point searches (`mdb_closest_points`,
  `mdb_nearest_vertex`); `segment_sum` is the deterministic gather behind the second one's gradient (`mdb_segment_sum`).
* `GridFitter` -- the sign, then `iters` Adam steps on the deformation through the differentiable marching tets with the
  topology the sign fixes. Loss per mesh: mean over marching-tet vertices m of |m - cp(m)|^2 (cp: closest point on the
  source, held fixed within a step), plus mean over source samples s of |s - nn(s)|^2 (nn: nearest marching-tet vertex),
  plus reg * mean |deform|^2. The deformation is clamped to [-0.99, 0.99] after every step (the reference's
  `clamp_deform`) and zeroed off the vertices of the surface tets (fit_dmtets.py:784-789).

Every step is deterministic (no float atomics), so fitting the same meshes twice gives the same grids bit for bit, and a
mesh's grid does not depend on the other meshes of its batch.
"""
import time

import numpy as np
import torch

from .. import _native
from . import dmtet
from .formats import tets_to_3dgrid
from .pointcloud import chamfer_matrix, sample_surface_points
from .singleview import _MAX_JOB_PIXELS, _pack, _raster_packed

# the cameras: a Fibonacci sphere of CAMERA_DISTANCE around the grid, a square image of half-angle atan(TAN_HALF_FOV).
# At distance 3 a sphere of radius r < 0.96 (the grid's corners at mesh_scale 1.1 are at 0.923) subtends a half-angle
# tangent of r / sqrt(9 - r^2) < 0.34, so every grid vertex is in every view, at w in [2, 4]
CAMERA_DISTANCE = 3.0
TAN_HALF_FOV = 0.36
NEAR, FAR = 1.0, 10.0

# defaults of the `config.data.fit_*` options (DESIGN.md, "Fitting training grids" has the convergence run they come from)
VIEWS, RES, WINDOW = 64, 1024, 2
ITERS, LR, POINTS, REG, BATCH = 100, 0.01, 10000, 1e-4, 4
# surface points per mesh of the Chamfer distances in the report (N + M within mdb_chamfer_matrix's shared memory)
REPORT_POINTS = 16384


def camera_mvps(n_views, distance=CAMERA_DISTANCE):
    """fp32 [n_views, 4, 4] (row-major, the mdb_raster_depth convention): perspective cameras at `distance` from the
    origin on a Fibonacci sphere (direction i: y = 1 - (2 i + 1) / n, azimuth i times the golden angle), each looking at
    the origin with a square field of view of half-angle tangent TAN_HALF_FOV. Computed in float64."""
    golden = np.pi * (3.0 - np.sqrt(5.0))
    t = TAN_HALF_FOV
    proj = np.array([[1 / t, 0, 0, 0], [0, 1 / t, 0, 0],
                     [0, 0, -(FAR + NEAR) / (FAR - NEAR), -2 * FAR * NEAR / (FAR - NEAR)], [0, 0, -1, 0]])
    out = []
    for i in range(n_views):
        y = 1.0 - (2 * i + 1) / n_views
        r = np.sqrt(max(0.0, 1.0 - y * y))
        eye = distance * np.array([r * np.cos(i * golden), y, r * np.sin(i * golden)])
        f = -eye / np.linalg.norm(eye)
        up = np.array([0.0, 1.0, 0.0]) if abs(f[1]) < 0.99 else np.array([1.0, 0.0, 0.0])
        s = np.cross(f, up)
        s /= np.linalg.norm(s)
        u = np.cross(s, f)
        view = np.eye(4)
        view[0, :3], view[1, :3], view[2, :3] = s, u, -f
        view[:3, 3] = -view[:3, :3] @ eye
        out.append(proj @ view)
    return torch.tensor(np.stack(out), dtype=torch.float32)


def _host_off(off, n=None):
    o = np.asarray(off.cpu() if torch.is_tensor(off) else off, dtype=np.int64).reshape(-1)
    if o.shape[0] < 1 or o[0] != 0 or np.any(np.diff(o) < 0) or (n is not None and o[-1] != n):
        raise ValueError("offsets must be non-decreasing, start at 0 and end at the packed size")
    return o


def carve_outside(meshes, points, mvps, res=RES, window=WINDOW):
    """meshes: list of M (verts fp32 [V,3], faces int [F,3]) on one CUDA device; points fp32 [N,3]; mvps [V,4,4].
    -> bool [M, N]: True where one of the views sees the point (mdb_carve_vertices on mdb_raster_depth's buffers)."""
    dev = points.device
    verts, faces, vert_off, face_off = _pack(meshes, dev)
    points = points.float().contiguous()
    mvps = torch.as_tensor(mvps, dtype=torch.float32).reshape(-1, 16).to(dev).contiguous()
    out = torch.zeros(len(meshes), points.shape[0], dtype=torch.uint8, device=dev)
    step = max(1, _MAX_JOB_PIXELS // (res * res))
    for b in range(len(meshes)):
        for v0 in range(0, mvps.shape[0], step):
            mv = mvps[v0:v0 + step].contiguous()
            job_mesh = torch.full((mv.shape[0],), b, dtype=torch.int32, device=dev)
            depth, face_id = _raster_packed(verts, faces, vert_off, face_off, job_mesh, mv, res)
            _native.check(_native.lib().mdb_carve_vertices(_native.ptr(points), points.shape[0], _native.ptr(mv), mv.shape[0],
                                                           1, res, int(window), _native.ptr(depth), _native.ptr(face_id),
                                                           _native.ptr(out[b]), _native.current_stream()))
    return out.bool()


def carve_signs(meshes, points, mvps, res=RES, window=WINDOW):
    """-> fp32 [M, N]: +1 inside (no view sees the point), -1 outside; the sign convention of channel 0."""
    return 1.0 - 2.0 * carve_outside(meshes, points, mvps, res, window).float()


def closest_points(queries, query_off, verts, faces, vert_off, face_off):
    """Packed queries fp32 [Q,3] against packed meshes (verts fp32 [V,3], faces int64 [F,3] local to their mesh); the
    three offsets are host sequences (or tensors) of M + 1 exclusive sums. -> (dist2 fp32 [Q], face int64 [Q] within its
    mesh, ties to the lower index, closest fp32 [Q,3]); a mesh without faces gives inf, -1 and NaN."""
    q, v, f = queries.float().contiguous(), verts.float().contiguous(), faces.long().contiguous()
    qo, vo, fo = _host_off(query_off, q.shape[0]), _host_off(vert_off, v.shape[0]), _host_off(face_off, f.shape[0])
    M = qo.shape[0] - 1
    if vo.shape[0] != M + 1 or fo.shape[0] != M + 1:
        raise ValueError("query, vertex and face offsets must describe the same number of meshes")
    if f.shape[0]:
        nv = torch.from_numpy(np.repeat(np.diff(vo), np.diff(fo))).to(f.device)
        if bool(((f < 0) | (f >= nv[:, None])).any()):
            raise ValueError("face index out of range for its mesh")
    dev = q.device
    d2 = torch.empty(q.shape[0], device=dev, dtype=torch.float32)
    face = torch.empty(q.shape[0], device=dev, dtype=torch.int64)
    cp = torch.empty_like(q)
    qo_d, vo_d, fo_d = (torch.from_numpy(o).to(dev) for o in (qo, vo, fo))
    _native.check(_native.lib().mdb_closest_points(_native.ptr(q), _native.ptr(qo_d), M, int(np.diff(qo).max(initial=0)),
                                                   _native.ptr(v), _native.ptr(f), _native.ptr(vo_d), _native.ptr(fo_d),
                                                   _native.ptr(d2), _native.ptr(face), _native.ptr(cp), _native.current_stream()))
    return d2, face, cp


def nearest_vertex(queries, query_off, points, point_off):
    """Packed queries fp32 [Q,3] against packed point sets fp32 [P,3] (host offsets of M + 1 exclusive sums each)
    -> (dist2 fp32 [Q], index int64 [Q] within its set, ties to the lower index, -1 for an empty set)."""
    q, p = queries.float().contiguous(), points.float().contiguous()
    qo, po = _host_off(query_off, q.shape[0]), _host_off(point_off, p.shape[0])
    if qo.shape[0] != po.shape[0]:
        raise ValueError("query and point offsets must describe the same number of sets")
    dev = q.device
    d2 = torch.empty(q.shape[0], device=dev, dtype=torch.float32)
    idx = torch.empty(q.shape[0], device=dev, dtype=torch.int64)
    qo_d, po_d = torch.from_numpy(qo).to(dev), torch.from_numpy(po).to(dev)
    _native.check(_native.lib().mdb_nearest_vertex(_native.ptr(q), _native.ptr(qo_d), qo.shape[0] - 1,
                                                   int(np.diff(qo).max(initial=0)), _native.ptr(p), _native.ptr(po_d),
                                                   _native.ptr(d2), _native.ptr(idx), _native.current_stream()))
    return d2, idx


def segment_sum(src, keys, n_rows):
    """out [n_rows, W] with out[r] = sum of src[k] (fp32 [K, W]) over the k with keys[k] == r, added in k order: a stable
    sort of the keys, then mdb_segment_sum over the CSR rows. Deterministic, unlike a float index_add_."""
    src = src.float().contiguous()
    keys = keys.long().contiguous()
    dev = src.device
    out = torch.empty(n_rows, src.shape[1], device=dev, dtype=torch.float32)
    sorted_keys, perm = torch.sort(keys, stable=True)
    row_off = torch.searchsorted(sorted_keys, torch.arange(n_rows + 1, device=dev, dtype=torch.int64))
    _native.check(_native.lib().mdb_segment_sum(_native.ptr(src), src.shape[1], _native.ptr(perm.contiguous()),
                                                _native.ptr(row_off), n_rows, _native.ptr(out), _native.current_stream()))
    return out


def _mesh_points(verts, faces, vo, fo, n, seed, ids):
    """Surface points [B, n, 3] of packed meshes, mesh b keyed by ids[b] (independent of the batch it is in)."""
    pts = []
    for b, i in enumerate(ids):
        v, f = verts[vo[b]:vo[b + 1]], faces[fo[b]:fo[b + 1]]
        p, _ = sample_surface_points(v, f, [0, v.shape[0]], [0, f.shape[0]], n, seed, first_id=int(i))
        pts.append(p)
    return torch.cat(pts)


def _point_to_mesh(points, verts, faces, vo, fo):
    """mean over each row's points of the squared distance to its mesh -> float64 [B]."""
    B, n = points.shape[0], points.shape[1]
    d2, _, _ = closest_points(points.reshape(-1, 3), np.arange(B + 1) * n, verts, faces, vo, fo)
    return d2.view(B, n).double().mean(1)


def sample_grad(q, off, samples, s_off, s_mesh, n_points):
    """mesh -> samples: d/dm mean_s |s - nn(s)|^2 over the n_points samples of each mesh (packed [B * n_points, 3], s_mesh
    their mesh), nn the nearest marching-tet vertex of q (packed by off[:, 0]), gathered onto the vertices in a fixed
    order."""
    _, nn = nearest_vertex(samples, s_off, q, off[:, 0])
    hit = nn >= 0
    rows = nn + torch.from_numpy(off[:-1, 0]).to(q.device)[s_mesh]
    contrib = 2.0 * (q[rows.clamp(min=0)] - samples) / n_points
    return segment_sum(contrib[hit], rows[hit], q.shape[0])


def fit_deformation(mt, pos, sdf, n_verts, iters, lr, reg, data_grad):
    """The deformation fit of GridFitter and of the depth partials: `iters` Adam steps on deform [B, n_verts, 3] (from
    zero) through the differentiable marching tets `mt` with the topology the sign `sdf` [B, n_verts] fixes, pos(deform)
    placing the tet vertices. data_grad(q, off) -> fp32 [Q, 3], the gradient of the data terms with respect to the
    marching-tet vertices q (packed by off[:, 0], detached); reg * mean |deform|^2 per mesh is added. The deformation is
    clamped to [-0.99, 0.99] after every step (the reference's `clamp_deform`)."""
    deform = torch.zeros(sdf.shape[0], n_verts, 3, device=sdf.device, requires_grad=True)
    opt = torch.optim.Adam([deform], lr=lr)
    for _ in range(iters):
        mverts, _, _, _, _ = dmtet._ExtractFn.apply(mt, pos(deform), sdf)
        grad = data_grad(mverts.detach(), mt._last_off)
        r = reg * deform.square().mean(dim=(1, 2)).sum()
        opt.zero_grad()
        torch.autograd.backward([mverts, r], [grad, torch.ones_like(r)])
        opt.step()
        with torch.no_grad():
            deform.clamp_(-0.99, 0.99)
    return deform


def zero_off_surface(mt, pos, sdf, deform):
    """deform * vert_mask (fit_dmtets.py:784-789): the deformation with zeros off the vertices of the surface tets."""
    B, Nv, dev = deform.shape[0], deform.shape[1], deform.device
    _, _, _, _, vvi, off = mt._extract_raw(pos(deform), sdf)
    mask = torch.zeros(B * Nv, device=dev)
    packed_ids = vvi + torch.arange(B, device=dev).repeat_interleave(
        torch.from_numpy(np.diff(off[:, 2])).to(dev), output_size=vvi.shape[0]) * Nv
    mask[packed_ids] = 1.0
    return deform.detach() * mask.view(B, Nv, 1)


class GridFitter:
    """Meshes -> DMTet training grids for a fixed tet grid; holds the device state between batches."""

    def __init__(self, resolution, views=VIEWS, res=RES, window=WINDOW, iters=ITERS, lr=LR, points=POINTS, reg=REG,
                 max_batch=BATCH, mesh_scale=1.1, deform_scale=3.0, seed=42, device="cuda"):
        verts, tets = dmtet.load_tet_grid(resolution)
        self.R, self.res, self.window = int(resolution), int(res), int(window)
        self.iters, self.lr, self.points, self.reg = int(iters), float(lr), int(points), float(reg)
        self.max_batch, self.mesh_scale, self.deform_scale, self.seed = int(max_batch), float(mesh_scale), float(deform_scale), int(seed)
        self.device = torch.device(device)
        self.n_verts = verts.shape[0]
        self.verts = torch.tensor(verts, device=self.device)
        self.coords = dmtet.grid_coords_of_tet_vertices(self.verts.cpu()).to(self.device)
        self.mt = dmtet.MarchingTets(tets, self.n_verts, max_batch=self.max_batch)
        self.mvps = camera_mvps(int(views)).to(self.device)
        # the carved points: the tet vertices at zero deformation, placed as grid_to_tet_inputs places them
        self.grid_points = self._pos(torch.zeros(1, self.n_verts, 3, device=self.device))[0].contiguous()

    def _pos(self, deform):
        return self.verts[None] * self.mesh_scale + 2 / (self.R * 2) * deform * self.deform_scale

    def _sync(self):
        torch.cuda.synchronize(self.device)
        return time.perf_counter()

    def signs(self, meshes):
        """list of (verts, faces) -> sdf fp32 [B, Nv], +1 inside."""
        return carve_signs(meshes, self.grid_points, self.mvps, self.res, self.window)

    def __call__(self, meshes, ids=None):
        """meshes: list of (verts fp32 [V,3], faces int [F,3]), normalised (geometry.mesh_io.normalize); ids: their keys
        for the seeded surface samples (default 0..B-1). Batches of max_batch. Returns one dict per mesh: `grid` fp32
        [4,R,R,R] (CPU), `mesh` (verts, faces) extracted from that grid through grid_to_tet_inputs, and the report
        fields (counts, Chamfer distances before and after the fit, seconds of the carve and fit stages)."""
        ids = list(range(len(meshes))) if ids is None else list(ids)
        out = []
        for b0 in range(0, len(meshes), self.max_batch):
            out += self._fit_batch(meshes[b0:b0 + self.max_batch], ids[b0:b0 + self.max_batch])
        return out

    def _fit_batch(self, meshes, ids):
        dev, B, Nv = self.device, len(meshes), self.n_verts
        meshes = [(torch.as_tensor(v).to(dev, torch.float32), torch.as_tensor(f).to(dev, torch.int64)) for v, f in meshes]
        t0 = self._sync()
        sdf = self.signs(meshes).contiguous()
        t1 = self._sync()
        src_v, src_f, _, _ = _pack(meshes, dev)
        vo = np.concatenate([[0], np.cumsum([m[0].shape[0] for m in meshes])])
        fo = np.concatenate([[0], np.cumsum([m[1].shape[0] for m in meshes])])
        samples = _mesh_points(src_v, src_f, vo, fo, self.points, self.seed, ids).reshape(-1, 3).contiguous()
        s_off = np.arange(B + 1) * self.points
        s_mesh = torch.arange(B, device=dev).repeat_interleave(self.points)


        def data_grad(q, off):
            counts = torch.from_numpy(np.diff(off[:, 0])).to(dev)
            v_mesh = torch.arange(B, device=dev).repeat_interleave(counts, output_size=q.shape[0])
            # surface -> mesh: d/dm mean_m |m - cp|^2, cp held fixed
            _, _, cp = closest_points(q, off[:, 0], src_v, src_f, vo, fo)
            grad = 2.0 * (q - cp) / counts[v_mesh].float()[:, None]
            return grad + sample_grad(q, off, samples, s_off, s_mesh, self.points)

        deform = fit_deformation(self.mt, self._pos, sdf, Nv, self.iters, self.lr, self.reg, data_grad)
        t2 = self._sync()

        with torch.no_grad():
            final = zero_off_surface(self.mt, self._pos, sdf, deform)
            grids = torch.stack([tets_to_3dgrid(self.coords, sdf[b], final[b], self.R) for b in range(B)])
            sdf_g, pos_g = dmtet.grid_to_tet_inputs(grids, self.coords, self.verts, self.R, self.mesh_scale, self.deform_scale)
            fv, ff, _, _, _, foff = self.mt._extract_raw(pos_g, sdf_g)
            bv, bf, _, _, _, boff = self.mt._extract_raw(self._pos(torch.zeros_like(final)), sdf)
            report = self._distances(src_v, src_f, vo, fo, ids, (bv, bf, boff), (fv, ff, foff))
        t3 = self._sync()
        res = []
        for b in range(B):
            v0, v1, f0, f1 = foff[b, 0], foff[b + 1, 0], foff[b, 1], foff[b + 1, 1]
            entry = {"grid": grids[b].cpu(), "mesh": (fv[v0:v1], ff[f0:f1]), "faces": int(meshes[b][1].shape[0]),
                     "inside_verts": int((sdf[b] > 0).sum()), "mt_verts": int(v1 - v0), "mt_faces": int(f1 - f0),
                     "seconds_carve": (t1 - t0) / B, "seconds_fit": (t2 - t1 + t3 - t2) / B}
            entry.update({k: v[b] for k, v in report.items()})
            res.append(entry)
        return res

    def _distances(self, src_v, src_f, vo, fo, ids, before, after):
        """Per mesh: the point-cloud Chamfer distance of eval_metrics (REPORT_POINTS surface points a side,
        sample_surface_points + chamfer_matrix), which includes the sampling's own floor, and the two-sided
        point-to-surface distance (mean squared distance of each side's points to the other surface), which does not;
        before and after the fit. None for a mesh that marching tets leaves empty."""
        out = {f"{k}_{n}": [None] * len(ids) for k in ("chamfer", "surface_distance") for n in ("before", "after")}
        for b, i in enumerate(ids):
            sv, sf = src_v[vo[b]:vo[b + 1]], src_f[fo[b]:fo[b + 1]]
            ref = _mesh_points(sv, sf, [0, sv.shape[0]], [0, sf.shape[0]], REPORT_POINTS, self.seed + 1, [i])
            for name, (v, f, off) in (("before", before), ("after", after)):
                mv, mf = v[off[b, 0]:off[b + 1, 0]], f[off[b, 1]:off[b + 1, 1]]
                if mf.shape[0] == 0:
                    continue
                pts = _mesh_points(mv, mf, [0, mv.shape[0]], [0, mf.shape[0]], REPORT_POINTS, self.seed + 1, [i])
                out[f"chamfer_{name}"][b] = float(chamfer_matrix(pts, ref)[0, 0])
                to_src = _point_to_mesh(pts, sv, sf, [0, sv.shape[0]], [0, sf.shape[0]])
                to_fit = _point_to_mesh(ref, mv, mf, [0, mv.shape[0]], [0, mf.shape[0]])
                out[f"surface_distance_{name}"][b] = float(to_src[0] + to_fit[0])
        return out
