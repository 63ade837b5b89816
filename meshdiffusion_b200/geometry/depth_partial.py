"""Partial DMTets from one observed depth map (`--mode=partial_from_depth`, and `--mode=make_partial` with
`eval.partial_from="depth"`).

`singleview.PartialDMTets` takes the sign and the deformation of a partial from a complete grid; only its visibility
comes from the view. Here everything comes from what one camera sees: a depth map and its camera (csrc/depth_partial.cu
plus the fitting and visibility kernels):

* `unproject` -- the depth map as the z / w and validity buffers the carving kernel reads, the world point of every
  pixel centre, and the pixels beside a depth step of more than one grid-cell edge (silhouettes, not surfaces)
  (`mdb_depth_unproject`);
* `depth_closest_points` -- the closest point on the observed surface, searched over the two triangles of every 2 x 2
  block of valid, non-edge pixels in a window of one cell edge around the query's projection, at most 64 px a side
  (`mdb_depth_closest_points`);
* `DepthPartials` -- observations -> partial DMTets: the sign by carving with the one view, the deformation by the Adam
  loop of `fit.GridFitter` against the observed surface, and the visibility of `PartialDMTets` on the fitted mesh.

A camera is `{"view": k}` (the reference's validation pose `singleview.view_mvp(k, res)`) or `{"mv": ..., "proj": ...}`,
two row-major 4 x 4 matrices in the OpenGL convention of `view_mvp`'s factors. A depth map is float32 [res, res], the
positive depth along -z_cam in the frame of `--mode=export`'s meshes, 0 or non-finite where there is no surface; row 0
is clip y = -1, the rasterizer's layout.

Every step is deterministic (no float atomics), so the same observations give the same partials bit for bit, and an
observation's partial does not depend on the other observations of its batch.
"""
import time

import numpy as np
import torch

from .. import _native
from . import dmtet
from .fit import ITERS, LR, POINTS, REG, WINDOW, _host_off, fit_deformation, sample_grad, zero_off_surface
from .formats import partial_dmtet_from_visibility
from .singleview import (FAR, FOVY, NEAR, RADIUS, VIEWS_PER_TURN, _MAX_JOB_PIXELS, _jobs, _perspective, _raster_packed,
                         _rotate_x, _rotate_y, _translate, _visible_packed)

MAX_RES = 4096  # the rasterizer behind the visible-tet test draws square images; 4096^2 keeps a batch's buffers small
_PERSPECTIVE_ZEROS = ((0, 1), (0, 3), (1, 0), (1, 3), (2, 0), (2, 1), (3, 0), (3, 1), (3, 3))


def view_camera(view):
    """(mv, proj) fp32 [4, 4] of the validation pose `view`; proj @ mv is singleview.view_mvp(view, res) bit for bit."""
    ang = (view / VIEWS_PER_TURN) * np.pi * 2
    return _translate(0, 0, -RADIUS) @ (_rotate_x(-0.4) @ _rotate_y(ang)), _perspective(FOVY, 1.0, NEAR, FAR)


def _matrix(value, name):
    m = torch.as_tensor(np.asarray(value, dtype=np.float64), dtype=torch.float32)
    if m.shape != (4, 4) or not bool(torch.isfinite(m).all()):
        raise ValueError(f"the camera's {name} must be a finite 4 x 4 matrix")
    return m


def check_perspective(proj):
    """Raises unless proj is an OpenGL perspective matrix: rows [p00 0 p02 0], [0 p11 p12 0], [0 0 A B], [0 0 -1 0] with
    p00, p11 and B non-zero (what the back-projection inverts)."""
    p = np.asarray(proj, np.float64)
    if (p[3, 2] != -1.0 or any(p[i, j] != 0.0 for i, j in _PERSPECTIVE_ZEROS) or p[0, 0] == 0.0 or p[1, 1] == 0.0
            or p[2, 3] == 0.0):
        raise ValueError("proj is not a perspective matrix: expected rows [p00 0 p02 0], [0 p11 p12 0], [0 0 A B], "
                         "[0 0 -1 0] with p00, p11, B non-zero")


def parse_camera(entry):
    """An observation's camera, `{"view": k}` or `{"mv": [[..]], "proj": [[..]]}` -> dict of fp32 [4, 4] tensors `mvp`
    (proj @ mv, in float32 as view_mvp multiplies), `proj`, `mv` and `inv_mv` (inverted in float64)."""
    has_view = "view" in entry
    has_matrices = "mv" in entry or "proj" in entry
    if has_view and has_matrices:
        raise ValueError("an observation gives its camera either as 'view' or as 'mv' and 'proj', not both")
    if has_view:
        view = entry["view"]
        if isinstance(view, bool) or not isinstance(view, (int, np.integer)):
            raise ValueError(f"'view' must be an integer, got {view!r}")
        mv, proj = view_camera(int(view))
    elif has_matrices:
        if "mv" not in entry or "proj" not in entry:
            raise ValueError("an observation's camera needs both 'mv' and 'proj'")
        mv, proj = _matrix(entry["mv"], "mv"), _matrix(entry["proj"], "proj")
    else:
        raise ValueError("an observation has no camera: give 'view' or 'mv' and 'proj'")
    check_perspective(proj)
    m = mv.double()
    if not bool((m[3] == torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64)).all()) or abs(float(torch.linalg.det(m))) < 1e-12:
        raise ValueError("mv must be an invertible affine matrix with last row [0 0 0 1]")
    return {"mvp": proj @ mv, "proj": proj, "mv": mv, "inv_mv": torch.linalg.inv(m).float()}


def check_depth(depth, name="depth"):
    """-> the depth map as fp32 [res, res]; raises on a non-square image, a side outside [2, MAX_RES] or a negative
    depth (0 and non-finite values mean no surface)."""
    d = np.asarray(depth)
    if d.ndim != 2 or d.shape[0] != d.shape[1]:
        raise ValueError(f"{name}: a depth map must be a square [res, res] image, got shape {d.shape}")
    if not 2 <= d.shape[0] <= MAX_RES:
        raise ValueError(f"{name}: the image side must be in [2, {MAX_RES}], got {d.shape[0]}")
    d = d.astype(np.float32)
    if bool((np.isfinite(d) & (d < 0)).any()):
        raise ValueError(f"{name}: negative depths (the depth is the positive distance along the viewing axis)")
    return d


def camera_depth(zbuf, face_id, proj):
    """The rasterizer's z / w buffers -> camera depth B / (z + A) (proj rows [0 0 A B], [0 0 -1 0]), 0 where empty."""
    A, Bc = float(proj[2, 2]), float(proj[2, 3])
    return torch.where(face_id >= 0, Bc / (zbuf + A), torch.zeros_like(zbuf))


def unproject(depth, proj, inv_mv, max_jump):
    """depth fp32 [B, res, res], proj / inv_mv [B, 16] on one CUDA device -> (zbuf fp32 [B, res, res], valid int32 (0
    surface, -1 empty), points fp32 [B, res, res, 3], edge uint8) as mdb_depth_unproject writes them."""
    depth = depth.float().contiguous()
    B, res = depth.shape[0], depth.shape[-1]
    dev = depth.device
    proj = proj.reshape(B, 16).to(dev, torch.float32).contiguous()
    inv_mv = inv_mv.reshape(B, 16).to(dev, torch.float32).contiguous()
    zbuf = torch.empty(B, res, res, device=dev, dtype=torch.float32)
    valid = torch.empty(B, res, res, device=dev, dtype=torch.int32)
    points = torch.empty(B, res, res, 3, device=dev, dtype=torch.float32)
    edge = torch.empty(B, res, res, device=dev, dtype=torch.uint8)
    _native.check(_native.lib().mdb_depth_unproject(_native.ptr(depth), B, res, _native.ptr(proj), _native.ptr(inv_mv),
                                                    float(max_jump), _native.ptr(zbuf), _native.ptr(valid),
                                                    _native.ptr(points), _native.ptr(edge), _native.current_stream()))
    return zbuf, valid, points, edge


def depth_closest_points(queries, query_off, mvp, proj, radius, points, valid, edge):
    """Packed queries fp32 [Q, 3] (host offsets of B + 1 exclusive sums) against B observations (mvp, proj [B, 16];
    points, valid, edge from `unproject`) -> (dist2 fp32 [Q], closest fp32 [Q, 3], found bool [Q])."""
    q = queries.float().contiguous()
    qo = _host_off(query_off, q.shape[0])
    B, res = points.shape[0], points.shape[1]
    if qo.shape[0] != B + 1:
        raise ValueError("query offsets must describe one set per observation")
    dev = q.device
    mvp = mvp.reshape(B, 16).to(dev, torch.float32).contiguous()
    proj = proj.reshape(B, 16).to(dev, torch.float32).contiguous()
    d2 = torch.empty(q.shape[0], device=dev, dtype=torch.float32)
    cp = torch.empty_like(q)
    found = torch.empty(q.shape[0], device=dev, dtype=torch.uint8)
    qo_d = torch.from_numpy(qo).to(dev)
    _native.check(_native.lib().mdb_depth_closest_points(_native.ptr(q), _native.ptr(qo_d), B, int(np.diff(qo).max(initial=0)),
                                                         res, _native.ptr(mvp), _native.ptr(proj), float(radius),
                                                         _native.ptr(points.contiguous()), _native.ptr(valid.contiguous()),
                                                         _native.ptr(edge.contiguous()), _native.ptr(d2), _native.ptr(cp),
                                                         _native.ptr(found), _native.current_stream()))
    return d2, cp, found.bool()


def render_depth(make, grids):
    """Camera depth maps fp32 [B, V, res, res] of the meshes of grids [B, 4, R, R, R] from the views of `make` (a
    singleview.PartialDMTets), drawn by the rasterizer the visible-tet test uses; 0 where the view sees no surface."""
    B, V, res = grids.shape[0], len(make.views), make.res
    sdf, pos = dmtet.grid_to_tet_inputs(grids.to(make.device, torch.float32), make.coords, make.verts, make.R,
                                        make.mesh_scale, make.deform_scale)
    verts, faces, _, _, _, off = make.mt._extract_raw(pos, sdf)
    vert_off = torch.from_numpy(np.ascontiguousarray(off[:-1, 0])).to(make.device)
    face_off = torch.from_numpy(np.ascontiguousarray(off[:, 1])).to(make.device)
    job_mesh, mvp = _jobs(B, make.mvps, make.device)
    proj = view_camera(0)[1]
    out = torch.empty(B * V, res, res, device=make.device)
    step = max(1, _MAX_JOB_PIXELS // (res * res))
    for j0 in range(0, B * V, step):
        z, fid = _raster_packed(verts, faces, vert_off, face_off, job_mesh[j0:j0 + step].contiguous(),
                                mvp[j0:j0 + step].contiguous(), res)
        out[j0:j0 + step] = camera_depth(z, fid, proj)
    return out.view(B, V, res, res)


def grid_box(resolution, mesh_scale=1.1, deform_scale=3.0):
    """(lo, hi) fp32 [3]: the box the tet vertices of the R grid can reach, placed at mesh_scale and moved by the largest
    deformation (0.99 * deform_scale / R)."""
    verts = torch.from_numpy(dmtet.load_tet_grid(resolution)[0]) * mesh_scale
    reach = 0.99 * 2 / (resolution * 2) * deform_scale
    return verts.min(0).values - reach, verts.max(0).values + reach


def check_inside_grid(points, valid, lo, hi, keys=None):
    """Raises when an observed point (points [B, res, res, 3] where valid == 0) lies outside the box lo .. hi."""
    outside = ((points < lo) | (points > hi)).any(-1) & (valid == 0)
    for b in range(points.shape[0]):
        n = int(outside[b].sum())
        if n:
            key = keys[b] if keys is not None else b
            raise ValueError(f"observation {key}: {n} observed points lie outside the grid (the box {lo.tolist()} .. "
                             f"{hi.tolist()} the deformed tet grid can reach); is the depth in the grid's units?")


class DepthPartials:
    """Observations (depth map + camera) -> partial DMTets for a fixed tet grid; holds the device state between calls."""

    def __init__(self, resolution, window=WINDOW, iters=ITERS, lr=LR, points=POINTS, reg=REG, max_batch=8, mesh_scale=1.1,
                 deform_scale=3.0, seed=42, device="cuda"):
        verts, tets = dmtet.load_tet_grid(resolution)
        self.R, self.window = int(resolution), int(window)
        self.iters, self.lr, self.points, self.reg = int(iters), float(lr), int(points), float(reg)
        self.max_batch, self.mesh_scale, self.deform_scale, self.seed = int(max_batch), float(mesh_scale), float(deform_scale), int(seed)
        self.device = torch.device(device)
        self.n_verts = verts.shape[0]
        self.verts = torch.tensor(verts, device=self.device)
        self.tets = torch.tensor(tets, device=self.device, dtype=torch.int32).contiguous()
        self.mt = dmtet.MarchingTets(tets, self.n_verts, max_batch=self.max_batch)
        # one grid-cell edge: the tet grid's vertex spacing, placed at mesh_scale
        self.cell = float(np.diff(np.unique(verts[:, 0]))[0]) * self.mesh_scale
        self.grid_points = self._pos(torch.zeros(1, self.n_verts, 3, device=self.device))[0].contiguous()
        self.lo, self.hi = (t.to(self.device) for t in grid_box(self.R, self.mesh_scale, self.deform_scale))

    def _pos(self, deform):
        return self.verts[None] * self.mesh_scale + 2 / (self.R * 2) * deform * self.deform_scale

    def _sync(self):
        torch.cuda.synchronize(self.device)
        return time.perf_counter()

    def __call__(self, depths, cameras, keys=None):
        """depths: list of fp32 [res, res] arrays (one res per call); cameras: parse_camera dicts; keys: per observation a
        tuple of non-negative ints that seeds its observed-point samples (default (0,), (1,), ...). Batches of max_batch.
        Returns one (the `dmtet.pt` dictionary, report) per observation; the report holds the visible tet and vertex
        counts, the mean distance to the observation before and after the fit and the seconds of each stage."""
        keys = [(i,) for i in range(len(depths))] if keys is None else [tuple(int(x) for x in k) for k in keys]
        depths = [check_depth(d, f"observation {k}") for d, k in zip(depths, keys)]
        if len({d.shape[0] for d in depths}) > 1:
            raise ValueError("the depth maps of one call must share one resolution")
        out = []
        for b0 in range(0, len(depths), self.max_batch):
            out += self._batch(depths[b0:b0 + self.max_batch], cameras[b0:b0 + self.max_batch], keys[b0:b0 + self.max_batch])
        return out

    def _observed_distance(self, deform, sdf, mvp, proj, pts, valid, edge):
        """Per observation: the mean distance to the observed surface of the marching-tet vertices within one cell edge of
        it (the vertices the fit pulls); None when there are none."""
        q, _, _, _, _, off = self.mt._extract_raw(self._pos(deform), sdf)
        d2, _, found = depth_closest_points(q, off[:, 0], mvp, proj, self.cell, pts, valid, edge)
        near = found & (d2 <= self.cell * self.cell)
        out = []
        for b in range(sdf.shape[0]):
            m = near[off[b, 0]:off[b + 1, 0]]
            out.append(float(d2[off[b, 0]:off[b + 1, 0]][m].double().sqrt().mean()) if bool(m.any()) else None)
        return out

    def _batch(self, depths, cameras, keys):
        dev, B, Nv = self.device, len(depths), self.n_verts
        res = depths[0].shape[0]
        mvp = torch.stack([c["mvp"].reshape(16) for c in cameras]).to(dev).contiguous()
        proj = torch.stack([c["proj"].reshape(16) for c in cameras]).to(dev).contiguous()
        inv_mv = torch.stack([c["inv_mv"].reshape(16) for c in cameras]).to(dev).contiguous()
        t0 = self._sync()
        zbuf, valid, pts, edge = unproject(torch.from_numpy(np.stack(depths)).to(dev), proj, inv_mv, self.cell)
        surface = valid == 0
        check_inside_grid(pts, valid, self.lo, self.hi, keys)
        usable = (surface & (edge == 0)).reshape(B, -1)
        samples = []
        for b in range(B):
            idx = usable[b].nonzero().view(-1)
            if idx.numel() == 0:
                raise ValueError(f"observation {keys[b]}: the depth map shows no surface away from depth steps")
            pick = np.random.default_rng([self.seed, *keys[b]]).integers(0, idx.numel(), self.points)
            samples.append(pts[b].reshape(-1, 3)[idx[torch.from_numpy(pick).to(dev)]])
        samples = torch.cat(samples).contiguous()
        s_off = np.arange(B + 1) * self.points
        s_mesh = torch.arange(B, device=dev).repeat_interleave(self.points)
        t1 = self._sync()

        # the sign: the one view carves the undeformed tet vertices; the rest, occluded vertices included, is inside
        outside_v = torch.zeros(B, Nv, dtype=torch.uint8, device=dev)
        for b in range(B):
            _native.check(_native.lib().mdb_carve_vertices(_native.ptr(self.grid_points), Nv, _native.ptr(mvp[b]), 1, 1, res,
                                                           self.window, _native.ptr(zbuf[b]), _native.ptr(valid[b]),
                                                           _native.ptr(outside_v[b]), _native.current_stream()))
        sdf = (1.0 - 2.0 * outside_v.float()).contiguous()
        t2 = self._sync()

        r2 = self.cell * self.cell

        def data_grad(q, off):
            counts = torch.from_numpy(np.diff(off[:, 0])).to(dev)
            v_mesh = torch.arange(B, device=dev).repeat_interleave(counts, output_size=q.shape[0])
            # observation -> mesh: d/dm mean_m |m - cp|^2 over the vertices within one cell edge of the observation
            d2, cp, found = depth_closest_points(q, off[:, 0], mvp, proj, self.cell, pts, valid, edge)
            near = found & (d2 <= r2)
            n_near = torch.bincount(v_mesh[near], minlength=B).clamp(min=1)
            grad = torch.where(near[:, None], 2.0 * (q - cp) / n_near[v_mesh].float()[:, None], torch.zeros_like(q))
            return grad + sample_grad(q, off, samples, s_off, s_mesh, self.points)

        zero = torch.zeros(B, Nv, 3, device=dev)
        before = self._observed_distance(zero, sdf, mvp, proj, pts, valid, edge)
        deform = fit_deformation(self.mt, self._pos, sdf, Nv, self.iters, self.lr, self.reg, data_grad)
        with torch.no_grad():
            final = zero_off_surface(self.mt, self._pos, sdf, deform)
        after = self._observed_distance(final, sdf, mvp, proj, pts, valid, edge)
        t3 = self._sync()

        # visibility of the fitted mesh from the same camera, as PartialDMTets computes it
        pos = self._pos(final).contiguous()
        verts, faces, _, f2t, _, off = self.mt._extract_raw(pos, sdf)
        vert_off = torch.from_numpy(np.ascontiguousarray(off[:-1, 0])).to(dev)
        face_off = torch.from_numpy(np.ascontiguousarray(off[:, 1])).to(dev)
        job_mesh = torch.arange(B, dtype=torch.int32, device=dev)
        visible = torch.empty(B, self.tets.shape[0], dtype=torch.bool, device=dev)
        rast = torch.empty_like(visible)
        step = max(1, _MAX_JOB_PIXELS // (res * res))
        for j0 in range(0, B, step):
            jm, mv = job_mesh[j0:j0 + step].contiguous(), mvp[j0:j0 + step].contiguous()
            depth_r, face_id = _raster_packed(verts, faces, vert_off, face_off, jm, mv, res)
            visible[j0:j0 + step], rast[j0:j0 + step] = _visible_packed(pos, self.tets, f2t, face_off, jm, mv, depth_r, face_id)
        out = []
        for b in range(B):
            vis_id = visible[b].nonzero().view(-1)
            d = partial_dmtet_from_visibility(self.tets, Nv, sdf[b], final[b], vis_id, rast[b].nonzero().view(-1))
            out.append((d, {"visible_tets": int(vis_id.numel()), "visible_verts": int(d["vis"].sum()),
                            "visible_and_rast_verts": int(d["vis_rast"].sum()), "observed_pixels": int(surface[b].sum()),
                            "edge_pixels": int(edge[b].sum()), "inside_verts": int((sdf[b] > 0).sum()),
                            "distance_before": before[b], "distance_after": after[b]}))
        t4 = self._sync()
        for _, rep in out:
            rep.update(seconds_unproject=(t1 - t0) / B, seconds_carve=(t2 - t1) / B, seconds_fit=(t3 - t2) / B,
                       seconds_visibility=(t4 - t3) / B)
        return out
