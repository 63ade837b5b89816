"""Single-view partial DMTets, the input of `--mode=cond_gen` (`config.eval.partial_dmtet_path`).

The reference makes that input at the end of nvdiffrec/fit_singleview.py:783-827: it renders the fitted DMTet from one
validation pose with nvdiffrast and marks the tetrahedra the view sees (nvdiffrec/lib/render/render.py:335-407). Here the
DMTet comes from a grid (the sign of channel 0 and the deformation of channels 1-3, which is what the fit approximates)
and the view is rendered by the library's own kernels (csrc/raster.cu):

* `view_mvp` -- the reference's validation camera;
* `rasterize` -- first-layer depth and face ids (`mdb_raster_depth`);
* `visible_tets` -- the reference's visible-tet test on those buffers and the tets owning rasterized faces
  (`mdb_visible_tets`);
* `partial_dmtets` -- grid -> tet inputs -> marching tets -> rasterization -> visibility -> the `dmtet.pt` dictionary.
"""
import ctypes

import numpy as np
import torch

from .. import _native
from . import dmtet
from .formats import partial_dmtet_from_visibility

RADIUS = 2.0           # fit_singleview.py:44
FOVY = np.deg2rad(45)  # DatasetMesh.fovy (dataset_mesh.py:35)
NEAR, FAR = 0.1, 1000.0  # cam_near_far (fit_singleview.py:637)
VIEWS_PER_TURN = 50    # the validation poses go round the object in 50 steps (dataset_mesh.py:70)
DEFAULT_RES = 1000     # train_res of nvdiffrec/configs/res{64,128}.json; spp 1
# the job buffers of one launch (depth, face id and the 64-bit depth-test scratch, 16 bytes a pixel) stay under ~1 GiB
_MAX_JOB_PIXELS = 1 << 26


def _perspective(fovy, aspect, n, f):
    y = np.tan(fovy / 2)
    return torch.tensor([[1 / (y * aspect), 0, 0, 0],
                         [0, 1 / -y, 0, 0],
                         [0, 0, -(f + n) / (f - n), -(2 * f * n) / (f - n)],
                         [0, 0, -1, 0]], dtype=torch.float32)


def _translate(x, y, z):
    return torch.tensor([[1, 0, 0, x], [0, 1, 0, y], [0, 0, 1, z], [0, 0, 0, 1]], dtype=torch.float32)


def _rotate_x(a):
    s, c = np.sin(a), np.cos(a)
    return torch.tensor([[1, 0, 0, 0], [0, c, s, 0], [0, -s, c, 0], [0, 0, 0, 1]], dtype=torch.float32)


def _rotate_y(a):
    s, c = np.sin(a), np.cos(a)
    return torch.tensor([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]], dtype=torch.float32)


def view_mvp(view, res=DEFAULT_RES):
    """fp32 [4, 4] model-view-projection of the reference's validation pose `itr = view` (DatasetMesh._rotate_scene,
    dataset_mesh.py:67-76) for a square res x res image.

    fit_singleview.py:786-788 advances the validation iterator `angle_ind` times before it renders, so the reference's
    `--angle-ind k` is `view = k - 1` here."""
    ang = (view / VIEWS_PER_TURN) * np.pi * 2
    mv = _translate(0, 0, -RADIUS) @ (_rotate_x(-0.4) @ _rotate_y(ang))
    return _perspective(FOVY, res / res, NEAR, FAR) @ mv


def _pack(meshes, device):
    """[(verts [V,3], faces [F,3])] -> packed verts, faces, device vert_off [M], face_off [M+1]."""
    nv = [int(v.shape[0]) for v, _ in meshes]
    nf = [int(f.shape[0]) for _, f in meshes]
    for (v, f), n in zip(meshes, nv):
        if f.numel() and (int(f.min()) < 0 or int(f.max()) >= n):
            raise ValueError("a face index is outside its mesh")
    verts = torch.cat([v.reshape(-1, 3) for v, _ in meshes]).to(device, torch.float32).contiguous()
    faces = torch.cat([f.reshape(-1, 3) for _, f in meshes]).to(device, torch.int64).contiguous()
    vert_off = torch.tensor(np.concatenate([[0], np.cumsum(nv)[:-1]]), dtype=torch.int64, device=device)
    face_off = torch.tensor(np.concatenate([[0], np.cumsum(nf)]), dtype=torch.int64, device=device)
    return verts, faces, vert_off, face_off


def _jobs(n_meshes, mvps, device):
    """Every mesh from every view, mesh-major: job_mesh int32 [M*V], mvp fp32 [M*V, 16]."""
    V = mvps.shape[0]
    job_mesh = torch.arange(n_meshes, dtype=torch.int32, device=device).repeat_interleave(V)
    mvp = mvps.reshape(V, 16).to(device, torch.float32).repeat(n_meshes, 1).contiguous()
    return job_mesh, mvp


def _raster_packed(verts, faces, vert_off, face_off, job_mesh, mvp, res):
    J = job_mesh.shape[0]
    dev = verts.device
    depth = torch.empty(J, res, res, device=dev, dtype=torch.float32)
    face_id = torch.empty(J, res, res, device=dev, dtype=torch.int32)
    scratch = torch.empty(J, res, res, device=dev, dtype=torch.int64)
    behind = torch.empty(J, device=dev, dtype=torch.int32)
    _native.check(_native.lib().mdb_raster_depth(_native.ptr(verts), _native.ptr(faces), _native.ptr(vert_off),
                                                 _native.ptr(face_off), _native.ptr(job_mesh), _native.ptr(mvp), J, res,
                                                 _native.ptr(scratch), _native.ptr(depth), _native.ptr(face_id),
                                                 _native.ptr(behind), _native.current_stream()))
    n = int(behind.sum())
    if n:
        raise ValueError(f"{n} triangles have a vertex at or behind the camera plane (w <= 0); there is no near-plane clipping")
    return depth, face_id


def rasterize(meshes, mvps, res=DEFAULT_RES):
    """Depth and face ids of every mesh from every view.

    meshes: list of M (verts fp32 [V,3], faces int [F,3]) on one CUDA device; mvps [V,4,4]. Returns depth fp32
    [M, V, res, res] (z / w of the nearest fragment, 100 where empty) and face_id int32 [M, V, res, res] (index of the
    face within its mesh, -1 where empty). Row 0 is clip y = -1, nvdiffrast's layout. Raises if a triangle has a vertex
    at w <= 0."""
    mvps = torch.as_tensor(mvps, dtype=torch.float32).reshape(-1, 4, 4)
    dev = meshes[0][0].device
    packed = _pack(meshes, dev)
    job_mesh, mvp = _jobs(len(meshes), mvps, dev)
    depth, face_id = _raster_packed(*packed, job_mesh, mvp, res)
    return depth.view(len(meshes), -1, res, res), face_id.view(len(meshes), -1, res, res)


def _visible_packed(pos, tets, f2t, face_off, job_mesh, mvp, depth, face_id):
    J, res = job_mesh.shape[0], depth.shape[-1]
    T = tets.shape[0]
    stride = 0 if pos.dim() == 2 else pos.shape[1] * 3
    vis = torch.empty(J, T, device=pos.device, dtype=torch.uint8)
    rast = torch.empty_like(vis)
    _native.check(_native.lib().mdb_visible_tets(_native.ptr(pos), stride, _native.ptr(tets), T, _native.ptr(f2t),
                                                 _native.ptr(face_off), _native.ptr(job_mesh), _native.ptr(mvp), J, res,
                                                 _native.ptr(depth), _native.ptr(face_id), _native.ptr(vis),
                                                 _native.ptr(rast), _native.current_stream()))
    return vis.bool(), rast.bool()


def visible_tets(pos, tets, f2t, mvps, depth, face_id):
    """The reference's visible-tet test (render.py:346-407) on the buffers `rasterize` returned.

    pos fp32 [M, Nv, 3] (or [Nv, 3], shared): the deformed tet vertices the meshes were extracted from; tets int [T, 4];
    f2t: list of M face -> tet maps (what MarchingTets.extract returns); mvps [V, 4, 4]; depth, face_id [M, V, res, res].
    Returns visible, rast: bool [M, V, T]. A tet is visible when its centre's pixel is in view and the 15 x 15 window
    around it is empty or nowhere nearer than the centre; it is rasterized when it owns a face in the buffer."""
    M, V, res = depth.shape[0], depth.shape[1], depth.shape[-1]
    dev = depth.device
    pos = pos.to(dev, torch.float32).contiguous()
    tets = torch.as_tensor(tets).to(dev, torch.int32).contiguous()
    f2t_packed = torch.cat([torch.as_tensor(f).reshape(-1) for f in f2t]).to(dev, torch.int64).contiguous()
    face_off = torch.tensor(np.concatenate([[0], np.cumsum([int(torch.as_tensor(f).numel()) for f in f2t])]),
                            dtype=torch.int64, device=dev)
    ids = face_id.reshape(M, -1)
    for m in range(M):
        hi = int(ids[m].max()) if ids[m].numel() else -1
        if hi >= int(face_off[m + 1] - face_off[m]):
            raise ValueError("a face id is outside its mesh's face -> tet map")
    job_mesh, mvp = _jobs(M, torch.as_tensor(mvps, dtype=torch.float32).reshape(-1, 4, 4), dev)
    vis, rast = _visible_packed(pos, tets, f2t_packed, face_off, job_mesh, mvp,
                                depth.reshape(M * V, res, res).contiguous(), face_id.reshape(M * V, res, res).contiguous())
    return vis.view(M, V, -1), rast.view(M, V, -1)


class PartialDMTets:
    """Grid -> partial DMTets for a fixed tet grid, set of views and resolution; holds the device state between calls."""

    def __init__(self, resolution, views=(0,), res=DEFAULT_RES, mesh_scale=1.1, deform_scale=3.0, device="cuda", max_batch=8):
        verts, tets = dmtet.load_tet_grid(resolution)
        self.R, self.res, self.views = resolution, int(res), tuple(int(v) for v in views)
        self.mesh_scale, self.deform_scale, self.max_batch = mesh_scale, deform_scale, max_batch
        self.device = torch.device(device)
        self.n_verts = verts.shape[0]
        self.verts = torch.tensor(verts, device=self.device)
        self.coords = dmtet.grid_coords_of_tet_vertices(self.verts.cpu()).to(self.device)
        self.tets = torch.tensor(tets, device=self.device, dtype=torch.int32).contiguous()
        self.mt = dmtet.MarchingTets(tets, self.n_verts, max_batch=max_batch)
        self.mvps = torch.stack([view_mvp(v, self.res) for v in self.views])

    def flags(self, grids):
        """grids [B,4,R,R,R] (B <= max_batch) -> (sdf [B,Nv], deform [B,Nv,3], visible, rast bool [B,V,T])."""
        B = grids.shape[0]
        grids = grids.to(self.device, torch.float32)
        sdf, pos = dmtet.grid_to_tet_inputs(grids, self.coords, self.verts, self.R, self.mesh_scale, self.deform_scale)
        c = self.coords
        deform = grids[:, 1:, c[:, 0], c[:, 1], c[:, 2]].transpose(1, 2)
        verts, faces, _, f2t, _, off = self.mt._extract_raw(pos, sdf)
        vert_off = torch.from_numpy(np.ascontiguousarray(off[:-1, 0])).to(self.device)
        face_off = torch.from_numpy(np.ascontiguousarray(off[:, 1])).to(self.device)
        V = len(self.views)
        visible = torch.empty(B, V, self.tets.shape[0], dtype=torch.bool, device=self.device)
        rast = torch.empty_like(visible)
        job_mesh, mvp = _jobs(B, self.mvps, self.device)
        step = max(1, _MAX_JOB_PIXELS // (self.res * self.res))
        for j0 in range(0, B * V, step):
            jm, mv = job_mesh[j0:j0 + step].contiguous(), mvp[j0:j0 + step].contiguous()
            depth, face_id = _raster_packed(verts, faces, vert_off, face_off, jm, mv, self.res)
            v, r = _visible_packed(pos, self.tets, f2t, face_off, jm, mv, depth, face_id)
            visible.view(B * V, -1)[j0:j0 + step] = v
            rast.view(B * V, -1)[j0:j0 + step] = r
        return sdf, deform, visible, rast

    def __call__(self, grids):
        """grids [B,4,R,R,R] -> out[b][v] = (the `dmtet.pt` dictionary, number of visible tets)."""
        out = []
        for b0 in range(0, grids.shape[0], self.max_batch):
            sdf, deform, visible, rast = self.flags(grids[b0:b0 + self.max_batch])
            for b in range(sdf.shape[0]):
                row = []
                for v in range(len(self.views)):
                    vis_id = visible[b, v].nonzero().view(-1)
                    d = partial_dmtet_from_visibility(self.tets, self.n_verts, sdf[b], deform[b], vis_id,
                                                      rast[b, v].nonzero().view(-1))
                    row.append((d, int(vis_id.numel())))
                out.append(row)
        return out


def partial_dmtets(grids, views=(0,), res=DEFAULT_RES, mesh_scale=1.1, deform_scale=3.0):
    """grids [B,4,R,R,R] (CUDA) -> out[b][v] = (partial DMTet dictionary {'sdf', 'deform', 'vis', 'vis_rast'} of shape b
    seen from validation view views[v], number of visible tets). `sdf` is sign(channel 0) and `deform` channels 1-3 at
    the tet vertices; the mesh is placed with `mesh_scale` and `deform_scale` as in eval (grid_to_tet_inputs)."""
    return PartialDMTets(grids.shape[-1], views, res, mesh_scale, deform_scale, grids.device)(grids)
