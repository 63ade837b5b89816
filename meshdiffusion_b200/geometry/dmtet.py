"""Marching tetrahedra on the sm_90a kernels, behind the reference's `DMTet()(pos_nx3, sdf_n, tet_fx4)` call
(nvdiffrec/lib/geometry/dmtet.py:32-163), plus the grid -> tet-vertex gather of nvdiffrec/eval.py:389-419 and the
vertex placement of dmtet.py:293-304. Integer outputs are int64 and bit-exact with the reference's ordering.
"""
import ctypes
import os

import numpy as np
import torch

from .. import _native

_DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data", "tets")


def tet_grid_path(resolution, root=None):
    """`<root>/data/tets/<R>_tets_cropped.npz` like DMTetGeometry (dmtet.py:219), else the in-tree copy."""
    if root is not None:
        p = os.path.join(root, "data/tets/{}_tets_cropped.npz".format(resolution))
        if os.path.exists(p):
            return p
    return os.path.join(_DATA, "{}_tets_cropped.npz".format(resolution))


def load_tet_grid(resolution, root=None):
    t = np.load(tet_grid_path(resolution, root))
    return t["vertices"].astype(np.float32), t["indices"].astype(np.int32)


def grid_coords_of_tet_vertices(vertices):
    """Integer cubic-grid coordinate of every tet vertex (eval.py:391-397, evaler.py:187-195)."""
    v = torch.as_tensor(vertices)
    u = v.unique()
    dx = u[1] - u[0]
    return torch.round((v - v.min()) / dx).long()


def grid_mask_from_tets(resolution, root=None):
    """data/get_tet_mask.py: 1 where a tet vertex lands. Identical to the shipped data/grid_mask_<R>.pt."""
    verts, _ = load_tet_grid(resolution, root)
    c = grid_coords_of_tet_vertices(verts)
    mask = torch.zeros(resolution, resolution, resolution)
    mask[c[:, 0], c[:, 1], c[:, 2]] = 1.0
    return mask


class MarchingTets:
    """Static tet grid prepared once on the device; extracts meshes for batches of samples."""

    def __init__(self, tets, n_verts, max_batch=1):
        L = _native.lib()
        tets = np.ascontiguousarray(np.asarray(tets, dtype=np.int32))
        self.F, self.Nv, self.max_batch = tets.shape[0], int(n_verts), max_batch
        self._h = ctypes.c_void_p()
        _native.check(L.mdb_marching_tets_prepare(tets.ctypes.data_as(ctypes.c_void_p), self.F, self.Nv, max_batch,
                                                  ctypes.byref(self._h)))
        e, n = ctypes.c_int(), ctypes.c_int()
        L.mdb_marching_tets_info(self._h, ctypes.byref(e), ctypes.byref(n))
        self.n_edges, self.uv_n = e.value, n.value
        self._uvs = None
        self._last_off = None

    def __del__(self):
        try:
            if self._h:
                _native.lib().mdb_marching_tets_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def uvs(self, device):
        if self._uvs is None:
            u = torch.empty(self.uv_n * self.uv_n * 4, 2, device=device, dtype=torch.float32)
            _native.check(_native.lib().mdb_marching_tets_uvs(self._h, _native.ptr(u), _native.current_stream()))
            self._uvs = u
        return self._uvs

    def _extract_raw(self, pos, sdf):
        """Packed outputs of the batch + the [B+1, 3] host table of (verts, faces, valid verts) offsets."""
        L = _native.lib()
        B = sdf.shape[0]
        stride = 0 if pos.dim() == 2 else self.Nv * 3
        counts = (ctypes.c_int * (3 * B))()
        stream = _native.current_stream()
        _native.check(L.mdb_marching_tets_count(self._h, _native.ptr(sdf), B, counts, stream))
        c = np.array(list(counts), dtype=np.int64).reshape(B, 3)
        off = np.concatenate([np.zeros((1, 3), np.int64), np.cumsum(c, 0)], 0)
        dev = sdf.device
        verts = torch.empty(int(off[-1, 0]), 3, device=dev, dtype=torch.float32)
        faces = torch.empty(int(off[-1, 1]), 3, device=dev, dtype=torch.int64)
        uv_idx = torch.empty_like(faces)
        f2t = torch.empty(int(off[-1, 1]), device=dev, dtype=torch.int64)
        vvi = torch.empty(int(off[-1, 2]), device=dev, dtype=torch.int64)
        # outputs are packed back to back in batch order: the library already holds those offsets on the device (NULL)
        _native.check(L.mdb_marching_tets_extract(self._h, _native.ptr(pos), stride, _native.ptr(sdf), B, _native.ptr(verts),
                                                  _native.ptr(faces), _native.ptr(uv_idx), _native.ptr(f2t), _native.ptr(vvi),
                                                  None, None, None, stream))
        return verts, faces, uv_idx, f2t, vvi, off

    def extract(self, pos, sdf):
        """pos [B,Nv,3] or [Nv,3] (shared), sdf [B,Nv] fp32 cuda -> list of per-sample
        (verts, faces, uvs, uv_idx, face_to_valid_tet, valid_vert_idx). `verts` is differentiable with respect to `pos`
        and `sdf` like the reference's (autograd through dmtet.py:125-132); the other outputs are integer tensors."""
        sdf = sdf.float().contiguous()
        pos = pos.float().contiguous()
        B = sdf.shape[0]
        if torch.is_grad_enabled() and (pos.requires_grad or sdf.requires_grad):
            verts, faces, uv_idx, f2t, vvi = _ExtractFn.apply(self, pos, sdf)
            off = self._last_off
        else:
            verts, faces, uv_idx, f2t, vvi, off = self._extract_raw(pos.detach(), sdf.detach())
        uvs = self.uvs(sdf.device)
        out = []
        for b in range(B):
            v0, v1 = off[b, 0], off[b + 1, 0]
            f0, f1 = off[b, 1], off[b + 1, 1]
            w0, w1 = off[b, 2], off[b + 1, 2]
            out.append((verts[v0:v1], faces[f0:f1], uvs, uv_idx[f0:f1], f2t[f0:f1], vvi[w0:w1]))
        return out


class _ExtractFn(torch.autograd.Function):
    """Marching tets as one autograd node: the backward pass is `mdb_marching_tets_backward` (a gather per grid vertex over
    its incident crossing edges), fed by the crossing-edge -> output-row map saved from the forward pass."""

    @staticmethod
    def forward(ctx, mt, pos, sdf):
        verts, faces, uv_idx, f2t, vvi, off = mt._extract_raw(pos, sdf)
        B = sdf.shape[0]
        vid = torch.empty(B, mt.n_edges, device=sdf.device, dtype=torch.int32)
        _native.check(_native.lib().mdb_marching_tets_vertex_ids(mt._h, B, _native.ptr(vid), _native.current_stream()))
        voff = torch.from_numpy(np.ascontiguousarray(off[:-1, 0])).to(sdf.device)
        ctx.mt = mt
        ctx.save_for_backward(pos, sdf, vid, voff)
        ctx.mark_non_differentiable(faces, uv_idx, f2t, vvi)
        mt._last_off = off
        return verts, faces, uv_idx, f2t, vvi

    @staticmethod
    def backward(ctx, gverts, *_unused):
        pos, sdf, vid, voff = ctx.saved_tensors
        mt = ctx.mt
        B = sdf.shape[0]
        need_pos, need_sdf = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        gpos = torch.empty(B, mt.Nv, 3, device=sdf.device, dtype=torch.float32) if need_pos else None
        gsdf = torch.empty(B, mt.Nv, device=sdf.device, dtype=torch.float32) if need_sdf else None
        stride = 0 if pos.dim() == 2 else mt.Nv * 3
        gverts = gverts.float().contiguous()
        _native.check(_native.lib().mdb_marching_tets_backward(mt._h, _native.ptr(pos), stride, _native.ptr(sdf), B, _native.ptr(vid),
                                                               _native.ptr(gverts), _native.ptr(voff), _native.ptr(gpos),
                                                               _native.ptr(gsdf), _native.current_stream()))
        if need_pos and pos.dim() == 2:
            gpos = gpos.sum(0)  # one vertex array shared by the batch
        return None, gpos, gsdf


class DMTet:
    """Call-compatible with the reference class: `DMTet()(pos_nx3, sdf_n, tet_fx4)`."""

    def __init__(self):
        self._cache = {}

    def __call__(self, pos_nx3, sdf_n, tet_fx4):
        key = (tet_fx4.data_ptr(), tuple(tet_fx4.shape), pos_nx3.shape[0])
        if key not in self._cache:
            self._cache = {key: MarchingTets(tet_fx4.detach().cpu().numpy(), pos_nx3.shape[0], 1)}
        mt = self._cache[key]
        return mt.extract(pos_nx3, sdf_n[None])[0]


def grid_to_tet_inputs(grids, coords, vertices, grid_res, mesh_scale=1.0, deform_scale=1.0):
    """Batched eval.py:412-419 + dmtet.py:303: grids [B,4,R,R,R] -> (sdf [B,Nv], pos [B,Nv,3])."""
    x, y, z = coords[:, 0], coords[:, 1], coords[:, 2]
    sdf = torch.sign(grids[:, 0, x, y, z])
    deform = grids[:, 1:, x, y, z].transpose(1, 2).clip(-1.0, 1.0)
    pos = vertices[None] * mesh_scale + 2 / (grid_res * 2) * deform * deform_scale
    return sdf.contiguous(), pos.contiguous()
