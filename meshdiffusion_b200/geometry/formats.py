"""On-disk formats either side of the hot path (SURVEY 8f-4), as device-side scatter / unique kernels of torch:

* `partial_dmtet_from_visibility` -- the `tets/dmtet.pt` dictionary that `--mode=cond_gen` consumes
  (`config.eval.partial_dmtet_path`), i.e. the tail of nvdiffrec/fit_singleview.py:783-827: per-vertex visibility from
  the ids of the tetrahedra a view sees. Those ids come from geometry/singleview.py (the library's first-layer depth /
  face-id rasterizer and the reference's visible-tet test in place of the nvdiffrast rasterisation of
  nvdiffrec/lib/render/render.py:335-407); shading and the rest of the renderer are out of scope.
* `tets_to_3dgrid` -- data/tets_to_3dgrid.py:7-15: a fitted DMTet (`sdf` [Nv], `deform` [Nv,3]) scattered onto the
  cubic grid the diffusion model trains on (`grid_*.pt`, [4,R,R,R]).
* the grid mask (data/get_tet_mask.py) lives in geometry/dmtet.py::grid_mask_from_tets.
"""
import torch


def partial_dmtet_from_visibility(tet_indices, n_verts, sdf_sign, deform, visible_tet_id, rast_tet_id=None):
    """fit_singleview.py:798-827. tet_indices [F,4] int; visible_tet_id: ids of the tetrahedra the view sees;
    rast_tet_id: ids of the tetrahedra owning rasterised surface triangles (already mapped through getValidTetIdx).
    Returns {'sdf', 'deform', 'vis' (float 0/1 [Nv]), 'vis_rast' (bool [Nv])} on the CPU, the layout torch.save'd by the
    reference."""
    idx = torch.as_tensor(tet_indices).long()
    dev = idx.device
    F = idx.shape[0]
    visible = torch.zeros(F, dtype=torch.bool, device=dev)
    visible[torch.as_tensor(visible_tet_id, device=dev).long()] = True
    vis_and_rast = visible.clone()
    if rast_tet_id is not None:
        vis_and_rast[torch.as_tensor(rast_tet_id, device=dev).long().unique()] = True
    vis = torch.zeros(n_verts, device=dev)
    vis[idx[visible].unique()] = 1
    vis_rast = vis.clone()
    vis_rast[idx[vis_and_rast].unique()] = 1
    return {"sdf": torch.as_tensor(sdf_sign).detach().cpu(), "deform": torch.as_tensor(deform).detach().cpu(),
            "vis": vis.cpu(), "vis_rast": vis_rast.bool().cpu()}


def tets_to_3dgrid(coords, sdf, deform, grid_size):
    """data/tets_to_3dgrid.py:7-15: grid[0] = sdf, grid[1:] = deform^T at the integer grid coordinate of every tet vertex
    (`coords` [Nv,3] from geometry.dmtet.grid_coords_of_tet_vertices); zero elsewhere."""
    coords = torch.as_tensor(coords).long()
    dev = coords.device
    grid = torch.zeros(4, grid_size, grid_size, grid_size, device=dev)
    x, y, z = coords[:, 0], coords[:, 1], coords[:, 2]
    grid[0, x, y, z] = torch.as_tensor(sdf, device=dev).float().reshape(-1)
    grid[1:, x, y, z] = torch.as_tensor(deform, device=dev).float().transpose(0, 1)
    return grid
