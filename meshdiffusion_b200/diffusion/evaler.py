"""`--mode=uncond_gen` / `--mode=cond_gen` drivers (reference: lib/diffusion/evaler.py:14-60, 134-211), and
`--mode=make_partial`, which makes `cond_gen`'s partial DMTets from dataset grids (nvdiffrec/fit_singleview.py:783-827).

One process per GPU: under torchrun every rank loads the checkpoint, draws `eval.batch_size` samples with its own
seed and writes `<eval_dir>/<rank>.npy` (rank 0 writes `0.npy`, the reference's single-process file name); no
collective is involved. Output files are float32 `[B, 4, R, R, R]`, consumed by nvdiffrec/eval.py:400-417.
"""
import logging
import os

import numpy as np
import torch

from . import sampling, sde_lib
from .models import utils as mutils
from .models.ema import ExponentialMovingAverage
from .utils import restore_checkpoint


def _rank():
    return int(os.environ.get("RANK", "0"))


def load_grid_mask(resolution, device):
    """`./data/grid_mask_<R>.pt` (cwd-relative like evaler.py:38) if present, else derived from the tet grid."""
    path = "./data/grid_mask_{}.pt".format(resolution)
    if os.path.exists(path):
        return torch.load(path, map_location=device).to(device)
    from ..geometry.dmtet import grid_mask_from_tets
    return grid_mask_from_tets(resolution).to(device)


def _setup(config):
    device = config.device
    score_model = mutils.create_model(config)
    from . import losses
    optimizer = losses.get_optimizer(config, score_model.parameters())
    ema = ExponentialMovingAverage(score_model.parameters(), decay=config.model.ema_rate)
    state = dict(optimizer=optimizer, model=score_model, ema=ema, step=0)
    if config.training.sde.lower() != "vpsde":
        raise NotImplementedError(f"SDE {config.training.sde} unknown.")
    sde = sde_lib.VPSDE(beta_min=config.model.beta_min, beta_max=config.model.beta_max, N=config.model.num_scales,
                        device=device)
    return score_model, ema, state, sde


def uncond_gen(config, idx=None):
    idx = _rank() if idx is None else idx
    eval_dir = config.eval.eval_dir
    os.makedirs(eval_dir, exist_ok=True)
    torch.manual_seed(int(config.get("seed", 42)) + idx)
    score_model, ema, state, sde = _setup(config)
    R = config.data.image_size
    grid_mask = load_grid_mask(R, config.device).view(1, R, R, R)
    shape = (config.eval.batch_size, config.data.num_channels, R, R, R)
    sampling_fn = sampling.get_sampling_fn(config, sde, shape, lambda x: x, 1e-3, grid_mask=grid_mask)
    state = restore_checkpoint(config.eval.ckpt_path, state, device=config.device)
    ema.copy_to(score_model.parameters())
    logging.info("rank %d: sampling %d grids of %d^3", idx, shape[0], R)
    samples, _ = sampling_fn(score_model)
    out = os.path.join(eval_dir, f"{idx}.npy")
    np.save(out, samples.cpu().numpy())
    return out


def tet_grid_coords(tet_path, device):
    """Integer grid coordinates int64 [Nv, 3] of the vertices of the tet grid stored at `tet_path` (`eval.tet_path`)."""
    from ..geometry.dmtet import grid_coords_of_tet_vertices
    tet = np.load(tet_path)
    return grid_coords_of_tet_vertices(torch.tensor(tet["vertices"])).to(device)


def partial_grids(partials, coords, R, device):
    """Partial DMTets ({'sdf', 'vis'} per tet vertex) -> the sampler's conditioning: sdf and visibility grids float32
    [n, 1, R, R, R] holding each vertex's value at its voxel `coords` and 0 elsewhere (evaler.py:198-201 of the
    reference)."""
    sdf_grid = torch.zeros(len(partials), 1, R, R, R, device=device)
    vis_grid = torch.zeros(len(partials), 1, R, R, R, device=device)
    for i, d in enumerate(partials):
        sdf_grid[i, 0, coords[:, 0], coords[:, 1], coords[:, 2]] = d["sdf"].to(device).float()
        vis_grid[i, 0, coords[:, 0], coords[:, 1], coords[:, 2]] = d["vis"].to(device).float()
    return sdf_grid, vis_grid


def cond_gen(config, save_fname=None):
    save_fname = str(_rank()) if save_fname is None else save_fname
    eval_dir = config.eval.eval_dir
    os.makedirs(eval_dir, exist_ok=True)
    torch.manual_seed(int(config.get("seed", 42)) + _rank())
    score_model, ema, state, sde = _setup(config)
    device = config.device
    R = config.data.image_size
    grid_mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    shape = (config.eval.batch_size, config.data.num_channels, R, R, R)
    sampling_fn = sampling.get_sampling_fn(config, sde, shape, lambda x: x, 1e-3, grid_mask=grid_mask)
    state = restore_checkpoint(config.eval.ckpt_path, state, device=device)
    ema.copy_to(score_model.parameters())

    partial = torch.load(config.eval.partial_dmtet_path, map_location=device)
    sdf_grid, vis_grid = partial_grids([partial], tet_grid_coords(config.eval.tet_path, device), R, device)
    samples, _ = sampling_fn(score_model, partial=sdf_grid, partial_mask=vis_grid,
                             freeze_iters=config.eval.freeze_iters)
    out = os.path.join(eval_dir, f"{save_fname}.npy")
    np.save(out, samples.cpu().numpy())
    return out


# second_stage_deform of nvdiffrec/configs/res{64,128}.json: the deformation scale the fitted grids were made with
_DEFORM_SCALE = {64: 3.0, 128: 1.5}


def make_partial(config):
    """`--mode=make_partial`: the partial DMTets `cond_gen` takes (`eval.partial_dmtet_path`), made from the shapes
    `config.data.meta_path` / `filter_meta_path` select (the reference set of `eval_metrics`) and the validation views
    `eval.partial_views` (default (0,)) at `eval.partial_res` (default 1000) pixels square.

    Writes `<eval_dir>/partial/<shape:06d>_view<v:02d>.pt` (the reference's `tets/dmtet.pt` layout; `shape` is the index
    in the selected list) and an index of the files it wrote: `index.json` in a single process, `index_<rank>.json` per
    rank under torchrun, where rank r takes the shapes i = r (mod world size). Returns the index entries."""
    import json

    from ..dataset.shapenet_dmtet_dataset import ShapeNetDMTetDataset
    from ..geometry.singleview import PartialDMTets
    from .trainer import _path_or_none
    device = config.device
    R = config.data.image_size
    rank, world = _rank(), int(os.environ.get("WORLD_SIZE", "1"))
    views = config.eval.get("partial_views", (0,))
    views = (views,) if isinstance(views, int) else tuple(views)
    res = int(config.eval.get("partial_res", 1000))
    mesh_scale = float(config.eval.get("mesh_scale", 1.1))
    deform_scale = float(config.eval.get("deform_scale", _DEFORM_SCALE.get(R, 3.0)))
    mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    ds = ShapeNetDMTetDataset(config.data.meta_path, mask.cpu(), filter_meta_path=_path_or_none(config.data.get("filter_meta_path", None)),
                              extension=config.data.get("extension", "pt"), aug=False, normalize_sdf=False)
    if len(ds) == 0:
        raise ValueError(f"the shape list {config.data.meta_path} selects no shapes")
    out_dir = os.path.join(config.eval.eval_dir, "partial")
    os.makedirs(out_dir, exist_ok=True)
    make = PartialDMTets(R, views, res, mesh_scale, deform_scale, device)
    mine = list(range(rank, len(ds), world))
    index = []
    for c0 in range(0, len(mine), make.max_batch):
        ids = mine[c0:c0 + make.max_batch]
        grids = torch.stack([ds[i] for i in ids]).to(device)
        for i, row in zip(ids, make(grids)):
            for k, (d, n_vis_tets) in enumerate(row):
                name = f"{i:06d}_view{views[k]:02d}.pt"
                torch.save(d, os.path.join(out_dir, name))
                index.append({"file": name, "shape": i, "source": ds.fpath_list[i].rstrip(), "view": views[k],
                              "mvp": make.mvps[k].tolist(), "res": res, "visible_tets": n_vis_tets,
                              "visible_verts": int(d["vis"].sum()), "visible_and_rast_verts": int(d["vis_rast"].sum())})
        logging.info("make_partial: rank %d, %d / %d shapes", rank, min(c0 + make.max_batch, len(mine)), len(mine))
    with open(os.path.join(out_dir, "index.json" if world == 1 else f"index_{rank}.json"), "w") as fh:
        json.dump({"resolution": R, "views": list(views), "res": res, "mesh_scale": mesh_scale,
                   "deform_scale": deform_scale, "files": index}, fh, indent=1)
    return index
