"""`--mode=fit_grids`: DMTet training grids fitted to the triangle meshes of a JSON list of `.obj` files, so that
`--mode=train` can learn a user's own shapes. Geometry only (geometry/fit.py); the reference's grids come from a rendering
fit (nvdiffrec/fit_dmtets.py) whose output layout this keeps.

Options are read with `config.data.get` (the config tree is unchanged): `mesh_meta_path` (the list), `grid_dir` (the
output directory), `fit_views`, `fit_res`, `fit_window`, `fit_iters`, `fit_lr`, `fit_points`, `fit_reg`, `fit_batch`.
"""
import json
import logging
import os
import time

import torch

from ..geometry import fit, mesh_io
from .evaler import _DEFORM_SCALE, _rank
from .trainer import _path_or_none


def fit_grids(config):
    """Writes `<grid_dir>/grid_<i:05d>.pt` ([4, R, R, R]: channel 0 = +-1 on the tet vertices, positive inside; channels
    1-3 = the deformation in [-0.99, 0.99], zero off the surface tets; 0 off the tet grid), `meta.json` (the absolute grid
    paths, what `config.data.meta_path` takes) and `fit_report.json` (per shape: source, counts, Chamfer distances before
    and after the fit, seconds per stage). i is the index in the mesh list. Under torchrun rank r takes the meshes
    i = r (mod world size) and writes `meta_<r>.json` / `fit_report_<r>.json`. Returns the report entries."""
    data = config.data
    meta = _path_or_none(data.get("mesh_meta_path", None))
    if meta is None:
        raise ValueError("--mode=fit_grids needs --config.data.mesh_meta_path, a JSON list of .obj files")
    with open(meta) as fh:
        paths = json.load(fh)
    if not isinstance(paths, list) or not paths:
        raise ValueError(f"the mesh list {meta} is empty: it must be a non-empty JSON list of .obj files")
    grid_dir = _path_or_none(data.get("grid_dir", None))
    if grid_dir is None:
        raise ValueError("--mode=fit_grids needs --config.data.grid_dir, the directory the grids are written to")
    grid_dir = os.path.abspath(grid_dir)
    os.makedirs(grid_dir, exist_ok=True)
    R = int(data.image_size)
    rank, world = _rank(), int(os.environ.get("WORLD_SIZE", "1"))
    settings = {"resolution": R, "views": int(data.get("fit_views", fit.VIEWS)), "res": int(data.get("fit_res", fit.RES)),
                "window": int(data.get("fit_window", fit.WINDOW)), "iters": int(data.get("fit_iters", fit.ITERS)),
                "lr": float(data.get("fit_lr", fit.LR)), "points": int(data.get("fit_points", fit.POINTS)),
                "reg": float(data.get("fit_reg", fit.REG)), "batch": int(data.get("fit_batch", fit.BATCH)),
                "mesh_scale": 1.1, "deform_scale": _DEFORM_SCALE.get(R, 3.0), "seed": int(config.get("seed", 42))}
    fitter = fit.GridFitter(R, settings["views"], settings["res"], settings["window"], settings["iters"], settings["lr"],
                            settings["points"], settings["reg"], settings["batch"], settings["mesh_scale"],
                            settings["deform_scale"], settings["seed"], config.device)
    mine = list(range(rank, len(paths), world))
    grids, report = [], []
    for c0 in range(0, len(mine), fitter.max_batch):
        ids = mine[c0:c0 + fitter.max_batch]
        meshes, load_s = [], []
        for i in ids:
            t = time.perf_counter()
            meshes.append(mesh_io.load_mesh(paths[i]))
            load_s.append(time.perf_counter() - t)
        for i, t_load, r in zip(ids, load_s, fitter([(torch.from_numpy(v), torch.from_numpy(f)) for v, f in meshes], ids)):
            t = time.perf_counter()
            path = os.path.join(grid_dir, f"grid_{i:05d}.pt")
            torch.save(r["grid"], path)
            grids.append(path)
            report.append({"index": i, "source": os.path.abspath(paths[i]), "grid": path, "faces": r["faces"],
                           "inside_verts": r["inside_verts"], "mt_verts": r["mt_verts"], "mt_faces": r["mt_faces"],
                           "chamfer_before": r["chamfer_before"], "chamfer_after": r["chamfer_after"],
                           "surface_distance_before": r["surface_distance_before"],
                           "surface_distance_after": r["surface_distance_after"],
                           "seconds": {"load": t_load, "carve": r["seconds_carve"], "fit": r["seconds_fit"],
                                       "write": time.perf_counter() - t}})
        logging.info("fit_grids: rank %d, %d / %d meshes", rank, min(c0 + fitter.max_batch, len(mine)), len(mine))
    suffix = "" if world == 1 else f"_{rank}"
    with open(os.path.join(grid_dir, f"meta{suffix}.json"), "w") as fh:
        json.dump(grids, fh, indent=1)
    with open(os.path.join(grid_dir, f"fit_report{suffix}.json"), "w") as fh:
        json.dump({**settings, "chamfer_points": fit.REPORT_POINTS, "shapes": report}, fh, indent=1)
    return report
