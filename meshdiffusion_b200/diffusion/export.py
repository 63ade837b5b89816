"""`--mode=export`: meshes and shaded previews of generated grids, what nvdiffrec/eval.py writes after sampling.

For every grid of every `*.npy` batch in `config.eval.eval_dir` (sorted by name, the set `eval_metrics` reads) this writes
under `<eval_dir>/export/`:

* `mesh/<stem>_<i:06d>.obj` -- the raw marching-tets mesh (no remeshing or smoothing), the text `tools/npy_to_obj.py`
  writes for the same grid;
* `viz/<stem>_<i:06d>_view<v:02d>.png` -- the diffuse preview from every view in `render.views` (default (25,), eval.py's
  `--angle-ind`), `render.res` pixels square (default 1000) with `render.ssaa` x `render.ssaa` supersampling (default 2),
  lit by `render.envmap` (a Radiance `.hdr`) or the built-in procedural sky;
* `index.json` -- one entry per sample (source file, batch index, vertex and face counts, `empty`), the views, res, ssaa,
  light and the seconds spent meshing, rendering and writing files. Under torchrun rank r takes the samples i = r (mod
  world size) of the concatenated list and writes `index_<rank>.json`.

A grid whose mesh is empty still gets its (faceless) `.obj` and background-only images, and is flagged in the index.
The options are read with `.get`, so the stock config tree has no `render` group: `--config.render.views="(0, 25)"` etc.
create it.
"""
import glob
import json
import logging
import os
import time

import numpy as np
import torch

from ..geometry import dmtet, mesh_ops, render
from .evaler import _DEFORM_SCALE, _rank
from .gen_metrics import _generated_batches

_BATCH = 8  # grids meshed and rendered together


def _render_options(config):
    opts = config.get("render", None) or {}
    views = opts.get("views", (render.DEFAULT_VIEW,))
    views = (views,) if isinstance(views, int) else tuple(int(v) for v in views)
    envmap = opts.get("envmap", None) or None
    return views, int(opts.get("res", render.DEFAULT_RES)), int(opts.get("ssaa", render.DEFAULT_SSAA)), envmap


def export(config):
    """Writes the meshes, images and index described in the module docstring; returns the index dictionary."""
    device = config.device
    R = config.data.image_size
    rank, world = _rank(), int(os.environ.get("WORLD_SIZE", "1"))
    views, res, ssaa, envmap = _render_options(config)
    mesh_scale = float(config.eval.get("mesh_scale", 1.1))
    deform_scale = float(config.eval.get("deform_scale", _DEFORM_SCALE.get(R, 3.0)))
    eval_dir = config.eval.eval_dir
    out_dir = os.path.join(eval_dir, "export")
    mesh_dir, viz_dir = os.path.join(out_dir, "mesh"), os.path.join(out_dir, "viz")
    os.makedirs(mesh_dir, exist_ok=True)
    os.makedirs(viz_dir, exist_ok=True)
    light = render.environment_light(envmap)

    # this rank's share of the samples in file order: (source file, stem, index in its batch, grid)
    files = sorted(glob.glob(os.path.join(eval_dir, "*.npy")))
    mine, n = [], 0
    for f, batch in zip(files, _generated_batches(eval_dir)):
        stem = os.path.splitext(os.path.basename(f))[0]
        for b in range(batch.shape[0]):
            if n % world == rank:
                mine.append((f, stem, b, batch[b]))
            n += 1

    verts, tets = dmtet.load_tet_grid(R)
    v = torch.tensor(verts, device=device)
    coords = dmtet.grid_coords_of_tet_vertices(v.cpu()).to(device)
    mt = dmtet.MarchingTets(tets, verts.shape[0], max_batch=_BATCH)
    seconds = {"meshing": 0.0, "render": 0.0, "write": 0.0}
    index = []
    for c0 in range(0, len(mine), _BATCH):
        chunk = mine[c0:c0 + _BATCH]
        torch.cuda.synchronize(device)
        t0 = time.perf_counter()
        grids = torch.from_numpy(np.stack([np.asarray(s[3], np.float32) for s in chunk])).to(device)
        if grids.shape[1:] != (4, R, R, R):
            raise ValueError(f"expected grids [B, 4, {R}, {R}, {R}], got {tuple(grids.shape)}")
        sdf, pos = dmtet.grid_to_tet_inputs(grids, coords, v, R, mesh_scale, deform_scale)
        meshes = [(m[0], m[1]) for m in mt.extract(pos, sdf)]
        normals = [mesh_ops.auto_normals(mv, mf)[0] for mv, mf in meshes]
        torch.cuda.synchronize(device)
        t1 = time.perf_counter()
        images = render.render_meshes(meshes, normals, views, res, ssaa, light).cpu().numpy()
        t2 = time.perf_counter()
        for (src, stem, b, _), (mv, mf), img in zip(chunk, meshes, images):
            name = f"{stem}_{b:06d}"
            mesh_ops.write_obj(mesh_dir, mv, mf, name=name + ".obj")
            pngs = []
            for k, view in enumerate(views):
                pngs.append(f"{name}_view{view:02d}.png")
                render.write_png(os.path.join(viz_dir, pngs[-1]), img[k])
            index.append({"source": src, "batch_index": b, "obj": name + ".obj", "png": pngs, "verts": int(mv.shape[0]),
                          "faces": int(mf.shape[0]), "empty": int(mf.shape[0]) == 0})
        t3 = time.perf_counter()
        seconds["meshing"] += t1 - t0
        seconds["render"] += t2 - t1
        seconds["write"] += t3 - t2
        logging.info("export: rank %d, %d / %d samples", rank, min(c0 + _BATCH, len(mine)), len(mine))
    result = {"resolution": R, "views": list(views), "res": res, "ssaa": ssaa, "light": envmap or "default",
              "mesh_scale": mesh_scale, "deform_scale": deform_scale, "seconds": seconds, "samples": index}
    with open(os.path.join(out_dir, "index.json" if world == 1 else f"index_{rank}.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    return result
