"""`--mode=edit`: regenerate boxed regions of DMTet grids and keep the rest. No reference counterpart.

Every grid-mask voxel whose tet vertex lies in one of the boxes is regenerated; every other grid-mask voxel is kept on
all four channels (sign and deformation). Sampling is RePaint resampling (Lugmayr et al., CVPR 2022) on the
DPM-Solver++(2M) label grid (`sampling.get_repaint_sampler`): the kept region is replaced on every entry, and every block
of `eval.edit_jump` solver steps is redone `eval.edit_resample` times (1 = plain replacement), so the regenerated part is
made to agree with the kept part at every noise level. The last entry writes the kept region exactly.

Inputs:
  * `eval.edit_source`: a `.npy` of float32 [S, 4, R, R, R] (what `uncond_gen` writes) or a `.pt` holding one grid
    [4, R, R, R] (what `fit_grids` writes);
  * `eval.edit_boxes`: one box [x0, y0, z0, x1, y1, z1] or a list of them, in the frame of `--mode=export`'s meshes:
    undeformed tet vertex positions times `eval.mesh_scale` (default 1.1); bounds inclusive;
  * `eval.edit_k` (default 4) variants per source, `eval.edit_jump` (default 5), `eval.edit_resample` (default 3);
  * `sampling.dpm_steps`, `sampling.dpm_sde`, `sampling.native_rng`, `eval.ckpt_path`, `eval.batch_size`.

Every call has batch `eval.batch_size`, a multiple of k, and holds batch_size / k sources in k consecutive slots each;
the last call is padded with copies of its last source, whose outputs are dropped. Under torchrun rank r takes the
sources s = r (mod world size), with the global torch RNG seeded `seed + rank` as in `cond_gen`.

Writes `<eval_dir>/edit/<stem>_<s:04d>.npy` (float32 [k, 4, R, R, R]; `stem` = the source file's) and `edit.json`
(`edit_<rank>.json` under torchrun): the settings, the network evaluations per call and, per source, the regenerated
vertex count, the TMD over its variants ((2 / (k - 1)) sum over i < j of CD(v_i, v_j)) and, per variant,
`known_max_abs_diff` (0 by construction), the share of regenerated vertices whose sign differs from the source, and the
Chamfer distance to the source mesh (`eval.metric_points`, default 2048, points per cloud; meshes placed with
`eval.mesh_scale` and `eval.deform_scale` as `eval_completion` places them). `--mode=export` with
`eval.eval_dir=<eval_dir>/edit` meshes and renders the variants.
"""
import json
import logging
import os
import time

import numpy as np
import torch

from ..geometry import dmtet, pointcloud
from . import sampling
from .completion import _int, _json_safe, _mean, _sync, extract_meshes, mesh, plan_calls, sample_meshes
from .evaler import _DEFORM_SCALE, _rank, _setup, load_grid_mask
from .utils import restore_checkpoint

ID_STRIDE = 1 << 40  # Philox cloud ids: source s, variant j of source s ID_STRIDE + s k + j


# ---- arguments ----------------------------------------------------------------------------------------------------
def edit_settings(ev):
    """(k, jump, resample) from the eval group, or ValueError."""
    out = []
    for key, default, low in (("edit_k", 4, 1), ("edit_jump", 5, 1), ("edit_resample", 3, 1)):
        v = ev.get(key, default)
        if not _int(v) or v < low:
            raise ValueError(f"edit: eval.{key} must be an integer >= {low}, got {v!r}")
        out.append(int(v))
    return tuple(out)


def sources_per_call(batch_size, k):
    if not _int(batch_size) or batch_size < k or batch_size % k:
        raise ValueError(f"edit: eval.batch_size = {batch_size!r} must be a positive multiple of eval.edit_k = {k}: a "
                         "sampling call holds batch_size / k sources in k slots each")
    return int(batch_size) // k


def parse_boxes(boxes):
    """eval.edit_boxes -> float64 [n, 6] (x0, y0, z0, x1, y1, z1), or ValueError for no box, a malformed one or one with
    x1 < x0 (likewise y, z)."""
    if boxes is None:
        raise ValueError("edit: eval.edit_boxes is required: one or more [x0, y0, z0, x1, y1, z1] boxes")
    try:
        b = np.asarray(boxes, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError(f"edit: eval.edit_boxes must be numbers [x0, y0, z0, x1, y1, z1], got {boxes!r}") from None
    if b.ndim == 1:
        b = b[None]
    if b.ndim != 2 or b.shape[0] == 0 or b.shape[1] != 6:
        raise ValueError(f"edit: eval.edit_boxes must be one or more [x0, y0, z0, x1, y1, z1] boxes, got shape {b.shape}")
    if not np.isfinite(b).all():
        raise ValueError("edit: eval.edit_boxes must be finite")
    for i, box in enumerate(b):
        if np.any(box[3:] < box[:3]):
            raise ValueError(f"edit: box {i} {box.tolist()} is empty (x1 < x0, y1 < y0 or z1 < z0)")
    return b


def region(boxes, vertices, coords, R, mesh_scale):
    """Boxes [n, 6] in the mesh frame, tet vertices [Nv, 3] (undeformed), their voxels [Nv, 3] -> (regenerated vertices
    bool [Nv], regenerated voxels float32 [R, R, R]). A vertex is regenerated when vertex * mesh_scale lies in any box;
    a box that selects no vertex is an error."""
    p = np.asarray(vertices, dtype=np.float64) * mesh_scale
    sel = np.zeros(p.shape[0], dtype=bool)
    for i, box in enumerate(boxes):
        inside = np.all((p >= box[:3]) & (p <= box[3:]), axis=1)
        if not inside.any():
            raise ValueError(f"edit: box {i} {box.tolist()} contains no tet vertex (vertices * mesh_scale span "
                             f"{p.min(0).round(4).tolist()} .. {p.max(0).round(4).tolist()})")
        sel |= inside
    c = torch.as_tensor(coords).cpu()
    vox = torch.zeros(R, R, R)
    s = torch.from_numpy(sel)
    vox[c[s, 0], c[s, 1], c[s, 2]] = 1.0
    return sel, vox


def load_sources(path, R, C):
    """eval.edit_source -> float32 [S, C, R, R, R] (CPU), or ValueError / FileNotFoundError."""
    if path is None or not os.path.exists(str(path)):
        raise FileNotFoundError(f"edit: eval.edit_source {path!r} does not exist")
    path = str(path)
    if path.endswith(".npy"):
        x = torch.from_numpy(np.load(path).astype(np.float32, copy=False))
        want = f"[S, {C}, {R}, {R}, {R}]"
    elif path.endswith(".pt"):
        x = torch.load(path, map_location="cpu")
        if not torch.is_tensor(x):
            raise ValueError(f"edit: {path} must hold one grid tensor [{C}, {R}, {R}, {R}], got {type(x).__name__}")
        x = x.float()[None] if x.dim() == 4 else x.float()
        want = f"[{C}, {R}, {R}, {R}]"
    else:
        raise ValueError(f"edit: eval.edit_source must be a .npy or .pt file, got {path}")
    if x.dim() != 5 or tuple(x.shape[1:]) != (C, R, R, R) or x.shape[0] == 0:
        raise ValueError(f"edit: {path} has shape {tuple(x.shape)}, expected {want} (data.image_size = {R})")
    if not torch.isfinite(x).all():
        raise ValueError(f"edit: {path} holds non-finite values")
    return x.contiguous()


def sampler_settings(config):
    method = str(config.sampling.method).lower()
    if method == "distilled":
        raise ValueError("edit: sampling.method='distilled' is not supported: RePaint resampling runs on the dpm_solver "
                         "grid and jumps back up it, which a distilled student was not trained for; edit with the "
                         "teacher's checkpoint and sampling.method='dpm_solver'")
    if method != "dpm_solver":
        logging.info("edit: sampling.method=%r is not used; editing samples with RePaint on the dpm_solver grid", method)
    return {"dpm_steps": int(config.sampling.get("dpm_steps", 25)), "dpm_sde": bool(config.sampling.get("dpm_sde", False)),
            "native_rng": bool(config.sampling.get("native_rng", False))}


# ---- metrics -----------------------------------------------------------------------------------------------------
def group_metrics(src_pts, src_empty, var_pts, var_empty, k):
    """One `mdb_chamfer_pairs` launch for n sources: src_pts [n, N, 3], var_pts [n k, N, 3] -> per source (cd [k], tmd).
    Pairs with an empty mesh are left out and give NaN."""
    n = src_pts.shape[0]
    pairs, roles = [], []
    for i in range(n):
        ok = [not var_empty[i * k + j] for j in range(k)]
        for j in range(k):
            if ok[j] and not src_empty[i]:
                pairs.append((n + i * k + j, i)); roles.append((i, j, None))
            for l in range(j + 1, k):
                if ok[j] and ok[l]:
                    pairs.append((n + i * k + j, n + i * k + l)); roles.append((i, j, l))
    cd = pointcloud.chamfer_pairs(torch.cat([src_pts, var_pts]), pairs)[0].cpu().tolist() if pairs else []
    out = [dict(cd=[float("nan")] * k, tmd_sum=0.0) for _ in range(n)]
    for (i, j, l), c in zip(roles, cd):
        if l is None:
            out[i]["cd"][j] = c
        else:
            out[i]["tmd_sum"] += c
    res = []
    for i in range(n):
        n_ok = sum(not var_empty[i * k + j] for j in range(k))
        res.append((out[i]["cd"], 2.0 * out[i]["tmd_sum"] / (n_ok - 1) if n_ok >= 2 else float("nan")))
    return res


# ---- the mode ----------------------------------------------------------------------------------------------------
def edit(config):
    """Writes this rank's variants and its report; returns the report. Every argument is checked (ValueError,
    FileNotFoundError) before a network is built."""
    from .classes import refuse_conditional
    refuse_conditional(config, "edit")
    ev = config.eval
    k, jump, resample = edit_settings(ev)
    B = ev.batch_size
    per_call = sources_per_call(B, k)
    steps = sampler_settings(config)
    device = config.device
    R, C = config.data.image_size, config.data.num_channels
    if C != 4:
        raise ValueError(f"edit: DMTet grids have 4 channels, the config {C}")
    seed = int(config.get("seed", 42))
    rank, world = _rank(), int(os.environ.get("WORLD_SIZE", "1"))
    n_points = int(ev.get("metric_points", 2048))
    mesh_scale = float(ev.get("mesh_scale", 1.1))
    deform_scale = float(ev.get("deform_scale", _DEFORM_SCALE.get(R, 3.0)))
    boxes = parse_boxes(ev.get("edit_boxes", None))
    src_path = ev.get("edit_source", None)
    sources = load_sources(src_path, R, C)
    verts, _ = dmtet.load_tet_grid(R)
    coords = dmtet.grid_coords_of_tet_vertices(torch.from_numpy(verts))
    regen_v, regen_vox = region(boxes, verts, coords, R, mesh_scale)
    mask = load_grid_mask(R, device).view(1, 1, R, R, R).float()
    regen_vox = regen_vox.to(device)
    keep = (mask[0, 0] * (1.0 - regen_vox)).reshape(1, R, R, R).contiguous()
    n_regen = int(regen_v.sum())

    out_dir = os.path.join(ev.eval_dir, "edit")
    os.makedirs(out_dir, exist_ok=True)
    stem = os.path.splitext(os.path.basename(str(src_path)))[0]
    torch.manual_seed(seed + rank)  # as cond_gen seeds it
    score_model, ema, state, sde = _setup(config)
    sampling_fn = sampling.get_repaint_sampler(sde, (B, C, R, R, R), lambda x: x, n_steps=steps["dpm_steps"], jump=jump,
                                               resample=resample, stochastic=steps["dpm_sde"], device=device,
                                               grid_mask=mask, native_rng=steps["native_rng"], seed=seed)
    state = restore_checkpoint(ev.ckpt_path, state, device=device)
    ema.copy_to(score_model.parameters())
    cdev = coords.to(device)
    rv = torch.from_numpy(regen_v).to(device)
    kept = keep[0] > 0

    secs = {"sampling": 0.0, "metrics": 0.0, "writing": 0.0}
    rows, nfe = [], None
    for ids, n_real in plan_calls(list(range(rank, sources.shape[0], world)), per_call):
        t0 = time.perf_counter()
        src = (sources[ids].to(device) * mask).contiguous()
        samples, nfe = sampling_fn(score_model, src.repeat_interleave(k, 0), keep, range(C))
        samples = samples[:n_real * k].float()
        _sync(device)
        t1 = time.perf_counter()
        real = ids[:n_real]
        src = src[:n_real]
        var = samples.view(n_real, k, C, R, R, R)
        diff = (var - src[:, None]).abs()[..., kept].amax(dim=(2, 3)).cpu().tolist()  # [n, k]
        s_src = torch.sign(src[:, 0, cdev[:, 0], cdev[:, 1], cdev[:, 2]][:, rv])
        s_var = torch.sign(samples[:, 0, cdev[:, 0], cdev[:, 1], cdev[:, 2]][:, rv]).view(n_real, k, -1)
        flipped = ((s_var != s_src[:, None]).sum(-1).double() / max(n_regen, 1)).cpu().tolist()
        src_mesh = extract_meshes(src, R, mesh_scale, deform_scale)
        var_mesh = extract_meshes(samples, R, mesh_scale, deform_scale)
        src_pts, src_empty, var_pts, var_empty = [], [], [], []
        for i, s in enumerate(real):  # clouds keyed by source index, so a source's metrics do not depend on its call
            pts, empty = sample_meshes([mesh(src_mesh, i)], n_points, seed, s)
            src_pts.append(pts)
            src_empty += empty.cpu().tolist()
            pts, empty = sample_meshes([mesh(var_mesh, i * k + j) for j in range(k)], n_points, seed, ID_STRIDE + s * k)
            var_pts.append(pts)
            var_empty += empty.cpu().tolist()
        metrics = group_metrics(torch.cat(src_pts), src_empty, torch.cat(var_pts), var_empty, k)
        t2 = time.perf_counter()
        host = samples.cpu().numpy()
        for i, s in enumerate(real):
            np.save(os.path.join(out_dir, f"{stem}_{s:04d}.npy"), host[i * k:(i + 1) * k])
            cd, tmd = metrics[i]
            rows.append({"source_index": s, "file": f"{stem}_{s:04d}.npy", "regenerated_vertices": n_regen, "tmd": tmd,
                         "source_empty": src_empty[i],
                         "variants": [{"known_max_abs_diff": diff[i][j], "regenerated_vertices": n_regen,
                                       "sign_flip_share": flipped[i][j], "chamfer_to_source": cd[j],
                                       "empty": bool(var_empty[i * k + j])} for j in range(k)]})
        t3 = time.perf_counter()
        for key, dt in zip(secs, (t1 - t0, t2 - t1, t3 - t2)):
            secs[key] += dt
        logging.info("edit: rank %d, %d / %d sources", rank, len(rows), len(range(rank, sources.shape[0], world)))
    report = {"settings": {"source": str(src_path), "boxes": boxes.tolist(), "k": k, "jump": jump, "resample": resample,
                           **steps, "nfe": None if nfe is None else int(nfe), "batch_size": int(B), "seed": seed,
                           "world_size": world, "rank": rank, "resolution": R, "mesh_scale": mesh_scale,
                           "deform_scale": deform_scale, "metric_points": n_points,
                           "regenerated_vertices": n_regen, "kept_voxels": int(kept.sum()),
                           "compute_dtype": str(config.model.get("compute_dtype", "fp32")),
                           "cd_convention": pointcloud.CD_CONVENTION},
              "means": {"tmd": _mean([r["tmd"] for r in rows]),
                        "chamfer_to_source": _mean([v["chamfer_to_source"] for r in rows for v in r["variants"]]),
                        "sign_flip_share": _mean([v["sign_flip_share"] for r in rows for v in r["variants"]]),
                        "known_max_abs_diff": max([v["known_max_abs_diff"] for r in rows for v in r["variants"]],
                                                  default=0.0)},
              "seconds": secs, "sources": rows}
    path = os.path.join(out_dir, "edit.json" if world == 1 else f"edit_{rank}.json")
    with open(path, "w") as fh:
        json.dump(_json_safe(report), fh, indent=1)
    logging.info("edit: %s -> %s", json.dumps(_json_safe(report["means"])), path)
    return report
