"""`--mode=eval_metrics`: how good generated shapes are, as the point-cloud metrics MeshDiffusion-style work reports
(no reference counterpart; the reference ships no evaluation code).

Generated set G: every `*.npy` grid batch in `config.eval.eval_dir` (what `uncond_gen` / `cond_gen` write, from any number
of ranks), in sorted file order then batch order. Reference set R: the grids `config.data.meta_path` lists, filtered by
`config.data.filter_meta_path` (a test-split id list selects the test split). Both go through the same tet grid, marching
tets and placement, so they share one frame; each mesh gets `eval.metric_points` (default 2048) area-weighted surface
points keyed by `config.seed` and its index within its own set. Empty meshes are dropped and counted. On the Chamfer
distance (geometry/pointcloud.py) between those clouds:

* MMD-CD  = mean over Y in R of min over X in G of CD(X, Y);
* COV-CD  = |{argmin over Y in R of CD(X, Y) : X in G}| / |R|;
* 1-NNA-CD = over G and R together, the share of shapes whose nearest other shape is in their own set (0.5 is ideal).

Ties go to the lowest index: in R for the argmin, in the concatenated order [G..., R...] for 1-NNA. With
`eval.metric_emd` set, the same three metrics are also computed over the Earth Mover's distance (`mmd_emd`, `cov_emd`,
`1nna_emd`, ...), each EMD solved to within EMD_EPS of the optimum; `emd_max_gap` is the largest certified gap over the
three EMD matrices. With `eval.metric_lfd` set, the same non-empty shapes also get light-field descriptors
(geometry/lfd.py) and the three metrics are computed over the light field distance (`mmd_lfd`, `cov_lfd`, `1nna_lfd`,
...; integer distances, ties as above); `lfd_empty_views` counts silhouettes with no pixel, `lfd_saturated` is the share
of descriptor coefficient bytes at 255.
"""
import glob
import json
import logging
import os
import time

import numpy as np
import torch

from ..geometry import lfd, pointcloud

# grids per marching-tets launch while the sets are streamed through; only the point clouds stay on the device
_CHUNK = 8
# the EMD entries' tolerance: at most this far above the optimum (sampled shapes span ~1.2 units, EMD values 1e-2..1e-1)
EMD_EPS = 1e-5


def metrics_from_matrices(d_gr, d_gg, d_rr, suffix="cd"):
    """The three metrics from distance matrices G x R, G x G and R x R (numpy float64); keys end in `_<suffix>`."""
    d_gr, d_gg, d_rr = (np.asarray(d, dtype=np.float64) for d in (d_gr, d_gg, d_rr))
    ng, nr = d_gr.shape
    mmd = float(d_gr.min(axis=0).mean())
    cov = float(np.unique(d_gr.argmin(axis=1)).size / nr)  # np.argmin returns the first (lowest) index of a tie
    full = np.block([[d_gg, d_gr], [d_gr.T, d_rr]])
    np.fill_diagonal(full, np.inf)
    label = np.concatenate([np.zeros(ng, bool), np.ones(nr, bool)])
    same = label[full.argmin(axis=1)] == label
    return {f"mmd_{suffix}": mmd, f"cov_{suffix}": cov, f"1nna_{suffix}": float(same.mean()),
            f"1nna_{suffix}_gen": float(same[:ng].mean()), f"1nna_{suffix}_ref": float(same[ng:].mean())}


def generation_metrics(gen_points, ref_points, emd=False):
    """gen_points [nG, N, 3], ref_points [nR, N, 3] (CUDA, fp32) -> metrics dict (+ `matrix_seconds`). emd: also the
    metrics over the EMD (+ `emd_max_gap`, `emd_seconds`)."""
    if gen_points.shape[0] < 1 or ref_points.shape[0] < 1 or gen_points.shape[0] + ref_points.shape[0] < 2:
        raise ValueError("need at least one generated and one reference shape")
    torch.cuda.synchronize(gen_points.device)
    t0 = time.perf_counter()
    d_gr = pointcloud.chamfer_matrix(gen_points, ref_points)
    d_gg = pointcloud.chamfer_matrix(gen_points)
    d_rr = pointcloud.chamfer_matrix(ref_points)
    torch.cuda.synchronize(gen_points.device)
    seconds = time.perf_counter() - t0
    out = metrics_from_matrices(d_gr.cpu().numpy(), d_gg.cpu().numpy(), d_rr.cpu().numpy())
    out["matrix_seconds"] = seconds
    if emd:
        torch.cuda.synchronize(gen_points.device)
        t0 = time.perf_counter()
        (e_gr, g_gr), (e_gg, g_gg), (e_rr, g_rr) = (pointcloud.emd_matrix(gen_points, ref_points, EMD_EPS),
                                                    pointcloud.emd_matrix(gen_points, eps=EMD_EPS),
                                                    pointcloud.emd_matrix(ref_points, eps=EMD_EPS))
        torch.cuda.synchronize(gen_points.device)
        out["emd_seconds"] = time.perf_counter() - t0
        out.update(metrics_from_matrices(e_gr.cpu().numpy(), e_gg.cpu().numpy(), e_rr.cpu().numpy(), suffix="emd"))
        out["emd_max_gap"] = max(float(g.max()) for g in (g_gr, g_gg, g_rr))
    return out


def _clouds(grid_batches, resolution, n_points, seed, device, light_fields=False):
    """Streams [b,4,R,R,R] host batches through marching tets + sampling -> (non-empty clouds [n,N,3], n_empty, lfd) where
    lfd is None, or with light_fields (descriptors uint8 [n,10,10,48] of the same shapes, their empty views, seconds)."""
    kept, descs, n_empty, next_id, empty_views, lfd_seconds = [], [], 0, 0, 0, 0.0
    for batch in grid_batches:
        for c0 in range(0, batch.shape[0], _CHUNK):
            g = torch.as_tensor(batch[c0:c0 + _CHUNK], dtype=torch.float32).to(device)
            verts, faces, vert_off, face_off = pointcloud.grids_to_meshes(g, resolution)
            pts, empty = pointcloud.sample_surface_points(verts, faces, vert_off, face_off, n_points, seed, first_id=next_id)
            next_id += g.shape[0]
            n_empty += int(empty.sum())
            kept.append(pts[~empty])
            if light_fields:
                torch.cuda.synchronize(device)
                t0 = time.perf_counter()
                d, ev = lfd.lfd_descriptors(verts, faces, vert_off, face_off)
                keep = ~empty
                descs.append(d[keep])
                empty_views += int(ev[keep.cpu().numpy()].sum())
                torch.cuda.synchronize(device)
                lfd_seconds += time.perf_counter() - t0
    pts = torch.cat(kept) if kept else torch.empty(0, n_points, 3, device=device)
    if not light_fields:
        return pts, n_empty, None
    shape = (lfd.N_FIELDS, lfd.N_VIEWS, lfd.DESC_BYTES)
    d = torch.cat(descs) if descs else torch.empty((0,) + shape, device=device, dtype=torch.uint8)
    return pts, n_empty, (d, empty_views, lfd_seconds)


def lfd_metrics(gen_desc, ref_desc):
    """gen_desc [nG,10,10,48], ref_desc [nR,10,10,48] (CUDA, uint8) -> the metrics over the light field distance
    (+ `lfd_matrix_seconds`)."""
    torch.cuda.synchronize(gen_desc.device)
    t0 = time.perf_counter()
    d_gr, d_gg, d_rr = lfd.lfd_matrix(gen_desc, ref_desc), lfd.lfd_matrix(gen_desc), lfd.lfd_matrix(ref_desc)
    torch.cuda.synchronize(gen_desc.device)
    out = metrics_from_matrices(d_gr.cpu().numpy(), d_gg.cpu().numpy(), d_rr.cpu().numpy(), suffix="lfd")
    out["lfd_matrix_seconds"] = time.perf_counter() - t0
    return out


def _generated_batches(eval_dir):
    files = sorted(glob.glob(os.path.join(eval_dir, "*.npy")))
    if not files:
        raise FileNotFoundError(f"no *.npy grids in {eval_dir}")
    for f in files:
        x = np.load(f)
        yield x[None] if x.ndim == 4 else x


def _reference_batches(config, resolution, device):
    from ..dataset.shapenet_dmtet_dataset import ShapeNetDMTetDataset
    from .evaler import load_grid_mask
    from .trainer import _path_or_none
    mask = load_grid_mask(resolution, device).view(1, 1, resolution, resolution, resolution)
    ds = ShapeNetDMTetDataset(config.data.meta_path, mask.cpu(), filter_meta_path=_path_or_none(config.data.get("filter_meta_path", None)),
                              extension=config.data.get("extension", "pt"), aug=False, normalize_sdf=False)
    if len(ds) == 0:
        raise ValueError(f"the reference list {config.data.meta_path} selects no shapes")
    for i in range(0, len(ds), _CHUNK):
        yield torch.stack([ds[k] for k in range(i, min(i + _CHUNK, len(ds)))])


def eval_metrics(config):
    """Writes `<eval_dir>/metrics.json` and returns its content."""
    device = config.device
    R = config.data.image_size
    n_points = int(config.eval.get("metric_points", 2048))
    seed = int(config.get("seed", 42))
    eval_dir = config.eval.eval_dir
    torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    light_fields = bool(config.eval.get("metric_lfd", False))
    gen, n_empty_gen, gen_lf = _clouds(_generated_batches(eval_dir), R, n_points, seed, device, light_fields)
    ref, n_empty_ref, ref_lf = _clouds(_reference_batches(config, R, device), R, n_points, seed, device, light_fields)
    torch.cuda.synchronize(device)
    sample_seconds = time.perf_counter() - t0
    if light_fields:
        sample_seconds -= gen_lf[2] + ref_lf[2]
    logging.info("eval_metrics: %d generated (%d empty), %d reference (%d empty) shapes, %d points each",
                 gen.shape[0], n_empty_gen, ref.shape[0], n_empty_ref, n_points)
    emd = bool(config.eval.get("metric_emd", False))
    m = generation_metrics(gen, ref, emd=emd)
    out = {k: m[k] for k in ("mmd_cd", "cov_cd", "1nna_cd", "1nna_cd_gen", "1nna_cd_ref")}
    out.update(n_gen=int(gen.shape[0]), n_ref=int(ref.shape[0]), n_empty_gen=n_empty_gen, n_empty_ref=n_empty_ref,
               n_points=n_points, seed=seed, cd_convention=pointcloud.CD_CONVENTION,
               sample_seconds=sample_seconds, matrix_seconds=m["matrix_seconds"])
    if emd:
        out.update({k: m[k] for k in ("mmd_emd", "cov_emd", "1nna_emd", "1nna_emd_gen", "1nna_emd_ref")})
        out.update(emd_convention=pointcloud.EMD_CONVENTION, emd_eps=EMD_EPS, emd_max_gap=m["emd_max_gap"],
                   emd_seconds=m["emd_seconds"])
    if light_fields:
        ml = lfd_metrics(gen_lf[0], ref_lf[0])
        out.update({k: ml[k] for k in ("mmd_lfd", "cov_lfd", "1nna_lfd", "1nna_lfd_gen", "1nna_lfd_ref")})
        coefs = torch.cat([gen_lf[0], ref_lf[0]])[..., :lfd.COEFS]
        out.update(lfd_convention=lfd.LFD_CONVENTION, lfd_seconds=gen_lf[2] + ref_lf[2] + ml["lfd_matrix_seconds"],
                   lfd_empty_views=gen_lf[1] + ref_lf[1],
                   lfd_saturated=float((coefs == 255).sum()) / max(1, coefs.numel()))
    path = os.path.join(eval_dir, "metrics.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=2)
    logging.info("eval_metrics: %s -> %s", json.dumps({k: out[k] for k in ("mmd_cd", "cov_cd", "1nna_cd")}), path)
    return out
