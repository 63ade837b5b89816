"""`--mode=eval_completion`: shape completion at scale. Every partial DMTet `--mode=make_partial` wrote is completed k times
by conditional sampling, many partials per sampling call, and each completion is scored against its ground-truth shape,
against the other completions of its partial, and against the visible part it was conditioned on. No reference
counterpart: the reference completes one partial per run (`cond_gen`) and ships no evaluation code.

Inputs: the partial index `eval.partial_dir` (default `<eval_dir>/partial`: `index.json`, or the union of the per-rank
`index_<r>.json`, ordered by (shape, view)); the checkpoint `eval.ckpt_path`, `eval.tet_path`, `eval.freeze_iters` and
`sampling.*` as `cond_gen` uses them; `eval.completion_k` (default 10, >= 2) completions per partial; `eval.metric_points`
(default 2048) points per cloud. The ground truth is item `shape` of the shape list `data.meta_path` /
`data.filter_meta_path` selects, as make_partial read it; its file must be the index's `source`.

Sampling: every call has batch `eval.batch_size`, a multiple of k, and holds batch_size / k partials in k consecutive
slots each (per-sample conditioning). The last call is padded with copies of its last partial, whose outputs are dropped,
so one engine size serves the run. `dpm_solver` (ODE or SDE) takes any multiple of k; `pc` only batch_size == k (one
partial per call, `cond_gen`'s exact path: its step-0 initialisation broadcasts the first partial over the batch, the
reference's behaviour); `ddim` is refused. Under torchrun rank r takes the partials p = r (mod world size), with the
global torch RNG seeded `seed + rank` as in `cond_gen`. A completion therefore depends on the seed, its slot in the
batch, `eval.batch_size` and the world size (the native loops key their noise by element index).

Writes `<eval_dir>/completion/<stem>.npy` (float32 [k, 4, R, R, R], the partial file's stem) and `metrics.json`
(`metrics_<rank>.json` per rank under torchrun). `--mode=export` with `eval.eval_dir=<eval_dir>/completion` meshes and
renders the completions.

Metrics (squared distances as in eval_metrics; every mesh placed with the index's mesh_scale and deform_scale):
  * cd_gt[j]: CD(completion j, ground truth), with cd_gt_min and cd_gt_mean (accuracy);
  * tmd: (2 / (k - 1)) sum over i < j of CD(c_i, c_j) (diversity; total mutual difference, Wu et al. 2020);
  * uhd[j]: max over x in the partial cloud of min over y in c_j of |x - y|, Euclidean (fidelity; unidirectional
    Hausdorff distance, same paper), with uhd_mean;
  * p2c[j]: mean over x in the partial cloud of min over y in c_j of |x - y|^2 (the partial's half of the CD);
  * sign_agreement[j]: the share of the partial's visible tet vertices where sign(channel 0 of c_j) is the partial's sdf.
The partial cloud is sampled over the faces of the ground-truth mesh that own at least one pixel of the recorded view (a
partly visible face contributes its whole area). Point clouds are keyed by the partial's position p in the index and
not by batch or rank: ground truth id p, partial cloud id ID_STRIDE + p, completion j id 2 ID_STRIDE + p k + j, so a
partial's metrics depend only on its completions.
"""
import glob
import json
import logging
import math
import os
import time

import numpy as np
import torch

from ..geometry import pointcloud
from . import sampling
from .evaler import _rank, _setup, load_grid_mask, partial_grids, tet_grid_coords
from .utils import restore_checkpoint

# Philox cloud-id ranges: ground truth p, partial cloud ID_STRIDE + p, completion j of partial p 2 ID_STRIDE + p k + j
ID_STRIDE = 1 << 40
PHASES = ("sampling", "meshing", "distances", "writing")
SET_MEANS = ("cd_gt_min", "cd_gt_mean", "tmd", "uhd_mean", "p2c_mean", "sign_agreement_mean")


# ---- arguments ----------------------------------------------------------------------------------------------------
def _int(v):
    return not isinstance(v, bool) and isinstance(v, (int, np.integer))


def completion_k(ev):
    k = ev.get("completion_k", 10)
    if not _int(k) or k < 2:
        raise ValueError(f"eval_completion: eval.completion_k must be an integer >= 2, got {k!r}")
    return int(k)


def partials_per_call(batch_size, k):
    if not _int(batch_size) or batch_size < k or batch_size % k:
        raise ValueError(f"eval_completion: eval.batch_size = {batch_size!r} must be a positive multiple of "
                         f"eval.completion_k = {k}: a sampling call holds batch_size / k partials in k slots each")
    return int(batch_size) // k


def sampler(config, batch_size, k):
    """(method, steps description) or ValueError for a sampler the mode cannot use."""
    method = str(config.sampling.method).lower()
    if method == "dpm_solver":
        return method, {"dpm_steps": int(config.sampling.get("dpm_steps", 25)),
                        "dpm_sde": bool(config.sampling.get("dpm_sde", False))}
    if method == "pc":
        if batch_size != k:
            raise ValueError(f"eval_completion: sampling.method='pc' needs eval.batch_size == eval.completion_k ({k}), "
                             f"got {batch_size}: its step-0 initialisation broadcasts the first partial of a batch over "
                             "every sample (the reference's behaviour, kept for parity), so a call can hold one partial "
                             "only; use 'dpm_solver' to pack several partials per call")
        return method, {"max_iters": config.sampling.get("max_iters", None)}
    if method == "ddim":
        raise ValueError("eval_completion: sampling.method='ddim' is not supported; use 'dpm_solver' or 'pc'")
    raise ValueError(f"eval_completion: unknown sampling.method {method!r}")


def read_index(partial_dir):
    """make_partial's index in `partial_dir` -> (settings dict, entries sorted by (shape, view)). Reads `index.json`, or
    the union of the per-rank `index_<r>.json`. Refuses an empty index, a missing `.pt` file, a partial listed twice and
    rank files made with different settings."""
    single = os.path.join(partial_dir, "index.json")
    paths = [single] if os.path.exists(single) else sorted(glob.glob(os.path.join(partial_dir, "index_*.json")))
    if not paths:
        raise FileNotFoundError(f"eval_completion: no index.json or index_<rank>.json in {partial_dir}; run "
                                "--mode=make_partial first")
    settings, entries = None, []
    for path in paths:
        with open(path) as fh:
            idx = json.load(fh)
        s = {key: idx[key] for key in ("resolution", "res", "mesh_scale", "deform_scale")}
        if settings is not None and s != settings:
            raise ValueError(f"eval_completion: {path} was made with {s}, {paths[0]} with {settings}")
        settings = s
        entries += idx["files"]
    if not entries:
        raise ValueError(f"eval_completion: the partial index in {partial_dir} lists no files")
    entries.sort(key=lambda e: (int(e["shape"]), int(e["view"])))
    seen = set()
    for e in entries:
        if e["file"] in seen:
            raise ValueError(f"eval_completion: {e['file']} is listed twice in {partial_dir}")
        seen.add(e["file"])
        if not os.path.exists(os.path.join(partial_dir, e["file"])):
            raise FileNotFoundError(f"eval_completion: {e['file']} is in the index but not in {partial_dir}")
    return settings, entries


def plan_calls(positions, per_call):
    """Index positions -> [(positions of the call, padded to per_call with its last position, number of real ones)]."""
    calls = []
    for c0 in range(0, len(positions), per_call):
        ids = list(positions[c0:c0 + per_call])
        calls.append((ids + [ids[-1]] * (per_call - len(ids)), len(ids)))
    return calls


def check_sources(entries, fpath_list):
    for e in entries:
        i = int(e["shape"])
        if not 0 <= i < len(fpath_list):
            raise ValueError(f"eval_completion: {e['file']} is shape {i}, but the shape list selects {len(fpath_list)}")
        if fpath_list[i].rstrip() != e["source"]:
            raise ValueError(f"eval_completion: {e['file']} was made from {e['source']}, but item {i} of the shape list "
                             f"is {fpath_list[i].rstrip()}; use the data.meta_path / filter_meta_path make_partial used")


def complete(sampling_fn, model, partials, coords, R, k, method, freeze_iters):
    """One sampling call: partial i conditions slots i k .. i k + k - 1 of the batch (len(partials) k samples) ->
    (samples, network evaluations). `pc` takes a single partial, passed with batch 1 as `cond_gen` passes it."""
    sdf_grid, vis_grid = partial_grids(partials, coords, R, coords.device)
    if method == "pc":
        assert len(partials) == 1
        return sampling_fn(model, partial=sdf_grid, partial_mask=vis_grid, freeze_iters=freeze_iters)
    return sampling_fn(model, partial=sdf_grid.repeat_interleave(k, 0), partial_mask=vis_grid.repeat_interleave(k, 0),
                       freeze_iters=freeze_iters)


# ---- point clouds ------------------------------------------------------------------------------------------------
def extract_meshes(grids, resolution, mesh_scale, deform_scale):
    """grids [B,4,R,R,R] (CUDA) -> packed marching-tets meshes (verts, faces, vert_off [B+1], face_off [B+1]) in the
    frame of grids_to_point_clouds."""
    from ..geometry import dmtet
    v, coords, idx, engines = pointcloud._tet_grid(resolution, grids.device)
    B = grids.shape[0]
    if B not in engines:
        engines[B] = dmtet.MarchingTets(idx, v.shape[0], max_batch=B)
    sdf, pos = dmtet.grid_to_tet_inputs(grids.float(), coords, v, resolution, mesh_scale, deform_scale)
    verts, faces, _, _, _, off = engines[B]._extract_raw(pos, sdf)
    return verts, faces, off[:, 0], off[:, 1]


def mesh(packed, b):
    verts, faces, vo, fo = packed
    return verts[vo[b]:vo[b + 1]], faces[fo[b]:fo[b + 1]]


def sample_meshes(meshes, n_points, seed, first_id):
    """[(verts, faces)] -> (points [n, n_points, 3], empty bool [n]), mesh i keyed by cloud id first_id + i."""
    vo = np.concatenate([[0], np.cumsum([int(v.shape[0]) for v, _ in meshes])])
    fo = np.concatenate([[0], np.cumsum([int(f.shape[0]) for _, f in meshes])])
    verts = torch.cat([v for v, _ in meshes])
    faces = torch.cat([f for _, f in meshes])
    return pointcloud.sample_surface_points(verts, faces, vo, fo, n_points, seed, first_id=first_id)


def visible_faces(verts, faces, mvp, res):
    """Sorted ids of the faces of one mesh that own at least one pixel of the view (`singleview.rasterize`)."""
    from ..geometry import singleview
    if faces.shape[0] == 0:
        return torch.empty(0, dtype=torch.int64, device=faces.device)
    _, face_id = singleview.rasterize([(verts, faces)], torch.as_tensor(mvp, dtype=torch.float32).reshape(1, 4, 4), res)
    ids = face_id.reshape(-1)
    return torch.unique(ids[ids >= 0]).long()


def sign_agreement(grids, sdf, vis, coords):
    """grids [k,4,R,R,R]; sdf, vis [Nv] of the partial -> share of the vis vertices where sign(channel 0) == sdf, [k]."""
    m = vis.to(grids.device) > 0
    n = int(m.sum())
    if n == 0:
        return [float("nan")] * grids.shape[0]
    s = torch.sign(grids[:, 0, coords[:, 0], coords[:, 1], coords[:, 2]].float())[:, m]
    return ((s == sdf.to(grids.device).float()[m]).sum(1).double() / n).tolist()


# ---- metrics -----------------------------------------------------------------------------------------------------
def group_pairs(n, k, valid_partial, comp_ok):
    """Cloud layout [gt 0..n) | partial n..2n) | completions 2n + i k + j] -> the listed (a, b) pairs and, per pair, its
    role (partial i, kind, j or (j, l)). Pairs touching an empty completion or a partial without visible faces are left
    out."""
    pairs, roles = [], []
    for i in range(n):
        if not valid_partial[i]:
            continue
        comp = [2 * n + i * k + j for j in range(k)]
        for j in range(k):
            if comp_ok[i * k + j]:
                pairs.append((comp[j], i)); roles.append((i, "gt", j))
        for j in range(k):
            for l in range(j + 1, k):
                if comp_ok[i * k + j] and comp_ok[i * k + l]:
                    pairs.append((comp[j], comp[l])); roles.append((i, "tmd", (j, l)))
        for j in range(k):
            if comp_ok[i * k + j]:
                pairs.append((n + i, comp[j])); roles.append((i, "partial", j))
    return pairs, roles


def _mean(values):
    v = [x for x in values if not math.isnan(x)]
    return float(np.mean(v)) if v else float("nan")


def group_metrics(gt, part, comp, comp_empty, valid_partial, k):
    """One `mdb_chamfer_pairs` launch for a group of n partials. gt, part [n, N, 3] and comp [n k, N, 3] (CUDA clouds);
    comp_empty bool [n k]; valid_partial bool [n] (the partial's view shows a face). Returns n dicts of the distance
    metrics (None for an invalid partial); NaN for an empty completion, whose partial's means skip it."""
    n = gt.shape[0]
    comp_ok = [not bool(e) for e in comp_empty]
    pairs, roles = group_pairs(n, k, valid_partial, comp_ok)
    cd, mean_ab, max_ab = pointcloud.chamfer_pairs(torch.cat([gt, part, comp]), pairs)
    cd, mean_ab, max_ab = cd.cpu().tolist(), mean_ab.cpu().tolist(), max_ab.cpu().tolist()
    nan = float("nan")
    rows = [dict(cd_gt=[nan] * k, uhd=[nan] * k, p2c=[nan] * k, tmd_sum=0.0) if valid_partial[i] else None
            for i in range(n)]
    for (i, kind, j), c, m, x in zip(roles, cd, mean_ab, max_ab):
        r = rows[i]
        if kind == "gt":
            r["cd_gt"][j] = c
        elif kind == "tmd":
            r["tmd_sum"] += c
        else:
            r["uhd"][j] = math.sqrt(x)
            r["p2c"][j] = m
    for i, r in enumerate(rows):
        if r is None:
            continue
        n_ok = sum(comp_ok[i * k:(i + 1) * k])
        tmd_sum = r.pop("tmd_sum")
        ok = [v for v in r["cd_gt"] if not math.isnan(v)]
        r.update(empty=k - n_ok, cd_gt_min=min(ok) if ok else nan, cd_gt_mean=_mean(r["cd_gt"]),
                 tmd=2.0 * tmd_sum / (n_ok - 1) if n_ok >= 2 else nan, uhd_mean=_mean(r["uhd"]), p2c_mean=_mean(r["p2c"]))
    return rows


def _json_safe(x):
    if isinstance(x, float):
        return None if math.isnan(x) else x
    if isinstance(x, dict):
        return {key: _json_safe(v) for key, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_json_safe(v) for v in x]
    return x


def _sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize(device)


# ---- the mode ----------------------------------------------------------------------------------------------------
def eval_completion(config):
    """Writes this rank's completions and its metrics file; returns the report. Every argument is checked (ValueError,
    FileNotFoundError) before a network is built."""
    from ..dataset.shapenet_dmtet_dataset import ShapeNetDMTetDataset
    from .trainer import _path_or_none
    ev = config.eval
    k = completion_k(ev)
    B = ev.batch_size
    per_call = partials_per_call(B, k)
    method, steps = sampler(config, B, k)
    device = config.device
    R, C = config.data.image_size, config.data.num_channels
    seed = int(config.get("seed", 42))
    rank, world = _rank(), int(os.environ.get("WORLD_SIZE", "1"))
    n_points = int(ev.get("metric_points", 2048))
    partial_dir = ev.get("partial_dir", None) or os.path.join(ev.eval_dir, "partial")
    settings, entries = read_index(partial_dir)
    if not os.path.exists(str(ev.tet_path)):
        raise FileNotFoundError(f"eval_completion: eval.tet_path {ev.tet_path!r} does not exist")
    if settings["resolution"] != R:
        raise ValueError(f"eval_completion: the partials are for R = {settings['resolution']}, the config for R = {R}")
    mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    ds = ShapeNetDMTetDataset(config.data.meta_path, mask.cpu(), filter_meta_path=_path_or_none(config.data.get("filter_meta_path", None)),
                              extension=config.data.get("extension", "pt"), aug=False, normalize_sdf=False)
    check_sources(entries, ds.fpath_list)
    mesh_scale, deform_scale = float(settings["mesh_scale"]), float(settings["deform_scale"])

    out_dir = os.path.join(ev.eval_dir, "completion")
    os.makedirs(out_dir, exist_ok=True)
    torch.manual_seed(seed + rank)  # as cond_gen seeds it
    score_model, ema, state, sde = _setup(config)
    sampling_fn = sampling.get_sampling_fn(config, sde, (B, C, R, R, R), lambda x: x, 1e-3, grid_mask=mask)
    state = restore_checkpoint(ev.ckpt_path, state, device=device)
    ema.copy_to(score_model.parameters())
    coords = tet_grid_coords(ev.tet_path, device)

    secs = dict.fromkeys(PHASES, 0.0)
    rows, nfe = [], None
    for ids, n_real in plan_calls(list(range(rank, len(entries), world)), per_call):
        t0 = time.perf_counter()
        partials = [torch.load(os.path.join(partial_dir, entries[p]["file"]), map_location=device) for p in ids]
        samples, nfe = complete(sampling_fn, score_model, partials, coords, R, k, method, ev.freeze_iters)
        samples = samples[:n_real * k].float()
        _sync(device)
        t1 = time.perf_counter()
        real = ids[:n_real]
        gt_grids = torch.stack([ds[int(entries[p]["shape"])] for p in real]).to(device)
        gt_mesh = extract_meshes(gt_grids, R, mesh_scale, deform_scale)
        comp_mesh = extract_meshes(samples, R, mesh_scale, deform_scale)
        gt_pts, vis_faces, part_pts, comp_pts, comp_empty = [], [], [], [], []
        for i, p in enumerate(real):
            v, f = mesh(gt_mesh, i)
            gt_pts.append(sample_meshes([(v, f)], n_points, seed, p)[0])
            faces_seen = visible_faces(v, f, entries[p]["mvp"], int(entries[p]["res"]))
            vis_faces.append(int(faces_seen.numel()))
            part_pts.append(sample_meshes([(v, f[faces_seen])], n_points, seed, ID_STRIDE + p)[0])
            pts, empty = sample_meshes([mesh(comp_mesh, i * k + j) for j in range(k)], n_points, seed, 2 * ID_STRIDE + p * k)
            comp_pts.append(pts)
            comp_empty += empty.cpu().tolist()
        _sync(device)
        t2 = time.perf_counter()
        metrics = group_metrics(torch.cat(gt_pts), torch.cat(part_pts), torch.cat(comp_pts), comp_empty,
                                [nv > 0 for nv in vis_faces], k)
        agree = [sign_agreement(samples[i * k:(i + 1) * k], partials[i]["sdf"], partials[i]["vis"], coords)
                 for i in range(n_real)]
        t3 = time.perf_counter()
        host = samples.cpu().numpy()
        for i, p in enumerate(real):
            e = entries[p]
            np.save(os.path.join(out_dir, os.path.splitext(e["file"])[0] + ".npy"), host[i * k:(i + 1) * k])
            row = {"file": e["file"], "index": p, "shape": int(e["shape"]), "view": int(e["view"]), "source": e["source"],
                   "visible_faces": vis_faces[i]}
            if metrics[i] is not None:
                row.update(metrics[i], sign_agreement=agree[i], sign_agreement_mean=_mean(agree[i]))
            rows.append(row)
        t4 = time.perf_counter()
        for key, dt in zip(PHASES, (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
            secs[key] += dt
        logging.info("eval_completion: rank %d, %d / %d partials", rank, len(rows), len(range(rank, len(entries), world)))
    scored = [r for r in rows if r["visible_faces"] > 0]
    means = {key: _mean([r[key] for r in scored]) for key in SET_MEANS}
    means.update(partials=len(rows), scored=len(scored), empty_completions=sum(r.get("empty", 0) for r in scored))
    report = {"settings": {"k": k, "sampler": method, **steps, "nfe": None if nfe is None else int(nfe),
                           "freeze_iters": int(ev.freeze_iters), "metric_points": n_points, "batch_size": int(B),
                           "seed": seed, "world_size": world, "rank": rank, "resolution": R, "mesh_scale": mesh_scale,
                           "deform_scale": deform_scale, "compute_dtype": str(config.model.get("compute_dtype", "fp32")),
                           "cd_convention": pointcloud.CD_CONVENTION, "partial_dir": partial_dir},
              "means": means, "seconds": secs, "partials": rows}
    path = os.path.join(out_dir, "metrics.json" if world == 1 else f"metrics_{rank}.json")
    with open(path, "w") as fh:
        json.dump(_json_safe(report), fh, indent=1)
    logging.info("eval_completion: %s -> %s", json.dumps(_json_safe(means)), path)
    return report
