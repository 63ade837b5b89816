"""Benchmark of partial DMTets from depth maps (geometry/depth_partial.py, csrc/depth_partial.cu).

1. Kernels: `mdb_depth_unproject` on a 1000 x 1000 depth map and `mdb_depth_closest_points` for the marching-tet
   vertices of a sphere grid against that map, at R = 64 and R = 128, timed with CUDA events over 20 launches after a
   warm-up.
2. A batch of 8 observations end to end (`DepthPartials`), split into unproject (with the point samples), carve, fit and
   visibility + write (the `dmtet.pt` dictionaries saved to a temporary directory).
3. `--mode=make_partial` from the grid against from depth (`eval.partial_from`), on `--shapes` synthetic shapes x 8 views
   at 1000 x 1000.
4. `--mode=eval_completion` on both partial sets of the first `--completion-shapes` shapes, with synthetic weights (an
   absent checkpoint): the numbers show cost and plumbing only, not completion quality.

Prints the card's name, power limit and SM clock with the numbers, as one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

VIEWS = (0, 6, 12, 18, 25, 31, 37, 43)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit, sm, sm_max = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": limit, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown", "sm_clock": "unknown"}


def _events(fn, n=20):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1000 / n


def _sphere_observations(R, n, res=1000):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry.depth_partial import parse_camera, render_depth
    from meshdiffusion_b200.geometry.singleview import PartialDMTets
    grids = synthetic_grids(n, R, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(1))
    make = PartialDMTets(R, (0,), res, 1.1, 3.0 if R == 64 else 1.5, "cuda")
    depth = render_depth(make, grids)[:, 0].cpu().numpy()
    return depth, [parse_camera({"view": 0})] * n


def _kernels(R):
    from meshdiffusion_b200.geometry import dmtet
    from meshdiffusion_b200.geometry.depth_partial import DepthPartials, depth_closest_points, unproject
    depth, cams = _sphere_observations(R, 1)
    fit = DepthPartials(R, deform_scale=3.0 if R == 64 else 1.5, max_batch=1)
    d = torch.from_numpy(depth).cuda()
    proj, inv_mv, mvp = (cams[0][k].reshape(1, 16).cuda() for k in ("proj", "inv_mv", "mvp"))
    z, valid, pts, edge = unproject(d, proj, inv_mv, fit.cell)
    sdf = (fit.grid_points.norm(dim=1) < 0.33).float()[None] * 2 - 1
    q, _, _, _, _, off = fit.mt._extract_raw(fit._pos(torch.zeros(1, fit.n_verts, 3, device="cuda")), sdf.contiguous())
    t_u = _events(lambda: unproject(d, proj, inv_mv, fit.cell))
    t_c = _events(lambda: depth_closest_points(q, off[:, 0], mvp, proj, fit.cell, pts, valid, edge))
    found = depth_closest_points(q, off[:, 0], mvp, proj, fit.cell, pts, valid, edge)[2]
    card = _card()
    return {"R": R, "res": 1000, "unproject_s": t_u, "unproject_gb_per_s": 1000 * 1000 * (4 + 4 + 4 + 12 + 1) / t_u / 1e9,
            "closest_queries": int(q.shape[0]), "closest_found": int(found.sum()), "closest_s": t_c,
            "closest_queries_per_s": q.shape[0] / t_c, "sm_clock": card["sm_clock"]}


def _batch(R=64, n=8):
    from meshdiffusion_b200.geometry.depth_partial import DepthPartials
    depth, cams = _sphere_observations(R, n)
    fit = DepthPartials(R, max_batch=n)
    fit(depth[:1], cams[:1])  # warm-up
    torch.cuda.synchronize()
    t = time.perf_counter()
    res = fit(list(depth), cams)
    with tempfile.TemporaryDirectory() as tmp:
        for i, (d, _) in enumerate(res):
            torch.save(d, os.path.join(tmp, f"{i}.pt"))
    wall = time.perf_counter() - t
    rep = [r for _, r in res]
    stages = {k: sum(r[k] for r in rep) for k in ("seconds_unproject", "seconds_carve", "seconds_fit", "seconds_visibility")}
    return {"R": R, "observations": n, "wall_s": wall, **stages,
            "seconds_write": wall - sum(stages.values()),
            "distance_before": [r["distance_before"] for r in rep], "distance_after": [r["distance_after"] for r in rep]}


def _make_partial(tmp, shapes, completion_shapes):
    from configs import res64
    from meshdiffusion_b200.diffusion import completion, evaler
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet
    grids = synthetic_grids(shapes, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(3)).cpu()
    paths = []
    for i in range(shapes):
        p = os.path.join(tmp, f"grid_{i:04d}.pt")
        torch.save(grids[i].clone(), p)
        paths.append(p)
    metas = {}
    for name, sel in (("all", paths), ("subset", paths[:completion_shapes])):
        metas[name] = os.path.join(tmp, f"meta_{name}.json")
        with open(metas[name], "w") as fh:
            json.dump(sel, fh)
    out = {"shapes": shapes, "views": len(VIEWS)}
    for source in ("grid", "depth"):
        cfg = res64.get_config()
        cfg.device = torch.device("cuda:0")
        cfg.set_by_path("data.meta_path", metas["all"])
        cfg.set_by_path("eval.eval_dir", os.path.join(tmp, source))
        cfg.set_by_path("eval.partial_views", VIEWS)
        cfg.set_by_path("eval.partial_from", source)
        torch.cuda.synchronize()
        t = time.perf_counter()
        index = evaler.make_partial(cfg)
        torch.cuda.synchronize()
        sec = time.perf_counter() - t
        out[f"make_partial_{source}_s"] = sec
        out[f"make_partial_{source}_ms_per_file"] = sec / len(index) * 1e3
        out[f"visible_verts_{source}_mean"] = float(np.mean([e["visible_verts"] for e in index]))
    # completion on the first completion_shapes shapes of each set, views 0 and 25 only
    for source in ("grid", "depth"):
        part = os.path.join(tmp, f"{source}_subset")
        cfg = res64.get_config()
        cfg.device = torch.device("cuda:0")
        cfg.set_by_path("data.meta_path", metas["subset"])
        cfg.set_by_path("eval.eval_dir", part)
        cfg.set_by_path("eval.partial_views", (0, 25))
        cfg.set_by_path("eval.partial_from", source)
        evaler.make_partial(cfg)
        cfg = res64.get_config()
        cfg.device = torch.device("cuda:0")
        cfg.set_by_path("data.meta_path", metas["subset"])
        cfg.set_by_path("eval.eval_dir", os.path.join(tmp, f"completion_{source}"))
        cfg.set_by_path("eval.partial_dir", os.path.join(part, "partial"))
        cfg.set_by_path("eval.ckpt_path", os.path.join(tmp, "missing", "checkpoint.pth"))
        cfg.set_by_path("eval.tet_path", dmtet.tet_grid_path(64))
        cfg.set_by_path("eval.completion_k", 2)
        cfg.set_by_path("eval.batch_size", 8)
        cfg.set_by_path("eval.metric_points", 2048)
        cfg.set_by_path("sampling.method", "dpm_solver")
        cfg.set_by_path("sampling.dpm_steps", 10)
        cfg.model.compute_dtype = "bf16"
        t = time.perf_counter()
        completion.eval_completion(cfg)
        sec = time.perf_counter() - t
        with open(os.path.join(tmp, f"completion_{source}", "completion", "metrics.json")) as fh:
            m = json.load(fh)
        out[f"completion_{source}"] = {"seconds": sec, "partials": len(m["partials"]), "means": m["means"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=64)
    ap.add_argument("--completion-shapes", type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    out = dict(_card())
    out["kernels"] = [_kernels(R) for R in (64, 128)]
    out["batch"] = _batch()
    with tempfile.TemporaryDirectory() as tmp:
        out["make_partial"] = _make_partial(tmp, args.shapes, args.completion_shapes)
    out["sm_clock_after"] = _card()["sm_clock"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
