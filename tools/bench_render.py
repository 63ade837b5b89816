"""Shaded previews (`--mode=export`): 64 synthetic res64 shapes (trainer.synthetic_grids) x 8 views at 1000 x 1000, ssaa 2.

    python tools/bench_render.py [--shapes 64] [--views 8] [--res 1000] [--ssaa 2] [--iters 3] [--no-e2e]

1. Kernels: rasterization at res * ssaa (mdb_raster_depth) plus shading (mdb_render_shade) of every (shape, view) job
   through `render.render_meshes`, on meshes extracted once, timed with CUDA events over `--iters` passes after a
   warm-up pass; reported per view.
2. End to end: one `--mode=export` run (export.export) over the same shapes, written as two `.npy` batches to a temporary
   directory that is removed afterwards: a host clock around a device synchronise, split into meshing, kernels (render
   and the copy of the images to the host) and file writes (OBJ and PNG) as the mode's index reports them.
Prints the card's name, power limit and SM clock with the numbers, as one JSON line.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit, clock = (s.strip() for s in q.split(","))
        return name, limit, clock
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=64)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--res", type=int, default=1000)
    ap.add_argument("--ssaa", type=int, default=2)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    from configs import res64
    from meshdiffusion_b200.diffusion import export
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet, mesh_ops, render
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    R, S, res, ssaa = 64, args.shapes, args.res, args.ssaa
    views = tuple(range(0, 50, 50 // args.views))[:args.views]
    grids = synthetic_grids(S, R, dev, generator=torch.Generator(device=dev).manual_seed(0))
    light = render.environment_light()

    # 1. kernels on meshes extracted once, 8 shapes per call as the mode renders them
    verts, tets = dmtet.load_tet_grid(R)
    v = torch.tensor(verts, device=dev)
    coords = dmtet.grid_coords_of_tet_vertices(v.cpu()).to(dev)
    mt = dmtet.MarchingTets(tets, verts.shape[0], max_batch=8)
    batches, n_faces = [], 0
    for b0 in range(0, S, 8):
        sdf, pos = dmtet.grid_to_tet_inputs(grids[b0:b0 + 8], coords, v, R, 1.1, 3.0)
        meshes = [(m[0], m[1]) for m in mt.extract(pos, sdf)]
        n_faces += sum(int(f.shape[0]) for _, f in meshes)
        batches.append((meshes, [mesh_ops.auto_normals(mv, mf)[0] for mv, mf in meshes]))

    def one_pass():
        return sum(render.render_meshes(m, n, views, res, ssaa, light).shape[0] * len(views) for m, n in batches)

    one_pass()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    jobs = sum(one_pass() for _ in range(args.iters))
    e1.record()
    torch.cuda.synchronize()
    ms_per_view = e0.elapsed_time(e1) / jobs
    out = {"workload": f"{S} synthetic res{R} shapes x {len(views)} views at {res}x{res}, ssaa {ssaa}",
           "views": list(views), "faces_per_shape": n_faces / S, "raster_shade_ms_per_view": ms_per_view,
           "views_per_s": 1e3 / ms_per_view}

    # 2. one export run end to end
    if not args.no_e2e:
        tmp = tempfile.mkdtemp(prefix="bench_render_")
        try:
            ev = os.path.join(tmp, "eval")
            os.makedirs(ev)
            g = grids.cpu().numpy()
            np.save(os.path.join(ev, "0.npy"), g[:S // 2])
            np.save(os.path.join(ev, "1.npy"), g[S // 2:])
            cfg = res64.get_config()
            cfg.device = dev
            cfg.eval.eval_dir = ev
            cfg.set_by_path("render.views", views)
            cfg.set_by_path("render.res", res)
            cfg.set_by_path("render.ssaa", ssaa)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            index = export.export(cfg)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            n_png = sum(len(e["png"]) for e in index["samples"])
            png_bytes = sum(os.path.getsize(os.path.join(ev, "export", "viz", p)) for e in index["samples"] for p in e["png"])
            out.update(export_seconds=sec, export_split_seconds=index["seconds"], export_samples=len(index["samples"]),
                       export_pngs=n_png, mean_png_kib=png_bytes / n_png / 1024)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    name, limit, clock = _card()
    out.update(gpu=name, power_limit=limit, sm_clock=clock)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
