"""Single-view partial DMTets: 64 synthetic res64 shapes (trainer.synthetic_grids) x 50 validation views at 1000 x 1000.

    python tools/bench_partial_views.py [--shapes 64] [--views 50] [--res 1000] [--iters 5] [--no-e2e]

1. Kernels: rasterization (mdb_raster_depth) plus visibility (mdb_visible_tets) of every (shape, view) job, on meshes
   extracted once, timed with CUDA events over `--iters` passes after a warm-up pass; reported per view.
2. End to end: one `--mode=make_partial` run (evaler.make_partial) over the same shapes and views, written to a temporary
   directory that is removed afterwards; a host clock around a device synchronise.
Prints the card name and power limit with the numbers, as one JSON line.
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=64)
    ap.add_argument("--views", type=int, default=50)
    ap.add_argument("--res", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    from configs import res64
    from meshdiffusion_b200.diffusion import evaler
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import singleview
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    R, S, V, res = 64, args.shapes, args.views, args.res
    grids = synthetic_grids(S, R, dev, generator=torch.Generator(device=dev).manual_seed(0))
    make = singleview.PartialDMTets(R, tuple(range(V)), res, 1.1, 3.0, dev, max_batch=8)

    # 1. kernels on meshes extracted once per batch of 8 shapes
    batches = []
    for b0 in range(0, S, make.max_batch):
        g = grids[b0:b0 + make.max_batch]
        sdf, pos = singleview.dmtet.grid_to_tet_inputs(g, make.coords, make.verts, R, 1.1, 3.0)
        verts, faces, _, f2t, _, off = make.mt._extract_raw(pos, sdf)
        vert_off = torch.from_numpy(np.ascontiguousarray(off[:-1, 0])).to(dev)
        face_off = torch.from_numpy(np.ascontiguousarray(off[:, 1])).to(dev)
        job_mesh, mvp = singleview._jobs(g.shape[0], make.mvps, dev)
        batches.append((verts, faces, vert_off, face_off, pos, f2t, job_mesh, mvp, int(off[-1, 1])))
    step = max(1, singleview._MAX_JOB_PIXELS // (res * res))

    def one_pass():
        n = 0
        for verts, faces, vert_off, face_off, pos, f2t, job_mesh, mvp, _ in batches:
            for j0 in range(0, job_mesh.shape[0], step):
                jm, mv = job_mesh[j0:j0 + step].contiguous(), mvp[j0:j0 + step].contiguous()
                depth, face_id = singleview._raster_packed(verts, faces, vert_off, face_off, jm, mv, res)
                singleview._visible_packed(pos, make.tets, f2t, face_off, jm, mv, depth, face_id)
                n += jm.shape[0]
        return n

    one_pass()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    jobs = sum(one_pass() for _ in range(args.iters))
    e1.record()
    torch.cuda.synchronize()
    ms_per_view = e0.elapsed_time(e1) / jobs
    out = {"workload": f"{S} synthetic res{R} shapes x {V} validation views at {res}x{res}",
           "faces_per_shape": sum(b[-1] for b in batches) / S, "tets": int(make.tets.shape[0]),
           "raster_visibility_ms_per_view": ms_per_view, "views_per_s": 1e3 / ms_per_view}

    # 2. one make_partial run end to end
    if not args.no_e2e:
        tmp = tempfile.mkdtemp(prefix="bench_partial_")
        try:
            paths = []
            for i in range(S):
                p = os.path.join(tmp, f"grid_{i}.pt")
                torch.save(grids[i].cpu().clone(), p)
                paths.append(p)
            meta = os.path.join(tmp, "meta.json")
            with open(meta, "w") as fh:
                json.dump(paths, fh)
            cfg = res64.get_config()
            cfg.device = dev
            cfg.data.meta_path = meta
            cfg.eval.eval_dir = os.path.join(tmp, "eval")
            cfg.eval.partial_views = tuple(range(V))
            cfg.eval.partial_res = res
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            index = evaler.make_partial(cfg)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            out.update(make_partial_seconds=sec, make_partial_files=len(index), make_partial_ms_per_file=sec / len(index) * 1e3,
                       mean_visible_tets=float(np.mean([e["visible_tets"] for e in index])))
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    name, limit = _card()
    out.update(gpu=name, power_limit=limit)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
