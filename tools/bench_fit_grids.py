"""Benchmark of `--mode=fit_grids` (geometry/fit.py, csrc/fit.cu) on synthetic tori of about 20 k and 200 k faces at
R = 64 and R = 128.

1. End to end: the meshes are written as `.obj` files and fitted by the mode's driver with its defaults; reported per
   shape are the seconds of each stage (load / carve / fit / write) from its report, and the Chamfer distances.
2. Kernels: `mdb_closest_points` (the fitted mesh's marching-tet vertices against the source mesh) and
   `mdb_nearest_vertex` (the source samples against those vertices), timed with CUDA events over 20 launches after a
   warm-up. Reported as pairs per second and as a share of an FP32 issue bound: pairs x instructions per pair /
   (SMs x 128 lanes x SM clock). The instructions per pair are counted on the shortest path of the search: 30 for a
   closest point (9 FADD for ab, ac, ap; 10 for d1, d2; 2 comparisons; 8 for the distance; 1 for the minimum), 9 for a
   nearest vertex (3 FADD, 3 FMUL, 2 FADD, 1 comparison); a pair that reaches an edge or the interior of its triangle
   issues up to about 80, so the share understates the closest-point kernel's use of the issue slots.
3. --sweep: the convergence run behind the defaults of fit_iters / fit_lr / fit_reg: the point-to-surface distance after
   a range of iteration counts for a few learning rates and regularisers on the test shapes (icosphere, torus) at R = 64.

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

FP32_LANES_PER_SM = 128
INSTR_CLOSEST, INSTR_NEAREST = 30, 9


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit, sm, sm_max = (s.strip() for s in q.split(","))
        return {"gpu": name, "power_limit": limit, "sm_clock": sm, "sm_clock_max": sm_max,
                "sm_clock_mhz": float(sm.split()[0])}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown", "sm_clock": "unknown", "sm_clock_mhz": 1980.0}


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


def _end_to_end(tmp, R, shapes):
    from configs import res64
    from meshdiffusion_b200.diffusion.fit_grids import fit_grids
    from meshdiffusion_b200.geometry.mesh_ops import write_obj
    paths = []
    for name, (v, f) in shapes.items():
        paths.append(write_obj(tmp, torch.from_numpy(v), torch.from_numpy(f), f"{name}.obj"))
    meta = os.path.join(tmp, "meshes.json")
    with open(meta, "w") as fh:
        json.dump(paths, fh)
    cfg = res64.get_config()
    cfg.data.image_size = R
    cfg.device = torch.device("cuda:0")
    cfg.set_by_path("data.mesh_meta_path", meta)
    cfg.set_by_path("data.grid_dir", os.path.join(tmp, f"grids{R}"))
    t = time.perf_counter()
    report = fit_grids(cfg)
    wall = time.perf_counter() - t
    return wall, [{"shape": os.path.basename(r["source"]), "R": R, "faces": r["faces"], "mt_verts": r["mt_verts"],
                   "seconds": r["seconds"], "chamfer_before": r["chamfer_before"], "chamfer_after": r["chamfer_after"],
                   "surface_distance_before": r["surface_distance_before"],
                   "surface_distance_after": r["surface_distance_after"]} for r in report]


def _kernels(R, v, f, card):
    from meshdiffusion_b200.geometry import fit
    fitter = fit.GridFitter(R, iters=0, max_batch=1)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    r = fitter([(vt, ft)])[0]
    q = r["mesh"][0].contiguous()
    samples = fit._mesh_points(vt, ft, [0, v.shape[0]], [0, f.shape[0]], fit.POINTS, 0, [0]).reshape(-1, 3)
    out = {}
    for name, fn, pairs, instr in (
            ("closest_points", lambda: fit.closest_points(q, [0, q.shape[0]], vt, ft, [0, v.shape[0]], [0, f.shape[0]]),
             q.shape[0] * f.shape[0], INSTR_CLOSEST),
            ("nearest_vertex", lambda: fit.nearest_vertex(samples, [0, samples.shape[0]], q, [0, q.shape[0]]),
             samples.shape[0] * q.shape[0], INSTR_NEAREST)):
        s = _events(fn)
        card = _card()  # the clock under load, read right after the timed window
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        bound = pairs * instr / (sms * FP32_LANES_PER_SM * card["sm_clock_mhz"] * 1e6)
        out[name] = {"sm_clock": card["sm_clock"], "R": R, "faces": int(f.shape[0]), "mt_verts": int(q.shape[0]), "pairs": int(pairs), "seconds": s, "pairs_per_s": pairs / s, "fp32_issue_bound_s": bound,
                     "share_of_fp32_issue_bound": bound / s}
    return out


def _sweep():
    from meshdiffusion_b200.geometry import fit
    from oracle import fit_oracle as fo
    shapes = {"icosphere": fo.icosphere(), "torus": fo.torus()}
    rows = []
    for lr in (0.01, 0.02, 0.05):
        for reg in (0.0, 1e-4):
            for iters in (50, 100, 200, 400):
                fitter = fit.GridFitter(64, iters=iters, lr=lr, reg=reg, max_batch=2)
                res = fitter([(torch.from_numpy(v), torch.from_numpy(f)) for v, f in shapes.values()])
                rows.append({"lr": lr, "reg": reg, "iters": iters,
                             **{k: r["surface_distance_after"] for k, r in zip(shapes, res)},
                             **{k + "_chamfer": r["chamfer_after"] for k, r in zip(shapes, res)}})
                print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    from oracle import fit_oracle as fo
    assert torch.cuda.is_available(), "the benchmark needs a GPU"
    card = _card()
    out = dict(card)
    shapes = {"torus_20k": fo.torus(0.3, 0.12, 100, 100), "torus_200k": fo.torus(0.3, 0.12, 320, 320)}
    if not args.no_e2e:
        with tempfile.TemporaryDirectory() as tmp:
            out["end_to_end"] = []
            for R in (64, 128):
                wall, rows = _end_to_end(tmp, R, shapes)
                out["end_to_end"] += rows
                out[f"wall_seconds_R{R}"] = wall
    out["kernels"] = [_kernels(R, *shapes["torus_200k"], card) for R in (64, 128)]
    out["sm_clock_after"] = _card()["sm_clock"]
    if args.sweep:
        out["sweep"] = _sweep()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
