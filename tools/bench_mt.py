"""Marching-tetrahedra + mesh post-op throughput (BASELINE.json configs[4] tail: grids -> meshes), one GPU.

    python tools/bench_mt.py [--resolution 64] [--batch 32] [--steps 20]

A step = one batch of `batch` samples through `MarchingTets.extract` (count pass, host read of the per-sample counts,
extract pass; the public call a user makes) followed by smooth normals for every sample. Inputs are noisy sphere SDFs with
random deformations on the reference's tet grid. Reports tets/s (all tets of the grid are visited per sample), ms per
batch and the effective HBM rate against the algorithmic bytes (tets 16 B + edge table + sdf/pos per sample).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolution", type=int, default=64)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    from meshdiffusion_b200.geometry import dmtet, mesh_ops
    dev = torch.device("cuda:0")
    verts, idx = dmtet.load_tet_grid(args.resolution)
    v = torch.tensor(verts, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    B, Nv, F = args.batch, verts.shape[0], idx.shape[0]
    radius = 0.25 + 0.1 * torch.rand(B, 1, device=dev, generator=g)
    sdf = torch.sign(radius - v.norm(dim=1)[None] + 0.02 * torch.randn(B, Nv, device=dev, generator=g))
    pos = v[None] + (torch.rand(B, Nv, 3, device=dev, generator=g) - 0.5) * (0.4 / args.resolution)
    mt = dmtet.MarchingTets(idx, Nv, max_batch=B)

    def step(with_normals):
        meshes = mt.extract(pos, sdf)
        if with_normals:
            for mv, mf, *_ in meshes:
                mesh_ops.auto_normals(mv, mf)
        return meshes

    res = {}
    for name, wn in (("extract", False), ("extract+normals", True)):
        for _ in range(3):
            meshes = step(wn)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            step(wn)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        res[name] = {"ms_per_batch": ms, "samples_per_s": B / (ms * 1e-3), "tets_per_s": B * F / (ms * 1e-3)}
    # differentiable path: extract with autograd + the backward gather kernel (d sum(verts) / d(pos, sdf))
    sdf_c = (sdf * (0.05 + torch.rand(B, Nv, device=dev, generator=g))).requires_grad_(True)
    pos_g = pos.clone().requires_grad_(True)

    def step_grad():
        ms_ = mt.extract(pos_g, sdf_c)
        loss = sum(m[0].sum() for m in ms_)
        pos_g.grad = sdf_c.grad = None
        loss.backward()

    for _ in range(3):
        step_grad()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step_grad()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    res["extract+backward"] = {"ms_per_batch": ms, "samples_per_s": B / (ms * 1e-3),
                               "note": "autograd node + mdb_marching_tets_backward (incl. the per-sample torch sum/slice ops of this loss)"}
    faces = sum(m[1].shape[0] for m in meshes)
    alg_bytes = B * (F * 16 + mt.n_edges * 8 + Nv * 16)
    ms = res["extract"]["ms_per_batch"]
    print(json.dumps({"metric": "marching-tet extraction", "resolution": args.resolution, "batch": B, "tets": F, "tet_vertices": Nv,
                      "unique_edges": mt.n_edges, "faces_per_batch": faces, **res,
                      "roofline": {"bound": "hbm", "algorithmic_bytes_per_batch": alg_bytes,
                                   "achieved_GBps": alg_bytes / (ms * 1e-3) / 1e9, "peak_GBps": 3350.0,  # H100 SXM data sheet (HBM3)
                                   "note": "latency / host-sync dominated at these sizes: the count pass returns per-sample sizes to the host"}}))


if __name__ == "__main__":
    main()
