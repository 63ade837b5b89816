"""GPU: the depth-map kernels against the float32 oracle (bit for bit); partial DMTets built from rendered depth alone
against make_partial's grid-sign partials of the same shapes and views; determinism and batch independence; and
`--mode=partial_from_depth` -> `cond_gen` -> `export`, `make_partial --config.eval.partial_from=depth` ->
`eval_completion` end to end."""
import glob
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import depth_oracle as do

pytestmark = pytest.mark.gpu

CELL = 1.1 / 64


def _cameras():
    from meshdiffusion_b200.geometry.depth_partial import parse_camera, view_camera
    mv, proj = view_camera(9)
    proj = proj.clone()
    proj[0, 2], proj[1, 2] = 0.05, -0.03  # an off-centre principal point
    return [parse_camera({"view": 0}), parse_camera({"mv": mv.tolist(), "proj": proj.tolist()})]


def _random_depth(rng, res):
    """A smooth surface at depth ~2 with ripples, a depth step, holes, and zero / non-finite pixels."""
    y, x = np.meshgrid(np.linspace(-1, 1, res), np.linspace(-1, 1, res), indexing="ij")
    d = 2.0 + 0.1 * np.sin(5 * x + rng.uniform(0, 6)) * np.cos(4 * y) + 0.001 * rng.standard_normal((res, res))
    d[:, res // 3:res // 3 + 4] += 0.2
    d[rng.random((res, res)) < 0.01] = 0.0
    d[0, :5] = np.nan
    d[-1, -3:] = np.inf
    d[(x ** 2 + y ** 2) > 0.85] = 0.0
    return d.astype(np.float32)


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("res", [97, 256])
def test_unproject_and_closest_points_bitwise(res):
    from meshdiffusion_b200.geometry.depth_partial import depth_closest_points, unproject
    rng = np.random.default_rng(res)
    cams = _cameras()
    depth = np.stack([_random_depth(rng, res) for _ in cams])
    proj = torch.stack([c["proj"].reshape(16) for c in cams]).cuda()
    inv_mv = torch.stack([c["inv_mv"].reshape(16) for c in cams]).cuda()
    mvp = torch.stack([c["mvp"].reshape(16) for c in cams]).cuda()
    z, valid, pts, edge = (t.cpu().numpy() for t in unproject(torch.from_numpy(depth).cuda(), proj, inv_mv, CELL))
    queries, off, expect = [], [0], []
    for b, cam in enumerate(cams):
        ez, ev, ep, ee = do.unproject(depth[b], cam["proj"], cam["inv_mv"], CELL)
        for got, want in ((z[b], ez), (valid[b], ev), (pts[b], ep), (edge[b], ee)):
            _bits_equal(got, want)
        assert 0 < ee.sum() < (ev == 0).sum()
        surf = ep[ev == 0]
        q = surf[rng.integers(0, surf.shape[0], 400)] + rng.normal(0, 0.01, (400, 3))
        far = rng.uniform(-1, 1, (40, 3)) * 4.0                           # mostly nothing to find
        corner = np.stack([ep[1, 1], ep[res // 2, 0], ep[res - 2, res // 2]]) + 0.003  # windows at the border
        behind = cam["inv_mv"].numpy()[:3, 3] + 0.5 * cam["inv_mv"].numpy()[:3, 2]      # behind the camera
        q = np.concatenate([q, far, corner, behind[None]]).astype(np.float32)
        queries.append(q)
        off.append(off[-1] + q.shape[0])
        expect.append(do.closest_points(q, cam["mvp"], cam["proj"], CELL, ep, ev, ee))
    d2, cp, found = depth_closest_points(torch.from_numpy(np.concatenate(queries)).cuda(), off, mvp, proj, CELL,
                                         torch.from_numpy(pts).cuda(), torch.from_numpy(valid).cuda(),
                                         torch.from_numpy(edge).cuda())
    d2, cp, found = d2.cpu().numpy(), cp.cpu().numpy(), found.cpu().numpy()
    for b, (ed2, ecp, ef) in enumerate(expect):
        s = slice(off[b], off[b + 1])
        _bits_equal(d2[s], ed2)
        _bits_equal(cp[s], ecp)
        assert np.array_equal(found[s], ef)
        assert ef.sum() > 300 and (~ef).sum() > 20


# ---- round trip on shapes with a known answer ----------------------------------------------------------------------
VIEWS = (0, 17)
RES = 1000


def _shapes():
    """Two spheres of trainer.synthetic_grids and a torus fitted by fit_grids, as R = 64 grids [3, 4, 64, 64, 64]."""
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry.fit import GridFitter
    from oracle import fit_oracle as fo
    spheres = synthetic_grids(2, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(5))
    v, f = fo.torus()
    torus = GridFitter(64, max_batch=1)([(torch.from_numpy(v), torch.from_numpy(f))])[0]["grid"].cuda()
    return torch.cat([spheres, torus[None]])


@pytest.fixture(scope="module")
def round_trip():
    from meshdiffusion_b200.geometry.depth_partial import DepthPartials, parse_camera, render_depth
    from meshdiffusion_b200.geometry.singleview import PartialDMTets
    grids = _shapes()
    make = PartialDMTets(64, VIEWS, RES, 1.1, 3.0, "cuda")
    from_grid = make(grids)
    depth = render_depth(make, grids).cpu().numpy()
    cams = [parse_camera({"view": v}) for v in VIEWS]
    fit = DepthPartials(64, device="cuda")
    obs = [(b, k) for b in range(grids.shape[0]) for k in range(len(VIEWS))]
    from_depth = fit([depth[b, k] for b, k in obs], [cams[k] for _, k in obs], [(b, VIEWS[k]) for b, k in obs])
    return grids, make, fit, depth, cams, obs, from_grid, from_depth


def _interior(depth, cam, verts, cell):
    """bool [Nv]: the vertex projects onto observed surface with no empty or edge pixel within one cell edge."""
    from oracle.fit_oracle import mvp_rows
    res = depth.shape[0]
    _, valid, _, edge = do.unproject(depth, cam["proj"], cam["inv_mv"], cell)
    bad = torch.from_numpy(((valid != 0) | (edge != 0)).astype(np.float32))[None, None]
    h = mvp_rows(cam["mvp"], verts)
    X = (h[:, 0] / h[:, 3] * 0.5 + 0.5) * res
    Y = (h[:, 1] / h[:, 3] * 0.5 + 0.5) * res
    half = int(math.ceil(cell * abs(float(cam["proj"][0, 0])) * 0.5 * res / float(h[:, 3].min())))
    near_bad = torch.nn.functional.max_pool2d(bad, 2 * half + 1, 1, half)[0, 0].numpy() > 0
    inside = (X >= 0) & (X < res) & (Y >= 0) & (Y < res)
    out = np.zeros(verts.shape[0], bool)
    k = np.nonzero(inside)[0]
    out[k] = ~near_bad[Y[k].astype(np.int64), X[k].astype(np.int64)]
    return out


def test_round_trip_against_grid_sign_partials(round_trip):
    grids, make, fit, depth, cams, obs, from_grid, from_depth = round_trip
    verts = fit.grid_points.cpu().numpy()
    rows = []
    for n, (b, k) in enumerate(obs):
        g, _ = from_grid[b][k]
        d, rep = from_depth[n]
        vg, vd = g["vis"] > 0, d["vis"] > 0
        iou = float((vg & vd).sum()) / float((vg | vd).sum())
        sel = (vg & vd).numpy() & _interior(depth[b, k], cams[k], verts, fit.cell)
        agree = float((torch.sign(g["sdf"]) == d["sdf"]).numpy()[sel].mean())
        rows.append({"shape": b, "view": VIEWS[k], "sign_agreement": agree, "compared_verts": int(sel.sum()),
                     "vis_iou": iou, "distance_before": rep["distance_before"], "distance_after": rep["distance_after"]})
    print("round trip:", json.dumps(rows))
    for r in rows:
        assert r["compared_verts"] > 100, r
        assert r["sign_agreement"] >= 0.99, r
        assert r["vis_iou"] >= 0.9, r
        assert r["distance_after"] < r["distance_before"], r


def test_two_runs_identical_and_batch_independent(round_trip):
    from meshdiffusion_b200.geometry.depth_partial import DepthPartials
    grids, make, fit, depth, cams, obs, from_grid, from_depth = round_trip
    again = fit([depth[b, k] for b, k in obs], [cams[k] for _, k in obs], [(b, VIEWS[k]) for b, k in obs])
    for (d1, _), (d2, _) in zip(from_depth, again):
        for key in d1:
            assert torch.equal(d1[key], d2[key]), key
    # observation 1 alone, and inside a batch of 8 (the other observations repeated around it)
    alone = DepthPartials(64, max_batch=1)([depth[0, 1]], [cams[1]], [(0, VIEWS[1])])[0][0]
    order = [2, 3, 4, 1, 5, 0, 2, 3]
    batch = DepthPartials(64, max_batch=8)([depth[obs[i][0], obs[i][1]] for i in order], [cams[obs[i][1]] for i in order],
                                           [(obs[i][0], VIEWS[obs[i][1]]) for i in order])
    for key in alone:
        assert torch.equal(alone[key], batch[3][0][key]), key
        assert torch.equal(alone[key], from_depth[1][0][key]), key


# ---- end to end ------------------------------------------------------------------------------------------------------
def _run(args, cwd):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main_diffusion.py")] + args, cwd=cwd, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _grid_files(tmp_path):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    grids = synthetic_grids(2, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(2)).cpu()
    paths = []
    for i in range(2):
        p = os.path.join(tmp_path, f"grid_{100 + i}.pt")
        torch.save(grids[i].clone(), p)
        paths.append(p)
    meta = os.path.join(tmp_path, "meta.json")
    with open(meta, "w") as fh:
        json.dump(paths, fh)
    return grids, meta


def test_partial_from_depth_then_cond_gen_then_export_cli(tmp_path):
    from meshdiffusion_b200.geometry import dmtet
    from meshdiffusion_b200.geometry.depth_partial import render_depth, view_camera
    from meshdiffusion_b200.geometry.singleview import PartialDMTets
    grids, _ = _grid_files(tmp_path)
    res = 256
    depth = render_depth(PartialDMTets(64, (0, 17), res, 1.1, 3.0, "cuda"), grids.cuda()).cpu().numpy()
    mv, proj = view_camera(17)
    np.save(os.path.join(tmp_path, "front.npy"), depth[0, 0])
    np.save(os.path.join(tmp_path, "side.npy"), depth[1, 1])
    meta = os.path.join(tmp_path, "depth.json")
    with open(meta, "w") as fh:
        json.dump([{"depth": "front.npy", "view": 0}, {"depth": "side.npy", "mv": mv.tolist(), "proj": proj.tolist()}], fh)
    ev = os.path.join(tmp_path, "eval")
    _run([f"--config={ROOT}/configs/res64.py", "--mode=partial_from_depth", f"--config.eval.eval_dir={ev}",
          f"--config.eval.depth_meta_path={meta}"], cwd=str(tmp_path))
    with open(os.path.join(ev, "partial", "index.json")) as fh:
        index = json.load(fh)
    assert [e["file"] for e in index["files"]] == ["front.pt", "side.pt"]
    nv = dmtet.load_tet_grid(64)[0].shape[0]
    for e in index["files"]:
        d = torch.load(os.path.join(ev, "partial", e["file"]))
        assert set(d) == {"sdf", "deform", "vis", "vis_rast"} and d["sdf"].shape == (nv,) and d["deform"].shape == (nv, 3)
        assert e["res"] == res and e["visible_verts"] == int(d["vis"].sum()) > 0 and e["visible_tets"] > 0
        assert e["distance_after"] < e["distance_before"]
    assert index["files"][1]["mvp"] == (proj @ mv).tolist()
    out = os.path.join(tmp_path, "cond")
    _run([f"--config={ROOT}/configs/res64.py", "--mode=cond_gen", f"--config.eval.eval_dir={out}",
          f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth", "--config.eval.batch_size=1",
          f"--config.eval.partial_dmtet_path={os.path.join(ev, 'partial', 'side.pt')}",
          f"--config.eval.tet_path={dmtet.tet_grid_path(64)}", "--config.sampling.max_iters=4", "--config.eval.freeze_iters=3",
          "--config.model.compute_dtype=bf16"], cwd=str(tmp_path))
    x = np.load(os.path.join(out, "0.npy"))
    assert x.shape == (1, 4, 64, 64, 64) and np.isfinite(x).all()
    _run([f"--config={ROOT}/configs/res64.py", "--mode=export", f"--config.eval.eval_dir={out}", "--config.render.res=64",
          "--config.render.ssaa=1"], cwd=str(tmp_path))
    assert glob.glob(os.path.join(out, "export", "mesh", "*.obj"))


def test_make_partial_from_depth_then_eval_completion_cli(tmp_path):
    from meshdiffusion_b200.geometry import dmtet
    _, meta = _grid_files(tmp_path)
    ev = os.path.join(tmp_path, "eval")
    base = [f"--config={ROOT}/configs/res64.py", f"--config.data.meta_path={meta}"]
    _run(base + ["--mode=make_partial", f"--config.eval.eval_dir={ev}", "--config.eval.partial_views=(0, 17)",
                 "--config.eval.partial_res=256", "--config.eval.partial_from=depth"], cwd=str(tmp_path))
    with open(os.path.join(ev, "partial", "index.json")) as fh:
        index = json.load(fh)
    assert index["partial_from"] == "depth" and len(index["files"]) == 4
    for e in index["files"]:
        assert {"file", "shape", "source", "view", "mvp", "res", "visible_tets", "visible_verts"} <= set(e)
        assert e["distance_after"] < e["distance_before"]
    out = os.path.join(tmp_path, "completion")
    _run(base + ["--mode=eval_completion", f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth",
                 f"--config.eval.tet_path={dmtet.tet_grid_path(64)}", "--config.eval.completion_k=2",
                 "--config.eval.metric_points=512", "--config.model.compute_dtype=bf16", "--config.sampling.method=dpm_solver",
                 "--config.sampling.dpm_steps=3", "--config.eval.batch_size=4", f"--config.eval.eval_dir={out}",
                 f"--config.eval.partial_dir={ev}/partial"], cwd=str(tmp_path))
    with open(os.path.join(out, "completion", "metrics.json")) as fh:
        m = json.load(fh)
    assert len(m["partials"]) == 4 and m["means"]["scored"] == 4
