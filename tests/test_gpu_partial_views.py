"""GPU: the single-view rasterizer and visible-tet kernels against the float32 oracle (bit for bit), visibility sanity on a
convex shape, and `--mode=make_partial` -> `--mode=cond_gen` -> `tools/npy_to_obj.py` end to end."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import raster_oracle as ro

pytestmark = pytest.mark.gpu


def _random_mesh(rng, n_verts, n_faces, spread):
    v = rng.uniform(-spread, spread, (n_verts, 3)).astype(np.float32)
    f = rng.integers(0, n_verts, (n_faces, 3))
    f[:n_faces // 4] = f[:n_faces // 4, ::-1]            # the other winding (random faces have both anyway)
    f[1::17, 2] = f[1::17, 1]                             # degenerate: a repeated corner
    dup = np.arange(2, n_faces - 1, 19)
    f[dup] = f[dup + 1]                                   # exact duplicates: depth ties, the lower index wins
    v[: n_verts // 8, 1] *= 2.5                           # off-screen and partly off-screen triangles, all with w > 0
    return v, f


def _sphere_meshes(batch, resolution, seed):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet
    gen = torch.Generator(device="cuda").manual_seed(seed)
    grids = synthetic_grids(batch, resolution, torch.device("cuda"), generator=gen)
    verts, tets = dmtet.load_tet_grid(resolution)
    v = torch.tensor(verts, device="cuda")
    coords = dmtet.grid_coords_of_tet_vertices(v.cpu()).cuda()
    sdf, pos = dmtet.grid_to_tet_inputs(grids, coords, v, resolution, 1.1, 3.0 if resolution == 64 else 1.5)
    meshes = dmtet.MarchingTets(tets, verts.shape[0], max_batch=batch).extract(pos, sdf)
    return grids, pos, tets, meshes


@pytest.mark.parametrize("res", [64, 257])
def test_raster_random_meshes_bitwise(res):
    from meshdiffusion_b200.geometry.singleview import rasterize, view_mvp
    rng = np.random.default_rng(res)
    meshes = [_random_mesh(rng, 90, 120, 0.9), _random_mesh(rng, 40, 60, 0.6)]
    mvps = torch.stack([view_mvp(v, res) for v in (0, 13)])
    depth, face = rasterize([(torch.tensor(v).cuda(), torch.tensor(f).cuda()) for v, f in meshes], mvps, res)
    assert depth.shape == (2, 2, res, res) and face.dtype == torch.int32
    for m, (v, f) in enumerate(meshes):
        for k in range(2):
            want_d, want_f, behind = ro.rasterize(v, f, mvps[k].numpy(), res)
            assert behind == 0
            np.testing.assert_array_equal(face[m, k].cpu().numpy(), want_f)
            np.testing.assert_array_equal(depth[m, k].cpu().numpy().view(np.uint32), want_d.view(np.uint32))
            assert 0 < (want_f >= 0).mean() < 1


def test_raster_refuses_triangles_behind_the_camera():
    from meshdiffusion_b200.geometry.singleview import rasterize, view_mvp
    v = torch.tensor([[0, 0, 0], [0.2, 0, 0], [0, 0, 5.0]], device="cuda")
    with pytest.raises(ValueError, match="w <= 0"):
        rasterize([(v, torch.tensor([[0, 1, 2]], device="cuda"))], view_mvp(0, 64)[None], 64)


def test_raster_marching_tets_mesh_full_image():
    from meshdiffusion_b200.geometry.singleview import rasterize, view_mvp
    _, _, _, meshes = _sphere_meshes(1, 64, seed=0)
    v, f = meshes[0][0], meshes[0][1]
    mvp = view_mvp(17, 256)
    depth, face = rasterize([(v, f)], mvp[None], 256)
    want_d, want_f, _ = ro.rasterize(v.cpu().numpy(), f.cpu().numpy(), mvp.numpy(), 256)
    np.testing.assert_array_equal(face[0, 0].cpu().numpy(), want_f)
    np.testing.assert_array_equal(depth[0, 0].cpu().numpy().view(np.uint32), want_d.view(np.uint32))
    assert (want_f >= 0).sum() > 1000


def test_raster_res1000_sampled_pixels_brute_force():
    from meshdiffusion_b200.geometry.singleview import rasterize, view_mvp
    _, _, _, meshes = _sphere_meshes(1, 64, seed=1)
    v, f = meshes[0][0], meshes[0][1]
    mvp = view_mvp(31, 1000)
    depth, face = rasterize([(v, f)], mvp[None], 1000)
    rng = np.random.default_rng(7)
    covered = np.argwhere(face[0, 0].cpu().numpy() >= 0)
    pix = np.concatenate([rng.integers(0, 1000, (2048, 2)), covered[rng.integers(0, covered.shape[0], 2048)]])
    want_d, want_f = ro.rasterize_pixels(v.cpu().numpy(), f.cpu().numpy(), mvp.numpy(), 1000, pix[:, 0], pix[:, 1])
    got_d = depth[0, 0].cpu().numpy()[pix[:, 0], pix[:, 1]]
    got_f = face[0, 0].cpu().numpy()[pix[:, 0], pix[:, 1]]
    np.testing.assert_array_equal(got_f, want_f)
    np.testing.assert_array_equal(got_d.view(np.uint32), want_d.view(np.uint32))


@pytest.mark.parametrize("resolution,batch", [(64, 2), (128, 1)])
def test_visible_tets_bitwise(resolution, batch):
    from meshdiffusion_b200.geometry.singleview import rasterize, view_mvp, visible_tets
    _, pos, tets, meshes = _sphere_meshes(batch, resolution, seed=resolution)
    mvps = torch.stack([view_mvp(v, 1000) for v in (0, 17, 33)])
    depth, face = rasterize([(m[0], m[1]) for m in meshes], mvps, 1000)
    vis, rast = visible_tets(pos, tets, [m[4] for m in meshes], mvps, depth, face)
    assert vis.shape == (batch, 3, tets.shape[0]) and vis.dtype == torch.bool
    for b in range(batch):
        for k in range(3):
            want_v, want_r = ro.visible_tets(pos[b].cpu().numpy(), tets, meshes[b][4].cpu().numpy(), mvps[k].numpy(),
                                             depth[b, k].cpu().numpy(), face[b, k].cpu().numpy())
            np.testing.assert_array_equal(vis[b, k].cpu().numpy(), want_v)
            np.testing.assert_array_equal(rast[b, k].cpu().numpy(), want_r)
            assert want_v.any() and want_r.any()


def test_partial_dmtet_sanity_on_convex_shape():
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet
    from meshdiffusion_b200.geometry.singleview import PartialDMTets
    grids = synthetic_grids(1, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(5))
    make = PartialDMTets(64, views=(0, 25), res=1000)
    sdf, _, visible, rast = make.flags(grids)
    _, tets = dmtet.load_tet_grid(64)
    inside = (sdf[0][torch.tensor(tets, device="cuda").long()] > 0).all(1)
    assert inside.any()
    assert not (visible[0] & inside).any(), "a tet with all four vertices inside the sphere is marked visible"
    for d, n_vis in make(grids)[0]:
        vis, vis_rast = d["vis"].bool(), d["vis_rast"]
        assert vis.shape == vis_rast.shape == (make.n_verts,) and d["sdf"].shape == (make.n_verts,)
        assert d["deform"].shape == (make.n_verts, 3)
        assert not (vis & ~vis_rast).any()
        assert 0 < int(vis.sum()) < make.n_verts and n_vis > 0


def _run(args, cwd):
    r = subprocess.run([sys.executable] + args, cwd=cwd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def test_make_partial_then_cond_gen_cli(tmp_path):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet
    grids = synthetic_grids(3, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(2)).cpu()
    paths = []
    for i in range(3):
        p = os.path.join(tmp_path, f"grid_{100 + i}.pt")
        torch.save(grids[i].clone(), p)
        paths.append(p)
    meta = os.path.join(tmp_path, "meta.json")
    with open(meta, "w") as fh:
        json.dump(paths, fh)
    ev = os.path.join(tmp_path, "eval")
    _run([os.path.join(ROOT, "main_diffusion.py"), f"--config={ROOT}/configs/res64.py", "--mode=make_partial",
          f"--config.eval.eval_dir={ev}", f"--config.data.meta_path={meta}", "--config.eval.partial_views=(0, 17)",
          "--config.eval.partial_res=512"], cwd=str(tmp_path))
    files = sorted(glob.glob(os.path.join(ev, "partial", "*.pt")))
    assert [os.path.basename(f) for f in files] == [f"{i:06d}_view{v:02d}.pt" for i in range(3) for v in (0, 17)]
    with open(os.path.join(ev, "partial", "index.json")) as fh:
        index = json.load(fh)
    assert len(index["files"]) == 6 and index["deform_scale"] == 3.0 and index["res"] == 512
    nv = dmtet.load_tet_grid(64)[0].shape[0]
    for f, entry in zip(files, index["files"]):
        d = torch.load(f)
        assert set(d) == {"sdf", "deform", "vis", "vis_rast"}
        assert d["sdf"].shape == d["vis"].shape == d["vis_rast"].shape == (nv,) and d["deform"].shape == (nv, 3)
        assert entry["visible_verts"] == int(d["vis"].sum()) > 0 and entry["source"] == paths[entry["shape"]]
    out = os.path.join(tmp_path, "cond")
    _run([os.path.join(ROOT, "main_diffusion.py"), f"--config={ROOT}/configs/res64.py", "--mode=cond_gen",
          f"--config.eval.eval_dir={out}", f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth",
          "--config.eval.batch_size=1", f"--config.eval.partial_dmtet_path={files[1]}",
          f"--config.eval.tet_path={dmtet.tet_grid_path(64)}", "--config.sampling.max_iters=4", "--config.eval.freeze_iters=3",
          "--config.model.compute_dtype=bf16"], cwd=str(tmp_path))
    x = np.load(os.path.join(out, "0.npy"))
    assert x.shape == (1, 4, 64, 64, 64) and np.isfinite(x).all()
    _run([os.path.join(ROOT, "tools", "npy_to_obj.py"), f"--sample_path={os.path.join(out, '0.npy')}",
          f"--out_dir={os.path.join(tmp_path, 'obj')}"], cwd=str(tmp_path))
    assert glob.glob(os.path.join(tmp_path, "obj", "*"))
