"""GPU: the preview shading kernel (`mdb_render_shade`) bit for bit against the float32 oracle on random and marching-tets
meshes, its error paths, and `--mode=export` end to end (file names, index, images, the `.obj` files against
`tools/npy_to_obj.py`, and a two-rank split)."""
import glob
import json
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import render_oracle as rdo

pytestmark = pytest.mark.gpu

KD = (0.75, 0.3, 0.6)
WHITE = (1.0, 1.0, 1.0)


def _random_mesh(rng, n_verts, n_faces, spread):
    """Random faces with both windings, degenerate faces, exact duplicates and (partly) off-screen faces, and random
    normals, some of them zero."""
    v = rng.uniform(-spread, spread, (n_verts, 3)).astype(np.float32)
    f = rng.integers(0, n_verts, (n_faces, 3))
    f[:n_faces // 4] = f[:n_faces // 4, ::-1]
    f[1::17, 2] = f[1::17, 1]
    dup = np.arange(2, n_faces - 1, 19)
    f[dup] = f[dup + 1]
    v[: n_verts // 8, 1] *= 2.5
    n = rng.normal(size=(n_verts, 3)).astype(np.float32)
    n[::11] = 0
    return v, f, n


def _synthetic_light(seed):
    """SH coefficients of a random smooth lat-long map."""
    rng = np.random.default_rng(seed)
    d, _ = rdo.latlong_dirs(32, 64)
    m = 0.4 + 0.3 * np.stack([np.cos(3 * d[..., k] + rng.uniform(0, 6)) for k in range(3)], -1)
    m += 4 * np.exp((d @ np.array([0.0, 0.6, 0.8]) - 1) / 0.05)[..., None]
    return rdo.sh9_irradiance(m)


def _check(images, meshes, normals, views, res, ssaa, light):
    from meshdiffusion_b200.geometry import render
    sh = np.asarray(light, np.float64).astype(np.float32)
    covered = 0
    for m, ((v, f), n) in enumerate(zip(meshes, normals)):
        v, f, n = (np.asarray(x.cpu()) if torch.is_tensor(x) else x for x in (v, f, n))
        for k, view in enumerate(views):
            mv, mvp = render.view_camera(view, res)
            want, face_id, behind = rdo.render(v, f, n, mvp.numpy(), render.camera_position(mv).numpy(), res, ssaa, sh, KD,
                                               WHITE)
            assert behind == 0
            np.testing.assert_array_equal(images[m, k].cpu().numpy(), want, err_msg=f"mesh {m} view {view}")
            covered += int((face_id >= 0).sum())
    assert covered > 0


@pytest.mark.parametrize("res,ssaa", [(64, 1), (61, 2), (48, 3)])
def test_shade_random_meshes_bitwise(res, ssaa):
    from meshdiffusion_b200.geometry import render
    rng = np.random.default_rng(res + ssaa)
    meshes = [_random_mesh(rng, 90, 120, 0.9), _random_mesh(rng, 40, 60, 0.6)]
    views = (0, 13, 25)
    light = _synthetic_light(ssaa)
    images = render.render_meshes([(torch.tensor(v).cuda(), torch.tensor(f).cuda()) for v, f, _ in meshes],
                                  [torch.tensor(n).cuda() for _, _, n in meshes], views, res, ssaa, light)
    assert images.shape == (2, 3, res, res, 3) and images.dtype == torch.uint8 and images.is_cuda
    _check(images, [(v, f) for v, f, _ in meshes], [n for _, _, n in meshes], views, res, ssaa, light)
    assert (images != 255).any() and (images == 255).any()


def _sphere_meshes(batch, seed):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet, mesh_ops
    gen = torch.Generator(device="cuda").manual_seed(seed)
    grids = synthetic_grids(batch, 64, torch.device("cuda"), generator=gen)
    verts, tets = dmtet.load_tet_grid(64)
    v = torch.tensor(verts, device="cuda")
    coords = dmtet.grid_coords_of_tet_vertices(v.cpu()).cuda()
    sdf, pos = dmtet.grid_to_tet_inputs(grids, coords, v, 64, 1.1, 3.0)
    meshes = [(m[0], m[1]) for m in dmtet.MarchingTets(tets, verts.shape[0], max_batch=batch).extract(pos, sdf)]
    return meshes, [mesh_ops.auto_normals(mv, mf)[0] for mv, mf in meshes]


@pytest.mark.parametrize("ssaa,light", [(1, "default"), (3, "synthetic")])
def test_shade_marching_tets_spheres_bitwise(ssaa, light):
    from meshdiffusion_b200.geometry import render
    meshes, normals = _sphere_meshes(2, seed=ssaa)
    views, res = (0, 25, 37), 96
    sh = render.environment_light() if light == "default" else _synthetic_light(7)
    images = render.render_meshes(meshes, normals, views, res, ssaa, sh)
    _check(images, meshes, normals, views, res, ssaa, sh)
    assert (images[:, :, 0, 0] == 255).all()
    if light == "default":  # a pink sphere on white: the centre is kd-tinted (red > blue > green)
        centre = images[:, :, res // 2, res // 2].int().cpu()
        assert (centre[..., 0] > centre[..., 2]).all() and (centre[..., 2] > centre[..., 1]).all()


def test_render_default_light_matches_explicit_default():
    from meshdiffusion_b200.geometry import render
    meshes, normals = _sphere_meshes(1, seed=4)
    a = render.render_meshes(meshes, normals, (25,), 64, 2)
    b = render.render_meshes(meshes, normals, (25,), 64, 2, render.environment_light())
    assert torch.equal(a, b)


def test_render_error_paths():
    from meshdiffusion_b200.geometry import render
    v = torch.tensor([[0, 0, 0], [0.2, 0, 0], [0, 0, 5.0]], device="cuda")  # (0, 0, 5) is behind view 0's camera
    f = torch.tensor([[0, 1, 2]], device="cuda")
    n = torch.zeros_like(v)
    with pytest.raises(ValueError, match="w <= 0"):
        render.render_meshes([(v, f)], [n], (0,), 64, 2)
    ok = [(torch.tensor([[0, 0, 0], [0.2, 0, 0], [0, 0.2, 0]], device="cuda"), f)]
    for res, ssaa, msg in ((64, 0, "ssaa"), (64, 5, "ssaa"), (8192, 3, "res \\* ssaa"), (0, 1, "res \\* ssaa")):
        with pytest.raises(ValueError, match=msg):
            render.render_meshes(ok, [n], (0,), res, ssaa)
    with pytest.raises(ValueError, match="normal"):
        render.render_meshes([(v, f)], [n[:2]], (25,), 64, 1)


def _read_png(path):
    data = open(path, "rb").read()
    pos, idat, ihdr = 8, b"", None
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if tag == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        pos += 12 + n
    w, h = ihdr[:2]
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 3 * w)
    return raw[:, 1:].reshape(h, w, 3)


def _run(args, cwd, env=None):
    r = subprocess.run([sys.executable] + args, cwd=cwd, capture_output=True, text=True, timeout=900,
                       env=None if env is None else {**os.environ, **env})
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _write_batches(tmp_path):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    grids = synthetic_grids(3, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(9)).cpu().numpy()
    empty = np.zeros_like(grids[:1])
    empty[:, 0] = -1.0  # every tet vertex outside: no surface
    ev = tmp_path / "eval"
    ev.mkdir()
    np.save(ev / "a.npy", grids[:2])
    np.save(ev / "b.npy", np.concatenate([grids[2:], empty]))
    return ev


def test_export_cli_end_to_end(tmp_path):
    ev = _write_batches(tmp_path)
    res = 200
    _run([os.path.join(ROOT, "main_diffusion.py"), f"--config={ROOT}/configs/res64.py", "--mode=export",
          f"--config.eval.eval_dir={ev}", "--config.render.views=(0, 25)", f"--config.render.res={res}"], cwd=str(tmp_path))
    out = ev / "export"
    names = [f"{s}_{i:06d}" for s, i in (("a", 0), ("a", 1), ("b", 0), ("b", 1))]
    assert sorted(os.listdir(out / "mesh")) == [n + ".obj" for n in names]
    assert sorted(os.listdir(out / "viz")) == [f"{n}_view{v:02d}.png" for n in names for v in (0, 25)]
    index = json.load(open(out / "index.json"))
    assert index["views"] == [0, 25] and index["res"] == res and index["ssaa"] == 2 and index["light"] == "default"
    assert index["deform_scale"] == 3.0 and set(index["seconds"]) == {"meshing", "render", "write"}
    got = [(os.path.basename(e["source"]), e["batch_index"], e["empty"]) for e in index["samples"]]
    assert got == [("a.npy", 0, False), ("a.npy", 1, False), ("b.npy", 0, False), ("b.npy", 1, True)]
    for e, n in zip(index["samples"], names):
        assert e["obj"] == n + ".obj" and e["png"] == [f"{n}_view00.png", f"{n}_view25.png"]
        assert (e["faces"] == 0) == e["empty"] and (e["verts"] == 0) == e["empty"]
        for png in e["png"]:
            img = _read_png(out / "viz" / png)
            assert img.shape == (res, res, 3)
            assert (img[0, 0] == 255).all() and (img[-1, -1] == 255).all()
            c = img[res // 2, res // 2].astype(int)
            if e["empty"]:
                assert (img == 255).all()
            else:
                assert c[0] > c[2] > c[1]  # kd = (0.75, 0.3, 0.6)
    # the meshes are the ones tools/npy_to_obj.py writes for the same grids
    for stem in ("a", "b"):
        obj = tmp_path / f"obj_{stem}"
        _run([os.path.join(ROOT, "tools", "npy_to_obj.py"), f"--sample_path={ev / (stem + '.npy')}", f"--out_dir={obj}"],
             cwd=str(tmp_path))
        for i in range(2):
            assert (obj / str(i) / "mesh.obj").read_bytes() == (out / "mesh" / f"{stem}_{i:06d}.obj").read_bytes()


def test_export_two_rank_split(tmp_path):
    ev = _write_batches(tmp_path)
    for rank in (0, 1):
        _run([os.path.join(ROOT, "main_diffusion.py"), f"--config={ROOT}/configs/res64.py", "--mode=export",
              f"--config.eval.eval_dir={ev}", "--config.render.res=64", "--config.render.ssaa=1"], cwd=str(tmp_path),
             env={"RANK": str(rank), "WORLD_SIZE": "2"})
    out = ev / "export"
    assert not (out / "index.json").exists()
    seen = []
    for rank in (0, 1):
        index = json.load(open(out / f"index_{rank}.json"))
        seen += [(os.path.basename(e["source"]), e["batch_index"]) for e in index["samples"]]
        assert len(index["samples"]) == 2
    assert sorted(seen) == [("a.npy", 0), ("a.npy", 1), ("b.npy", 0), ("b.npy", 1)]
    assert len(glob.glob(str(out / "mesh" / "*.obj"))) == 4 and len(glob.glob(str(out / "viz" / "*.png"))) == 4
