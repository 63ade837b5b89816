"""GPU: light field distance (geometry/lfd.py, csrc/lfd.cu) against the numpy restatement (oracle/lfd_oracle.py): camera
matrices bit for bit, descriptors byte for byte on the kernel's own face ids (random meshes, marching-tets meshes, a
one-pixel and an empty silhouette, res 256 and 97), the integer distance matrix, and `--mode=eval_metrics
--config.eval.metric_lfd=True` end to end."""
import json

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import lfd_oracle as lo

pytestmark = pytest.mark.gpu


def _random_mesh(rng, n_verts, n_faces, spread):
    """Random faces with both windings, degenerate faces and exact duplicates."""
    v = rng.uniform(-spread, spread, (n_verts, 3)).astype(np.float32)
    f = rng.integers(0, n_verts, (n_faces, 3))
    f[:n_faces // 4] = f[:n_faces // 4, ::-1]
    f[1::17, 2] = f[1::17, 1]
    dup = np.arange(2, n_faces - 1, 19)
    f[dup] = f[dup + 1]
    v[: n_verts // 8, 1] *= 2.5
    return v, f


def _pack(meshes):
    verts = torch.cat([torch.as_tensor(v) for v, _ in meshes]).cuda().float()
    faces = torch.cat([torch.as_tensor(f) for _, f in meshes]).cuda().long()
    vo = np.concatenate([[0], np.cumsum([len(v) for v, _ in meshes])])
    fo = np.concatenate([[0], np.cumsum([len(f) for _, f in meshes])])
    return verts, faces, vo, fo


def _mt_meshes(n=3, seed=5):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry.pointcloud import grids_to_meshes
    g = torch.Generator(device="cuda").manual_seed(seed)
    verts, faces, vo, fo = grids_to_meshes(synthetic_grids(n, 64, "cuda", generator=g), 64)
    return [(verts[vo[b]:vo[b + 1]].cpu().numpy(), faces[fo[b]:fo[b + 1]].cpu().numpy()) for b in range(n)]


def test_mvps_equal_the_oracle_bitwise():
    from meshdiffusion_b200.geometry import lfd
    rng = np.random.default_rng(3)
    meshes = [_random_mesh(rng, 200, 300, 0.7), _random_mesh(rng, 50, 80, 3.0)] + _mt_meshes(2)
    verts, _, vo, _ = _pack(meshes)
    centre, scale = lfd.normalization(verts, vo)
    got = lfd.camera_mvps(centre, scale)
    for b, (v, _) in enumerate(meshes):
        c, s = lo.centre_scale(v)
        np.testing.assert_array_equal(got[b].view(np.uint32), lo.mvps(lfd.ROTATIONS, c, s).view(np.uint32))


def _check_mesh_descriptors(meshes, res, views):
    from meshdiffusion_b200.geometry import lfd, singleview
    verts, faces, vo, fo = _pack(meshes)
    desc, empty = lfd.lfd_descriptors(verts, faces, vo, fo, res=res)
    assert desc.shape == (len(meshes), 10, 10, 48) and desc.dtype == torch.uint8
    centre, scale = lfd.normalization(verts, vo)
    mv = lfd.camera_mvps(centre, scale)
    covered = 0
    for b, (v, f) in enumerate(meshes):
        _, face_id = singleview.rasterize([(torch.as_tensor(v).cuda(), torch.as_tensor(f).cuda())], mv[b], res)
        masks = (face_id[0] >= 0).cpu().numpy()
        n_empty = 0
        for j in range(100):
            n_empty += not masks[j].any()
            if j in views:
                want, n = lo.descriptor(masks[j])
                np.testing.assert_array_equal(desc[b].view(100, 48)[j].cpu().numpy(), want, err_msg=f"mesh {b} view {j}")
                covered += n
        assert empty[b] == n_empty
    assert covered > 0


@pytest.mark.parametrize("res", [256, 97])
def test_descriptors_of_random_meshes_bitwise(res):
    rng = np.random.default_rng(res)
    meshes = [_random_mesh(rng, 120, 200, 0.8), _random_mesh(rng, 30, 40, 1.5)]
    _check_mesh_descriptors(meshes, res, views=set(range(0, 100, 9)))


def test_descriptors_of_marching_tets_meshes_bitwise():
    _check_mesh_descriptors(_mt_meshes(2), 256, views={0, 11, 37, 54, 99})


def test_an_empty_mesh_gets_empty_views_and_leaves_the_others_unchanged():
    from meshdiffusion_b200.geometry import lfd
    rng = np.random.default_rng(4)
    a, b = _random_mesh(rng, 60, 90, 0.8), _random_mesh(rng, 40, 50, 1.2)
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64))
    d3, e3 = lfd.lfd_descriptors(*_pack([a, empty, b]))
    d2, e2 = lfd.lfd_descriptors(*_pack([a, b]))
    assert not d3[1].any() and e3[1] == 100
    assert torch.equal(d3[[0, 2]], d2) and list(e3[[0, 2]]) == list(e2)
    d0, e0 = lfd.lfd_descriptors(*_pack([empty]))
    assert not d0.any() and list(e0) == [100]


@pytest.mark.parametrize("res", [256, 97])
def test_descriptors_of_small_and_empty_silhouettes(res):
    from meshdiffusion_b200.geometry import lfd
    ids = torch.full((5, res, res), -1, dtype=torch.int32)
    ids[1, 3, res - 2] = 0                        # one pixel
    ids[2, res // 2:res // 2 + 2, 10:13] = 4     # a 2 x 3 block
    ids[3, :, :] = 0                              # the whole image
    rng = np.random.default_rng(1)
    ids[4] = torch.from_numpy(np.where(rng.random((res, res)) < 0.3, 1, -1).astype(np.int32))  # scattered pixels
    desc, n = lfd.silhouette_descriptors(ids.cuda())
    for k in range(5):
        want, wn = lo.descriptor(ids[k].numpy() >= 0)
        assert int(n[k]) == wn
        np.testing.assert_array_equal(desc[k].cpu().numpy(), want, err_msg=f"image {k}")
    assert not desc[0].any() and int(n[0]) == 0


def test_native_argument_checks():
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.geometry import lfd
    with pytest.raises(_native.NativeError, match="res"):
        lfd.silhouette_descriptors(torch.zeros(1, 300, 300, dtype=torch.int32, device="cuda"))
    L = _native.lib()
    assert L.mdb_lfd_descriptors(None, 2, 64, None, None, None, None, None) != 0
    assert b"null pointer" in L.mdb_last_error()
    assert L.mdb_lfd_matrix(None, 3, None, 0, None, None, None) != 0
    assert L.mdb_lfd_matrix(None, 70000, None, 0, None, None, None) != 0
    with pytest.raises(ValueError):
        lfd.lfd_matrix(torch.zeros(2, 10, 10, 47, dtype=torch.uint8, device="cuda"))


def _random_descriptors(rng, n, base=None):
    """uint8 [n, 10, 10, 48] with zero padding bytes; with base, small perturbations of it (close pairs)."""
    if base is None:
        d = rng.integers(0, 256, (n, 10, 10, 48), dtype=np.int64)
    else:
        d = np.clip(base[rng.integers(0, len(base), n)] + rng.integers(-6, 7, (n, 10, 10, 48)), 0, 255)
    d[..., 45:] = 0
    return d.astype(np.uint8)


def test_matrix_matches_the_oracle():
    from meshdiffusion_b200.geometry import lfd
    rng = np.random.default_rng(7)
    A = _random_descriptors(rng, 13)
    B = np.concatenate([_random_descriptors(rng, 4), _random_descriptors(rng, 5, base=A)])  # nB = 9
    B[2] = A[5][:, lfd.PERMUTATIONS[23]]  # a rotated copy: distance 0
    got = lfd.lfd_matrix(torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()).cpu().numpy()
    want = lo.lfd_matrix(A, B, lfd.PERMUTATIONS)
    np.testing.assert_array_equal(got, want)
    assert got[5, 2] == 0
    self_ = lfd.lfd_matrix(torch.from_numpy(A).cuda()).cpu().numpy()
    np.testing.assert_array_equal(self_, lo.lfd_matrix(A, None, lfd.PERMUTATIONS))
    np.testing.assert_array_equal(self_, self_.T)
    assert not np.diag(self_).any()
    one = lfd.lfd_matrix(torch.from_numpy(A[7:8]).cuda(), torch.from_numpy(B[3:4]).cuda()).cpu().numpy()
    assert one.shape == (1, 1) and one[0, 0] == got[7, 3]


def test_matrix_is_batch_invariant_at_size():
    from meshdiffusion_b200.geometry import lfd
    rng = np.random.default_rng(9)
    A = torch.from_numpy(_random_descriptors(rng, 131)).cuda()
    B = torch.from_numpy(_random_descriptors(rng, 77, base=A.cpu().numpy())).cuda()
    big = lfd.lfd_matrix(A, B)
    assert torch.equal(lfd.lfd_matrix(A[40:45], B[70:77]), big[40:45, 70:77])
    s = lfd.lfd_matrix(A)
    assert torch.equal(s, s.T) and not bool(s.diagonal().any())
    assert torch.equal(lfd.lfd_matrix(A, A)[~torch.eye(131, dtype=torch.bool, device="cuda")],
                       s[~torch.eye(131, dtype=torch.bool, device="cuda")])


def _shape_grids(shapes, res=64):
    """[n,4,R,R,R] sign grids on the tet vertices: ('b', half sizes) boxes, ('s', radius) spheres, ('t', R, r) tori."""
    from meshdiffusion_b200.geometry import dmtet, formats
    verts, _ = dmtet.load_tet_grid(res)
    coords = dmtet.grid_coords_of_tet_vertices(verts)
    v = torch.tensor(verts)
    out = []
    for kind, *a in shapes:
        if kind == "s":
            sdf = a[0] - v.norm(dim=1)
        elif kind == "b":
            sdf = -(v.abs() / torch.tensor(a[0])).max(dim=1).values + 1
        else:
            q = torch.stack([(v[:, 0] ** 2 + v[:, 2] ** 2).sqrt() - a[0], v[:, 1]], 1)
            sdf = a[1] - q.norm(dim=1)
        out.append(formats.tets_to_3dgrid(coords, torch.sign(sdf), torch.zeros_like(v), res))
    return torch.stack(out)


GEN = [("s", 0.3), ("b", (0.25, 0.25, 0.25)), ("b", (0.35, 0.12, 0.2)), ("t", 0.25, 0.09), ("b", (0.1, 0.35, 0.1))]
REF = [("b", (0.3, 0.2, 0.08)), ("s", 0.22), ("t", 0.28, 0.06), ("b", (0.33, 0.11, 0.21))]


def _write_sets(tmp_path, gen, ref):
    eval_dir = tmp_path / "samples"
    eval_dir.mkdir()
    ref_dir = tmp_path / "ref"
    ref_dir.mkdir()
    np.save(eval_dir / "gen.npy", _shape_grids(gen).numpy())
    paths = []
    for k, g in enumerate(_shape_grids(ref).numpy()):
        p = str(ref_dir / f"shape_{k}.npy")
        np.save(p, g)
        paths.append(p)
    meta = tmp_path / "list.json"
    meta.write_text(json.dumps(sorted(paths)))
    return eval_dir, meta


def _eval(eval_dir, meta, lfd_flag):
    import main_diffusion
    args = [f"--config={ROOT}/configs/res64.py", "--mode=eval_metrics", f"--config.eval.eval_dir={eval_dir}",
            f"--config.data.meta_path={meta}", "--config.data.extension=npy", "--config.eval.metric_points=256"]
    if lfd_flag:
        args.append("--config.eval.metric_lfd=True")
    main_diffusion.main(args)
    return json.loads((eval_dir / "metrics.json").read_text())


def _descriptors(shapes):
    from meshdiffusion_b200.geometry import lfd
    from meshdiffusion_b200.geometry.pointcloud import grids_to_meshes
    verts, faces, vo, fo = grids_to_meshes(_shape_grids(shapes).cuda(), 64)
    return lfd.lfd_descriptors(verts, faces, vo, fo)[0].cpu().numpy()


def test_eval_metrics_with_lfd(tmp_path, monkeypatch):
    from meshdiffusion_b200.diffusion.gen_metrics import metrics_from_matrices
    from meshdiffusion_b200.geometry import lfd
    monkeypatch.chdir(tmp_path)
    eval_dir, meta = _write_sets(tmp_path, GEN, REF)
    plain = _eval(eval_dir, meta, False)
    assert not any("lfd" in k for k in plain)
    m = _eval(eval_dir, meta, True)
    for k, v in plain.items():
        if not k.endswith("_seconds"):
            assert m[k] == v, k
    g, r = _descriptors(GEN), _descriptors(REF)
    perms = lfd.PERMUTATIONS
    want = metrics_from_matrices(lo.lfd_matrix(g, r, perms), lo.lfd_matrix(g, None, perms), lo.lfd_matrix(r, None, perms),
                                 suffix="lfd")
    for k, v in want.items():
        assert m[k] == v, (k, m[k], v)
    assert m["mmd_lfd"] > 0 and 0 < m["cov_lfd"] <= 1
    assert m["lfd_convention"] == lfd.LFD_CONVENTION and m["lfd_empty_views"] == 0
    assert 0 <= m["lfd_saturated"] < 0.05 and m["lfd_seconds"] > 0


def test_eval_metrics_lfd_identical_sets(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    eval_dir, meta = _write_sets(tmp_path, GEN, GEN)
    m = _eval(eval_dir, meta, True)
    assert m["n_gen"] == m["n_ref"] == len(GEN)
    assert m["mmd_lfd"] == 0.0 and m["cov_lfd"] == 1.0 and m["1nna_lfd"] == 0.0
