"""Point-cloud metrics on the GPU: surface sampling and the Chamfer matrix kernel against the numpy oracle
(oracle/pc_metrics_oracle.py), their reproducibility and batch invariance, the MMD / COV / 1-NNA metrics on synthetic shape
sets, and `main_diffusion.py --mode=eval_metrics`."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import pc_metrics_oracle as pco
from oracle import synth

pytestmark = pytest.mark.gpu


def _packed_meshes(cases, res=64):
    """Marching-tet meshes of synth.synthetic_dmtet fields, packed: (verts, faces, off [B+1, 3])."""
    from meshdiffusion_b200.geometry import dmtet
    verts, idx = dmtet.load_tet_grid(res)
    sdfs, poss = zip(*[synth.synthetic_dmtet(verts, seed=s, noisy=n, res=res) for s, n in cases])
    mt = dmtet.MarchingTets(idx, verts.shape[0], max_batch=len(cases))
    v, f, _, _, _, off = mt._extract_raw(torch.tensor(np.stack(poss)).cuda(), torch.tensor(np.stack(sdfs)).cuda())
    return v, f, off


def test_sampling_with_given_uniforms_matches_the_oracle():
    from meshdiffusion_b200.geometry.pointcloud import sample_surface_points
    v, f, off = _packed_meshes([(0, False), (1, True)])
    N = 4096
    u = np.random.RandomState(5).rand(2, N, 3).astype(np.float32)
    pts, empty = sample_surface_points(v, f, off[:, 0], off[:, 1], N, seed=0, uniforms=torch.tensor(u).cuda())
    assert not empty.any().item()
    pts = pts.cpu().numpy()
    vh, fh = v.cpu().numpy(), f.cpu().numpy()
    for b in range(2):
        mv, mf = vh[off[b, 0]:off[b + 1, 0]], fh[off[b, 1]:off[b + 1, 1]]
        want, face = pco.sample_points(mv, mf, u[b])
        # agreement to 1e-6 means the same faces were chosen: the same (r1, r2) on another triangle lands elsewhere
        assert np.abs(pts[b] - want).max() < 1e-6, b
        assert len(np.unique(face)) > 100


def test_philox_sampling_is_reproducible_and_batch_invariant():
    from meshdiffusion_b200.geometry.pointcloud import sample_surface_points
    v, f, off = _packed_meshes([(0, False), (1, True), (2, True)])
    p1, _ = sample_surface_points(v, f, off[:, 0], off[:, 1], 1000, seed=123)
    p2, _ = sample_surface_points(v, f, off[:, 0], off[:, 1], 1000, seed=123)
    assert torch.equal(p1, p2)
    p3, _ = sample_surface_points(v, f, off[:, 0], off[:, 1], 1000, seed=124)
    assert not torch.equal(p1, p3)
    for b in range(3):
        vb, fb = v[off[b, 0]:off[b + 1, 0]], f[off[b, 1]:off[b + 1, 1]]
        alone, _ = sample_surface_points(vb, fb, [0, vb.shape[0]], [0, fb.shape[0]], 1000, seed=123, first_id=b)
        assert torch.equal(alone[0], p1[b]), b
    # the uniforms are in [0, 1): every point lies inside the mesh's bounding box
    for b in range(3):
        vb = v[off[b, 0]:off[b + 1, 0]]
        assert bool((p1[b] >= vb.min(0).values - 1e-6).all() and (p1[b] <= vb.max(0).values + 1e-6).all())


def test_empty_and_zero_area_meshes_are_flagged_and_not_written():
    from meshdiffusion_b200.geometry.pointcloud import sample_surface_points
    tri_v = [[0, 0, 0], [1, 0, 0], [0, 1, 0]]
    flat_v = [[0.5, 0.5, 0.5]] * 3
    verts = torch.tensor(tri_v + flat_v + tri_v + flat_v, dtype=torch.float32).cuda()
    # mesh 0: a triangle; mesh 1: three vertices, no faces; mesh 2: a triangle; mesh 3: a zero-area face
    faces = torch.tensor([[0, 1, 2], [0, 1, 2], [0, 0, 1]], dtype=torch.int64).cuda()
    pts, empty = sample_surface_points(verts, faces, [0, 3, 6, 9, 12], [0, 1, 1, 2, 3], 64, seed=1)
    assert empty.tolist() == [False, True, False, True]
    assert torch.isnan(pts[1]).all() and torch.isnan(pts[3]).all()
    assert torch.isfinite(pts[0]).all() and torch.isfinite(pts[2]).all()
    assert float(pts[0, :, 2].abs().max()) == 0.0 and float((pts[0, :, 0] + pts[0, :, 1]).max()) <= 1.0 + 1e-6


def test_out_of_range_faces_raise():
    from meshdiffusion_b200.geometry.pointcloud import sample_surface_points
    verts = torch.rand(6, 3).cuda()
    ok = torch.tensor([[0, 1, 2], [0, 1, 2]], dtype=torch.int64).cuda()
    sample_surface_points(verts, ok, [0, 3, 6], [0, 1, 2], 8, seed=0)
    for bad in ([[0, 1, 2], [0, 1, 3]], [[0, 1, -1], [0, 1, 2]]):
        with pytest.raises(ValueError):
            sample_surface_points(verts, torch.tensor(bad, dtype=torch.int64).cuda(), [0, 3, 6], [0, 1, 2], 8, seed=0)


def _sphere_clouds(n, pts, seed, jitter=0.05):
    """Unit-scale surfaces: noisy points on spheres of varying radius and centre (nearest-neighbour d ~ 1e-3)."""
    rng = np.random.RandomState(seed)
    x = rng.randn(n, pts, 3)
    x /= np.linalg.norm(x, axis=2, keepdims=True)
    x *= 0.3 + 0.2 * rng.rand(n, 1, 1)
    x += jitter * rng.randn(n, 1, 3) + 0.002 * rng.randn(n, pts, 3)
    return x.astype(np.float32)


@pytest.mark.parametrize("N,M", [(1, 1), (1, 17), (17, 2047), (2048, 2048), (2500, 2047), (2048, 1), (2047, 2500)])
def test_chamfer_matrix_matches_the_fp64_oracle(N, M):
    from meshdiffusion_b200.geometry.pointcloud import chamfer_matrix
    A, B = _sphere_clouds(3, N, N), _sphere_clouds(2, M, M + 1)
    got = chamfer_matrix(torch.tensor(A).cuda(), torch.tensor(B).cuda()).cpu().numpy()
    assert got.shape == (3, 2) and got.dtype == np.float64
    want = pco.chamfer_matrix(A, B)
    assert np.abs(got - want).max() / np.abs(want).max() < 2e-6
    assert np.all(np.abs(got - want) <= 2e-6 * want)


def test_chamfer_matrix_is_symmetric_batch_invariant_and_reproducible():
    from meshdiffusion_b200.geometry.pointcloud import chamfer_matrix
    A = torch.tensor(_sphere_clouds(5, 1100, 7)).cuda()
    B = torch.tensor(_sphere_clouds(4, 1100, 8)).cuda()
    ab = chamfer_matrix(A, B)
    ba = chamfer_matrix(B, A)
    assert torch.equal(ab, ba.T)
    assert torch.equal(ab, chamfer_matrix(A, B))
    for i, j in ((0, 0), (4, 3), (2, 1)):
        assert torch.equal(chamfer_matrix(A[i:i + 1], B[j:j + 1])[0, 0], ab[i, j])
    # different point counts: symmetry holds across N != M too
    C = torch.tensor(_sphere_clouds(3, 333, 9)).cuda()
    assert torch.equal(chamfer_matrix(A, C), chamfer_matrix(C, A).T)


def test_self_matrix_is_symmetric_with_zero_diagonal_and_equals_the_cross_call():
    from meshdiffusion_b200.geometry.pointcloud import chamfer_matrix
    A = torch.tensor(_sphere_clouds(6, 2048, 10)).cuda()
    s = chamfer_matrix(A)
    assert torch.equal(s, s.T)
    assert torch.equal(torch.diagonal(s), torch.zeros(6, dtype=torch.float64, device=s.device))
    cross = chamfer_matrix(A, A)
    off = ~torch.eye(6, dtype=torch.bool, device=s.device)
    assert torch.equal(s[off], cross[off])
    assert bool((s[off] > 0).all())
    assert torch.equal(s, chamfer_matrix(A))


def _shape_grids(shapes, res=64):
    """[n,4,R,R,R] grids of spheres ('s', radius) and boxes ('b', half size) on the tet vertices (tets_to_3dgrid)."""
    from meshdiffusion_b200.geometry import dmtet, formats
    verts, _ = dmtet.load_tet_grid(res)
    coords = dmtet.grid_coords_of_tet_vertices(verts)
    v = torch.tensor(verts)
    out = []
    for kind, size, centre in shapes:
        p = v - torch.tensor(centre)
        sdf = size - (p.norm(dim=1) if kind == "s" else p.abs().max(dim=1).values)
        out.append(formats.tets_to_3dgrid(coords, torch.sign(sdf), torch.zeros_like(v), res))
    return torch.stack(out)


GEN_SHAPES = [("s", 0.20, (0, 0, 0)), ("s", 0.31, (0.02, 0, 0)), ("b", 0.15, (0, 0, 0)), ("b", 0.26, (0, 0.03, 0)),
              ("s", 0.40, (0, 0, 0.01))]
REF_SHAPES = [("s", 0.24, (0, 0, 0)), ("b", 0.21, (0.01, 0, 0)), ("s", 0.35, (0, 0, 0)), ("b", 0.12, (0, 0, 0)),
              ("b", 0.32, (0, 0, 0.02)), ("s", 0.16, (0, 0.01, 0))]


def test_metrics_on_synthetic_shape_sets_match_the_oracle():
    from meshdiffusion_b200.diffusion.gen_metrics import generation_metrics
    from meshdiffusion_b200.geometry.pointcloud import grids_to_point_clouds
    gen, ge = grids_to_point_clouds(_shape_grids(GEN_SHAPES).cuda(), 64, 512, seed=3)
    ref, re_ = grids_to_point_clouds(_shape_grids(REF_SHAPES).cuda(), 64, 512, seed=3)
    assert not ge.any().item() and not re_.any().item()
    got = generation_metrics(gen, ref)
    g, r = gen.cpu().numpy(), ref.cpu().numpy()
    want = pco.metrics(pco.chamfer_matrix(g, r), pco.chamfer_matrix(g), pco.chamfer_matrix(r))
    for k in ("cov_cd", "1nna_cd", "1nna_cd_gen", "1nna_cd_ref"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert abs(got["mmd_cd"] - want["mmd_cd"]) <= 1e-6 * want["mmd_cd"]
    assert 0 < got["cov_cd"] <= 1 and got["mmd_cd"] > 0


def test_eval_metrics_command_line(tmp_path, monkeypatch):
    """The same shape files as the generated and the reference set: MMD = 0, COV = 1 and 1-NNA = 0 exactly."""
    import main_diffusion
    monkeypatch.chdir(tmp_path)
    shapes = GEN_SHAPES[:4]
    grids = _shape_grids(shapes).numpy()
    empty = np.zeros_like(grids[0])
    empty[0] = -1.0  # every vertex outside: no surface
    eval_dir = tmp_path / "samples"
    eval_dir.mkdir()
    paths = []
    for k, g in enumerate(list(grids) + [empty]):
        p = str(eval_dir / f"shape_{k}.npy")
        np.save(p, g)
        paths.append(p)
    meta = tmp_path / "list.json"
    meta.write_text(json.dumps(sorted(paths)))
    main_diffusion.main([f"--config={ROOT}/configs/res64.py", "--mode=eval_metrics", f"--config.eval.eval_dir={eval_dir}",
                         f"--config.data.meta_path={meta}", "--config.data.extension=npy", "--config.eval.metric_points=256"])
    m = json.loads((eval_dir / "metrics.json").read_text())
    for k in ("mmd_cd", "cov_cd", "1nna_cd", "1nna_cd_gen", "1nna_cd_ref", "n_gen", "n_ref", "n_empty_gen", "n_empty_ref",
              "n_points", "seed", "cd_convention", "sample_seconds", "matrix_seconds"):
        assert k in m, k
    assert m["n_gen"] == m["n_ref"] == 4 and m["n_empty_gen"] == m["n_empty_ref"] == 1
    assert m["n_points"] == 256 and m["seed"] == 42
    assert m["mmd_cd"] == 0.0 and m["cov_cd"] == 1.0 and m["1nna_cd"] == 0.0
    assert m["1nna_cd_gen"] == 0.0 and m["1nna_cd_ref"] == 0.0
