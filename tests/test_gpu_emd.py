"""Earth Mover's distance matrices on the GPU (`emd_matrix`, csrc/emd.cu) against the exact solver and the float32 auction
restatement (oracle/emd_oracle.py), their reproducibility, batch invariance and symmetry, the MMD / COV / 1-NNA metrics
over EMD on synthetic shape sets, and `main_diffusion.py --mode=eval_metrics` with `eval.metric_emd`."""
import json

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import emd_oracle as eo
from oracle import synth

pytestmark = pytest.mark.gpu

EPS = 1e-5


def _mesh_clouds(cases, n_points, seed=0):
    """Surface clouds of clean / noisy synth.synthetic_dmtet marching-tet meshes, [len(cases), n_points, 3] fp32 (CUDA)."""
    from meshdiffusion_b200.geometry import dmtet
    from meshdiffusion_b200.geometry.pointcloud import sample_surface_points
    verts, idx = dmtet.load_tet_grid(64)
    sdfs, poss = zip(*[synth.synthetic_dmtet(verts, seed=s, noisy=n, res=64) for s, n in cases])
    mt = dmtet.MarchingTets(idx, verts.shape[0], max_batch=len(cases))
    v, f, _, _, _, off = mt._extract_raw(torch.tensor(np.stack(poss)).cuda(), torch.tensor(np.stack(sdfs)).cuda())
    pts, empty = sample_surface_points(v, f, off[:, 0], off[:, 1], n_points, seed=seed)
    assert not empty.any().item()
    return pts


def _random_clouds(n, pts, seed):
    return torch.tensor((np.random.RandomState(seed).rand(n, pts, 3) - 0.5).astype(np.float32)).cuda()


def _check_bounds(emd, gap, x, y):
    exact = eo.emd_exact(x, y)
    tol = 1e-6 * exact
    assert exact - tol <= emd <= exact + EPS + tol, (emd, exact)
    assert -1e-12 <= gap <= EPS, gap
    assert emd - gap <= exact + tol


@pytest.mark.parametrize("N", [1, 2, 17, 256, 2048])
def test_entries_are_within_eps_of_the_exact_optimum(N):
    from meshdiffusion_b200.geometry.pointcloud import emd_matrix
    A = torch.cat([_mesh_clouds([(0, False), (1, True)], N, seed=N), _random_clouds(1, N, N)])
    B = torch.cat([_mesh_clouds([(2, True), (3, False)], N, seed=N + 1), _random_clouds(1, N, N + 1)])
    e, g = emd_matrix(A, B, EPS)
    assert e.dtype == torch.float64 and g.dtype == torch.float64 and e.shape == (3, 3)
    e, g, a, b = e.cpu().numpy(), g.cpu().numpy(), A.cpu().numpy(), B.cpu().numpy()
    pairs = [(i, j) for i in range(3) for j in range(3)] if N <= 256 else [(0, 0), (1, 1), (2, 2), (0, 2)]
    for i, j in pairs:
        _check_bounds(e[i, j], g[i, j], a[i], b[j])
        if N <= 256:  # the same decisions as the float32 restatement
            want_e, want_g, _ = eo.emd_auction(a[i], b[j], EPS)
            assert abs(e[i, j] - want_e) <= 1e-12 and abs(g[i, j] - want_g) <= 1e-12, (i, j)


def test_bitwise_reproducible_batch_invariant_and_symmetric_to_eps():
    from meshdiffusion_b200.geometry.pointcloud import emd_matrix
    A = _mesh_clouds([(0, False), (1, True), (4, True)], 700)
    B = torch.cat([_mesh_clouds([(5, False), (6, True)], 700, seed=9), _random_clouds(1, 700, 3)])
    ab, gab = emd_matrix(A, B)
    ab2, gab2 = emd_matrix(A, B)
    assert torch.equal(ab, ab2) and torch.equal(gab, gab2)
    for i, j in ((0, 0), (2, 1), (1, 2)):
        e, g = emd_matrix(A[i:i + 1], B[j:j + 1])
        assert torch.equal(e[0, 0], ab[i, j]) and torch.equal(g[0, 0], gab[i, j])
    ba, _ = emd_matrix(B, A)
    assert float((ab - ba.T).abs().max()) <= EPS


def test_self_matrix_is_symmetric_with_zero_diagonal():
    from meshdiffusion_b200.geometry.pointcloud import emd_matrix
    A = torch.cat([_mesh_clouds([(0, False), (1, True), (2, False)], 300), _random_clouds(2, 300, 4)])
    s, g = emd_matrix(A)
    assert torch.equal(s, s.T) and torch.equal(g, g.T)
    zero = torch.zeros(5, dtype=torch.float64, device=s.device)
    assert torch.equal(torch.diagonal(s), zero) and torch.equal(torch.diagonal(g), zero)
    # the self matrix computes i < j and mirrors it; the cross call's lower triangle solves EMD(A_j, A_i) instead
    cross, _ = emd_matrix(A, A)
    upper = torch.triu(torch.ones(5, 5, dtype=torch.bool, device=s.device), diagonal=1)
    assert torch.equal(s[upper], cross[upper])
    assert float((s - cross).abs().max()) <= EPS
    assert bool((s[upper] > 0).all())


def test_unequal_sizes_and_non_finite_input_raise():
    from meshdiffusion_b200.geometry.pointcloud import emd_matrix
    A, B = _random_clouds(2, 10, 0), _random_clouds(2, 11, 1)
    with pytest.raises(ValueError):
        emd_matrix(A, B)
    bad = A.clone()
    bad[1, 3, 2] = float("nan")
    with pytest.raises(ValueError):
        emd_matrix(bad)
    bad[1, 3, 2] = float("inf")
    with pytest.raises(ValueError):
        emd_matrix(A, bad)
    with pytest.raises(ValueError, match="fp32"):
        emd_matrix(A, eps=1e-9)


def test_degenerate_clouds_finish_within_the_bounds():
    from meshdiffusion_b200.geometry.pointcloud import emd_matrix
    rng = np.random.RandomState(3)
    same = np.full((40, 3), 0.25, np.float32)
    base = (rng.rand(8, 3) - 0.5).astype(np.float32)
    dup = np.repeat(base, 5, axis=0)[rng.permutation(40)]
    dup2 = np.repeat((rng.rand(8, 3) - 0.5).astype(np.float32), 5, axis=0)
    clouds = np.stack([same, dup, dup2, dup[rng.permutation(40)]])
    e, g = emd_matrix(torch.tensor(clouds).cuda(), torch.tensor(clouds[::-1].copy()).cuda())
    e, g = e.cpu().numpy(), g.cpu().numpy()
    rev = clouds[::-1]
    for i in range(4):
        for j in range(4):
            _check_bounds(e[i, j], g[i, j], clouds[i], rev[j])
            want_e, want_g, _ = eo.emd_auction(clouds[i], rev[j], EPS)
            assert abs(e[i, j] - want_e) <= 1e-12 and abs(g[i, j] - want_g) <= 1e-12
    assert e[0, 3] == 0.0  # the all-identical cloud against itself


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


def _min_competitor_margin(d):
    """The smallest difference between a row's minimum and its runner-up (ignoring the +inf diagonal)."""
    s = np.sort(d, axis=1)
    return float((s[:, 1] - s[:, 0]).min())


def test_emd_metrics_on_synthetic_shape_sets_match_the_oracle():
    from meshdiffusion_b200.diffusion.gen_metrics import generation_metrics
    from meshdiffusion_b200.geometry.pointcloud import grids_to_point_clouds
    gen, ge = grids_to_point_clouds(_shape_grids(GEN_SHAPES).cuda(), 64, 256, seed=3)
    ref, re_ = grids_to_point_clouds(_shape_grids(REF_SHAPES).cuda(), 64, 256, seed=3)
    assert not ge.any().item() and not re_.any().item()
    got = generation_metrics(gen, ref, emd=True)
    g, r = gen.cpu().numpy(), ref.cpu().numpy()
    d_gr, d_gg, d_rr = eo.emd_exact_matrix(g, r), eo.emd_exact_matrix(g), eo.emd_exact_matrix(r)
    # the decisions COV and 1-NNA make are separated by more than 2 eps, so the eps-accurate device matrices make the same
    full = np.block([[d_gg, d_gr], [d_gr.T, d_rr]])
    np.fill_diagonal(full, np.inf)
    assert _min_competitor_margin(d_gr) > 2 * EPS and _min_competitor_margin(full) > 2 * EPS
    want = eo.metrics(d_gr, d_gg, d_rr, suffix="emd")
    for k in ("cov_emd", "1nna_emd", "1nna_emd_gen", "1nna_emd_ref"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert -1e-6 * want["mmd_emd"] <= got["mmd_emd"] - want["mmd_emd"] <= EPS + 1e-6 * want["mmd_emd"]
    assert 0 < got["cov_emd"] <= 1 and got["mmd_emd"] > 0
    assert 0 <= got["emd_max_gap"] <= EPS and got["emd_seconds"] > 0
    # the Chamfer keys are unchanged by the flag
    plain = generation_metrics(gen, ref)
    for k in ("mmd_cd", "cov_cd", "1nna_cd", "1nna_cd_gen", "1nna_cd_ref"):
        assert plain[k] == got[k]


def _run_cli(tmp_path, monkeypatch, extra):
    import main_diffusion
    monkeypatch.chdir(tmp_path)
    grids = _shape_grids(GEN_SHAPES[:4]).numpy()
    eval_dir = tmp_path / "samples"
    eval_dir.mkdir()
    paths = []
    for k, g in enumerate(grids):
        p = str(eval_dir / f"shape_{k}.npy")
        np.save(p, g)
        paths.append(p)
    meta = tmp_path / "list.json"
    meta.write_text(json.dumps(sorted(paths)))
    main_diffusion.main([f"--config={ROOT}/configs/res64.py", "--mode=eval_metrics", f"--config.eval.eval_dir={eval_dir}",
                         f"--config.data.meta_path={meta}", "--config.data.extension=npy", "--config.eval.metric_points=256"]
                        + extra)
    return json.loads((eval_dir / "metrics.json").read_text())


CD_KEYS = {"mmd_cd", "cov_cd", "1nna_cd", "1nna_cd_gen", "1nna_cd_ref", "n_gen", "n_ref", "n_empty_gen", "n_empty_ref",
           "n_points", "seed", "cd_convention", "sample_seconds", "matrix_seconds"}
EMD_KEYS = {"mmd_emd", "cov_emd", "1nna_emd", "1nna_emd_gen", "1nna_emd_ref", "emd_convention", "emd_eps", "emd_max_gap",
            "emd_seconds"}


def test_eval_metrics_command_line_with_emd(tmp_path, monkeypatch):
    """The same shape files as both sets: COV-EMD = 1 and 1-NNA-EMD = 0 exactly, MMD-EMD and every gap within eps."""
    from meshdiffusion_b200.geometry.pointcloud import EMD_CONVENTION
    m = _run_cli(tmp_path, monkeypatch, ["--config.eval.metric_emd=True"])
    assert set(m) == CD_KEYS | EMD_KEYS
    assert m["n_gen"] == m["n_ref"] == 4
    assert m["cov_emd"] == 1.0 and m["1nna_emd"] == 0.0 and m["1nna_emd_gen"] == 0.0 and m["1nna_emd_ref"] == 0.0
    assert 0 <= m["mmd_emd"] <= EPS
    assert 0 <= m["emd_max_gap"] <= EPS
    assert m["emd_eps"] == EPS and m["emd_convention"] == EMD_CONVENTION
    assert m["mmd_cd"] == 0.0 and m["cov_cd"] == 1.0 and m["1nna_cd"] == 0.0


def test_eval_metrics_without_the_flag_writes_the_chamfer_keys_only(tmp_path, monkeypatch):
    m = _run_cli(tmp_path, monkeypatch, [])
    assert set(m) == CD_KEYS
