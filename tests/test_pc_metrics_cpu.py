"""CPU: the point-cloud metric oracle (oracle/pc_metrics_oracle.py) on cases whose answers are known by construction, the
host-side metric reductions of diffusion/gen_metrics.py against it, and the `--mode=eval_metrics` command line."""
import numpy as np
import pytest

from helpers import ROOT
from oracle import pc_metrics_oracle as pco


def _clouds(n, pts, seed):
    return np.random.RandomState(seed).rand(n, pts, 3).astype(np.float32)


@pytest.mark.parametrize("n,m", [(1, 1), (17, 40), (300, 257)])
def test_brute_force_chamfer_equals_kdtree(n, m):
    rng = np.random.RandomState(n + m)
    x, y = rng.rand(n, 3), rng.rand(m, 3) * 1.5
    assert pco.chamfer_brute(x, y) == pytest.approx(pco.chamfer_kdtree(x, y), rel=1e-12, abs=1e-15)


def test_chamfer_of_two_single_points_is_twice_their_squared_distance():
    x, y = np.array([[0.0, 1.0, 2.0]]), np.array([[0.5, -1.0, 2.25]])
    d = 0.25 + 4.0 + 0.0625
    assert pco.chamfer_brute(x, y) == 2 * d
    assert pco.chamfer_kdtree(x, y) == pytest.approx(2 * d, rel=1e-15)


def _both(d_gr, d_gg, d_rr):
    from meshdiffusion_b200.diffusion.gen_metrics import metrics_from_matrices
    want = pco.metrics(d_gr, d_gg, d_rr)
    got = metrics_from_matrices(d_gr, d_gg, d_rr)
    assert set(got) == set(want)
    for k in want:
        assert got[k] == pytest.approx(want[k], rel=1e-12, abs=0), k
    return want


def test_a_set_compared_with_itself_scores_perfectly():
    clouds = _clouds(6, 64, 0) + np.arange(6, dtype=np.float32)[:, None, None]  # distinct shapes
    d = pco.chamfer_matrix(clouds)
    assert np.all(np.diag(d) == 0) and np.all(d[~np.eye(6, dtype=bool)] > 0)
    m = _both(d, d, d)
    assert m["mmd_cd"] == 0 and m["cov_cd"] == 1 and m["1nna_cd"] == 0
    assert m["1nna_cd_gen"] == 0 and m["1nna_cd_ref"] == 0


def test_two_well_separated_families_are_told_apart():
    gen = _clouds(5, 32, 1)
    ref = _clouds(4, 32, 2) + np.float32(10.0)
    m = _both(pco.chamfer_matrix(gen, ref), pco.chamfer_matrix(gen), pco.chamfer_matrix(ref))
    assert m["1nna_cd"] == 1 and m["1nna_cd_gen"] == 1 and m["1nna_cd_ref"] == 1


def test_ties_go_to_the_lowest_index():
    # concatenated order [G0, G1, R0, R1]. COV: G1 is equally far from R0 and R1 -> R0, so only R0 is covered.
    # 1-NNA: G0 is equally far from G1 and R0 -> G1 (same set); R0 is equally far from G0 and R1 -> G0 (other set).
    d_gg = np.array([[0.0, 1.0], [1.0, 0.0]])
    d_rr = np.array([[0.0, 1.0], [1.0, 0.0]])
    d_gr = np.array([[1.0, 2.0], [3.0, 3.0]])
    m = _both(d_gr, d_gg, d_rr)
    assert m["cov_cd"] == 0.5
    assert m["mmd_cd"] == 1.5
    assert m["1nna_cd_gen"] == 1.0 and m["1nna_cd_ref"] == 0.5 and m["1nna_cd"] == 0.75


def _mesh():
    # four triangles of areas 0.5, sqrt(6), 0 and 1.5 in one mesh, not all in one plane
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0], [2, 0, 1], [0, 2, 1], [3, 3, 3], [0, 0, 1], [0, 3, 1],
                  [1, 0, 1], [3, 3, 3]], np.float32)
    f = np.array([[0, 1, 2], [3, 4, 5], [6, 6, 6], [7, 9, 8]], np.int64)
    return v, f


def test_sampled_points_lie_on_their_faces():
    v, f = _mesh()
    u = np.random.RandomState(3).rand(4000, 3).astype(np.float32)
    p, face = pco.sample_points(v, f, u)
    assert not np.any(face == 2)  # a zero-area face is never chosen
    a, b, c = (v[f[face, k]].astype(np.float64) for k in range(3))
    n = np.cross(b - a, c - a)
    assert np.abs(((p - a) * n).sum(1)).max() < 1e-12  # in the face's plane
    # barycentric weights of the point are non-negative: inside the triangle
    for e0, e1 in ((a, b), (b, c), (c, a)):
        assert (np.cross(e1 - e0, p - e0) * n).sum(1).min() > -1e-12


def test_face_frequencies_track_area_shares():
    v, f = _mesh()
    areas = pco.face_areas(v, f)
    assert np.allclose(areas, [0.5, np.sqrt(6.0), 0.0, 1.5], rtol=1e-15, atol=0)
    u = np.random.RandomState(4).rand(200000, 3).astype(np.float32)
    _, face = pco.sample_points(v, f, u)
    share = np.bincount(face, minlength=4) / face.size
    assert np.abs(share - areas / areas.sum()).max() < 0.005


def test_empty_and_zero_area_meshes_have_no_points():
    v, f = _mesh()
    assert pco.sample_points(v, f[:0], np.zeros((3, 3), np.float32)) is None
    assert pco.sample_points(v, f[2:3], np.zeros((3, 3), np.float32)) is None


def test_command_line_accepts_eval_metrics():
    import main_diffusion
    path, mode, overrides = main_diffusion.parse_args([f"--config={ROOT}/configs/res64.py", "--mode=eval_metrics",
                                                       "--config.eval.eval_dir=/tmp/x", "--config.eval.metric_points=512"])
    assert mode == "eval_metrics" and ("eval.metric_points", 512) in overrides
