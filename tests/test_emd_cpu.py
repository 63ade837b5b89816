"""CPU: the Earth Mover's distance oracle (oracle/emd_oracle.py). The exact solver on cases whose answers are known by
construction, the float32 auction restatement of the device kernel against it, the metric reductions keyed by distance,
and the `--config.eval.metric_emd` command line."""
import numpy as np
import pytest

from helpers import ROOT
from oracle import emd_oracle as eo
from oracle import pc_metrics_oracle as pco


def test_exact_emd_of_two_single_points_is_their_distance():
    x, y = np.array([[0.0, 1.0, 2.0]]), np.array([[3.0, 5.0, 2.0]])
    assert eo.emd_exact(x, y) == 5.0


def test_exact_emd_of_a_permuted_copy_is_zero():
    x = np.random.RandomState(0).rand(50, 3)
    assert eo.emd_exact(x, x[np.random.RandomState(1).permutation(50)]) == 0.0


def test_exact_emd_of_a_translated_copy_is_the_translation():
    # sum_i |x_i - y_pi(i)| >= |sum_i (x_i - y_pi(i))| = N |t| by the triangle inequality, and the identity reaches it
    x = np.random.RandomState(2).rand(40, 3)
    t = np.array([0.3, -0.4, 1.2])
    assert eo.emd_exact(x, x + t) == pytest.approx(np.linalg.norm(t), rel=1e-12)


def test_exact_emd_of_a_hand_solved_three_point_case():
    # points on a line: x = 0, 1, 2 and y = 1.5, 2.5, 10. Sorted matching is optimal in 1-D: |0-1.5| + |1-2.5| + |2-10|
    x = np.array([[0.0, 0, 0], [1.0, 0, 0], [2.0, 0, 0]])
    y = np.array([[10.0, 0, 0], [1.5, 0, 0], [2.5, 0, 0]])
    assert eo.emd_exact(x, y) == pytest.approx((1.5 + 1.5 + 8.0) / 3, rel=1e-15)


def test_unequal_sizes_are_rejected():
    with pytest.raises(ValueError):
        eo.emd_exact(np.zeros((3, 3)), np.zeros((4, 3)))
    with pytest.raises(ValueError):
        eo.emd_auction(np.zeros((3, 3)), np.zeros((4, 3)))


def _surface(n, seed, radius=0.35):
    """Points near a sphere of unit-scale size, as sampled shapes are (nearest-neighbour spacing ~ 1e-2 at n = 512)."""
    rng = np.random.RandomState(seed)
    x = rng.randn(n, 3)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return (x * radius * (1 + 0.3 * rng.rand(1, 3)) + 0.05 * rng.randn(1, 3) + 0.003 * rng.randn(n, 3)).astype(np.float32)


def _random(n, seed):
    return (np.random.RandomState(seed).rand(n, 3) - 0.5).astype(np.float32)


def _check_bounds(x, y, eps):
    emd, gap, scan = eo.emd_auction(x, y, eps)
    exact = eo.emd_exact(x, y)
    tol = 1e-6 * exact  # fp32 point distances against fp64 ones
    assert exact - tol <= emd <= exact + eps + tol, (emd, exact)
    assert -1e-12 <= gap <= eps, gap
    assert emd - gap <= exact + tol
    assert scan >= len(x) ** 2 * 2
    return emd, gap


@pytest.mark.parametrize("n", [1, 2, 3, 17, 100, 512])
@pytest.mark.parametrize("kind", ["random", "surface"])
def test_auction_is_within_eps_of_the_exact_optimum(n, kind):
    make = _random if kind == "random" else _surface
    x, y = make(n, n), make(n, n + 1000)
    for eps in (1e-5, 1e-4, 1e-2):
        _check_bounds(x, y, eps)


def test_auction_terminates_on_degenerate_clouds():
    same = np.full((40, 3), 0.25, np.float32)
    emd, gap = _check_bounds(same, same.copy(), 1e-5)
    assert emd == 0.0
    rng = np.random.RandomState(3)
    dup = np.repeat(_random(8, 4), 5, axis=0)[rng.permutation(40)]
    _check_bounds(dup, np.repeat(_random(8, 5), 5, axis=0), 1e-5)
    _check_bounds(dup, dup[rng.permutation(40)], 1e-5)
    _check_bounds(same, dup, 1e-5)


def test_an_eps_below_the_fp32_floor_is_rejected():
    x, y = _random(10, 0), _random(10, 1)
    cmax = float(eo.c_max(x, y))
    with pytest.raises(ValueError, match="fp32"):
        eo.emd_auction(x, y, eps=cmax * eo.FLOOR / 4)
    eo.emd_auction(x, y, eps=cmax * eo.FLOOR * 2)


def test_the_auction_is_symmetric_to_within_eps():
    x, y = _surface(200, 7), _surface(200, 8)
    a, _, _ = eo.emd_auction(x, y, 1e-5)
    b, _, _ = eo.emd_auction(y, x, 1e-5)
    assert abs(a - b) <= 1e-5


def _both(d_gr, d_gg, d_rr, suffix):
    from meshdiffusion_b200.diffusion.gen_metrics import metrics_from_matrices
    want = eo.metrics(d_gr, d_gg, d_rr, suffix=suffix)
    got = metrics_from_matrices(d_gr, d_gg, d_rr, suffix=suffix)
    assert set(got) == set(want)
    assert all(k.endswith(suffix) or k.endswith(suffix + "_gen") or k.endswith(suffix + "_ref") for k in got)
    for k in want:
        assert got[k] == pytest.approx(want[k], rel=1e-12, abs=0), k
    return got


def test_suffixed_metrics_match_the_loop_by_loop_oracle():
    rng = np.random.RandomState(9)
    gen = [_surface(24, s) for s in range(5)]
    ref = [_surface(24, 100 + s) for s in range(4)] + [_random(24, 7)]
    d_gr, _ = eo.emd_matrix(gen, ref)
    d_gg, _ = eo.emd_matrix(gen)
    d_rr, _ = eo.emd_matrix(ref)
    m = _both(d_gr, d_gg, d_rr, "emd")
    assert set(m) == {"mmd_emd", "cov_emd", "1nna_emd", "1nna_emd_gen", "1nna_emd_ref"}
    # ties to the lowest index, as for CD
    d = np.array([[1.0, 2.0], [3.0, 3.0]])
    m = _both(d, np.array([[0.0, 1.0], [1.0, 0.0]]), np.array([[0.0, 1.0], [1.0, 0.0]]), "emd")
    assert m["cov_emd"] == 0.5 and m["1nna_emd"] == 0.75
    # the default suffix returns exactly the Chamfer keys
    from meshdiffusion_b200.diffusion.gen_metrics import metrics_from_matrices
    c = rng.rand(3, 3)
    assert metrics_from_matrices(c, c, c) == pco.metrics(c, c, c)


def test_self_matrix_of_the_oracle_is_symmetric_with_zero_diagonal():
    clouds = [_surface(16, s) for s in range(4)]
    e, g = eo.emd_matrix(clouds)
    assert np.array_equal(e, e.T) and np.array_equal(g, g.T)
    assert np.all(np.diag(e) == 0) and np.all(np.diag(g) == 0)
    exact = eo.emd_exact_matrix(clouds)
    assert np.all(e >= exact - 1e-6 * exact) and np.all(e <= exact + 1e-5 + 1e-6 * exact)


def test_command_line_accepts_metric_emd():
    import main_diffusion
    path, mode, overrides = main_diffusion.parse_args([f"--config={ROOT}/configs/res64.py", "--mode=eval_metrics",
                                                       "--config.eval.eval_dir=/tmp/x", "--config.eval.metric_emd=True"])
    assert mode == "eval_metrics" and ("eval.metric_emd", True) in overrides
