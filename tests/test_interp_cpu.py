"""CPU: shape interpolation (`--mode=uncond_gen_interp`) -- the inversion schedule of DPM-Solver++(2M), the inverse map on an
analytic Gaussian model whose exact probability-flow latent is known, the sampler's `x0=` start, the slerp oracle
against the reference's own `slerp` (golden), and the driver's argument checks."""
import json
import math

import numpy as np
import pytest
import torch

from helpers import GOLD, ROOT  # noqa: F401  (puts the repository on sys.path)
from meshdiffusion_b200.diffusion import sampling, sde_lib
from oracle import interp_oracle

MU, S = 0.3, 0.5
SHAPE = (2, 4, 16, 16, 16)


def _sde():
    return sde_lib.VPSDE(0.1, 20.0, 1000, device="cpu")


def _tables(sde):
    abar = sde.alphas_cumprod.double().cpu().numpy()
    return np.sqrt(abar), np.sqrt(1.0 - abar)


class GaussianEps:
    """Exact noise prediction when every element of the data is independent N(MU, S^2):
    eps*(x, n) = sigma_n (x - alpha_n MU) / (alpha_n^2 S^2 + sigma_n^2), in float64, returned in float32."""

    def __init__(self, sde):
        self.alpha, self.sigma = _tables(sde)
        self.calls = []

    def __call__(self, x, labels):
        n = int(labels[0].item())
        assert labels.dtype == torch.float32 and torch.all(labels == n), "labels must be one integer per call"
        self.calls.append((n, x.clone()))
        a, s = self.alpha[n], self.sigma[n]
        return (s * (x.double() - a * MU) / (a * a * S * S + s * s)).float().to(x.device)


def _rel_l2(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm()).item()


def gaussian_inversion_errors(K, device="cpu"):
    """(latent vs the exact ODE latent, decode(encode(x)) vs x), both rel-L2, for x drawn from the model's label-0
    marginal (seed 0). The exact latent is the affine map of the probability-flow ODE between the marginals
    N(alpha_n MU, alpha_n^2 S^2 + sigma_n^2) at labels 0 and N - 1."""
    sde = _sde()
    alpha, sigma = _tables(sde)
    T = sde.N - 1
    g = torch.Generator().manual_seed(0)
    s0 = math.sqrt(alpha[0] ** 2 * S * S + sigma[0] ** 2)
    x = (alpha[0] * MU + s0 * torch.randn(SHAPE, generator=g, dtype=torch.float64)).float()
    exact = alpha[T] * MU + math.sqrt(alpha[T] ** 2 * S * S + sigma[T] ** 2) * (x.double() - alpha[0] * MU) / s0
    mask = torch.ones(1, *SHAPE[2:], device=device)
    invert = sampling.get_dpm_solver_inverter(sde, SHAPE, K, grid_mask=mask, device=device)
    z, nfe = invert(GaussianEps(sde), x.to(device))
    labels, _ = sampling.dpm_solver_schedule(sde, K)
    assert nfe == len(labels) - 1 and z.device.type == torch.device(device).type
    sample = sampling.get_dpm_solver_sampler(sde, SHAPE, lambda t: t, n_steps=K, device=device, grid_mask=mask)
    y, _ = sample(GaussianEps(sde), x0=z)
    return _rel_l2(z, exact), _rel_l2(y, x)


@pytest.mark.parametrize("K", [2, 10, 25, 50, 100])
def test_inversion_schedule(K):
    sde = _sde()
    alpha, sigma = _tables(sde)
    lam = np.log(alpha) - np.log(sigma)
    fwd, _ = sampling.dpm_solver_schedule(sde, K)
    labels, table = sampling.dpm_solver_inversion_schedule(sde, K)
    assert labels == fwd[::-1] and labels[0] == 0 and labels[-1] == sde.N - 1
    assert table.shape == (len(labels) - 1, 9) and table.dtype == np.float64
    h_prev = None
    for k, row in enumerate(table):
        s, t = labels[k], labels[k + 1]
        h = lam[t] - lam[s]
        assert h < 0
        b = -alpha[t] * np.expm1(-h)
        if k == 0:
            c_0, c_1 = b, 0.0
        else:
            r = h_prev / h
            c_0, c_1 = b * (1.0 + 1.0 / (2.0 * r)), -b / (2.0 * r)
        want = (s, sigma[s], 1.0 / alpha[s], sigma[t] / sigma[s], c_0, c_1, 0.0)
        assert np.array_equal(row[:7], np.array(want)), k
        h_prev = h
    assert table[0, 5] == 0.0 and np.all(table[:, 6] == 0.0)


def test_inversion_against_analytic_gaussian():
    e25, r25 = gaussian_inversion_errors(25)
    e50, r50 = gaussian_inversion_errors(50)
    print(f"inversion: latent rel-L2 K=25 {e25:.3e}, K=50 {e50:.3e} (ratio {e25 / e50:.2f}); "
          f"round trip K=25 {r25:.3e}, K=50 {r50:.3e}")
    assert e25 <= 1.2e-2 and e50 <= 3e-3 and e25 / e50 >= 3.0
    assert r25 <= 5e-4 and r50 <= 5e-5


def test_sampler_starts_from_x0():
    sde = _sde()
    R = 8
    shape = (2, 4, R, R, R)
    g = torch.Generator().manual_seed(1)
    mask = (torch.rand(1, R, R, R, generator=g) < 0.5).float()
    x0 = torch.randn(shape, generator=g)
    fn = sampling.get_dpm_solver_sampler(sde, shape, lambda t: t, n_steps=6, device="cpu", grid_mask=mask)
    model = GaussianEps(sde)
    state = torch.random.get_rng_state()
    out, nfe = fn(model, x0=x0)
    assert torch.equal(torch.random.get_rng_state(), state), "x0= must not draw a prior"
    assert nfe == 6 and torch.equal(model.calls[0][1], x0 * mask)
    # without x0 the sampler draws its prior as before: the same as passing that draw
    torch.manual_seed(7)
    a, _ = fn(GaussianEps(sde))
    torch.manual_seed(7)
    b, _ = fn(GaussianEps(sde), x0=sde.prior_sampling(shape))
    assert torch.equal(a, b)
    with pytest.raises(ValueError):
        fn(GaussianEps(sde), x0=x0[:1])


def test_oracle_matches_reference_golden():
    gold = np.load(f"{GOLD}/slerp_reference.npz")
    stride = int(gold["stride"])
    for p in range(gold["za"].shape[0]):
        a, b = gold["za"][p].astype(np.float32), gold["zb"][p].astype(np.float32)
        frames, coef, sums = interp_oracle.slerp_frames(a, b, gold["alphas"])
        want = gold["frames"][p]
        got = frames.reshape(frames.shape[0], -1)[:, ::stride]
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 5e-7, (p, err)
        theta = math.acos(sums[0] / math.sqrt(sums[1] * sums[2]))
        assert abs(theta - gold["theta"][p]) < 1e-6
        assert np.array_equal(coef[0], [1.0, 0.0]) and np.array_equal(coef[-1], [0.0, 1.0])
        assert np.array_equal(frames[0], a) and np.array_equal(frames[-1], b)


def test_oracle_degenerate_endpoints_lerp():
    g = np.random.default_rng(3)
    a = g.standard_normal(100).astype(np.float32)
    alphas = np.linspace(0.0, 1.0, 5)
    for b in (a.copy(), -a, np.zeros_like(a)):
        frames, coef, _ = interp_oracle.slerp_frames(a, b, alphas)
        assert np.all(np.isfinite(frames))
        assert np.array_equal(coef, np.stack([1.0 - alphas, alphas], 1).astype(np.float32))


# ---- driver and command line --------------------------------------------------------------------------------------
def _config(tmp_path, **eval_kw):
    from configs import res64
    cfg = res64.get_config()
    cfg.device = "cpu"
    cfg.eval.eval_dir = str(tmp_path / "out")
    cfg.eval.ckpt_path = str(tmp_path / "missing.pth")
    cfg.eval.batch_size = 4
    cfg.sampling.method = "dpm_solver"
    for k, v in eval_kw.items():
        cfg.eval[k] = v
    return cfg


@pytest.fixture
def no_model(monkeypatch):
    """Fails the test if the driver gets as far as building a network."""
    from meshdiffusion_b200.diffusion import interp

    def refuse(config):
        raise AssertionError("the driver built a model before checking its arguments")
    monkeypatch.setattr(interp, "_setup", refuse)
    return interp


@pytest.mark.parametrize("case", ["one_frame", "frames_not_int", "pc", "dpm_sde", "shapes_with_ddim", "bad_steps",
                                  "bad_pairs", "index_out_of_range", "malformed_shapes"])
def test_driver_rejects_bad_arguments(tmp_path, no_model, case):
    cfg = _config(tmp_path)
    meta = tmp_path / "list.json"
    meta.write_text(json.dumps([str(tmp_path / f"shape_{k}.npy") for k in range(3)]))
    cfg.data.meta_path = str(meta)
    cfg.data.extension = "npy"
    if case == "one_frame":
        cfg.eval.batch_size = 1
    elif case == "frames_not_int":
        cfg.eval.batch_size = 2.5
    elif case == "pc":
        cfg.sampling.method = "pc"
    elif case == "dpm_sde":
        cfg.sampling.dpm_sde = True
    elif case == "shapes_with_ddim":
        cfg.sampling.method = "ddim"
        cfg.eval.interp_shapes = ((0, 1),)
    elif case == "bad_steps":
        cfg.sampling.dpm_steps = 1
    elif case == "bad_pairs":
        cfg.eval.interp_pairs = 0
    elif case == "index_out_of_range":
        cfg.eval.interp_shapes = ((0, 1), (2, 3))
    elif case == "malformed_shapes":
        cfg.eval.interp_shapes = ((0, 1, 2),)
    with pytest.raises(ValueError):
        no_model.uncond_gen_interp(cfg)


def test_driver_accepts_valid_arguments_up_to_the_model(tmp_path, no_model):
    """Valid noise and shape configurations pass every check and reach the model build."""
    meta = tmp_path / "list.json"
    meta.write_text(json.dumps([str(tmp_path / f"shape_{k}.npy") for k in range(3)]))
    for kw, method in (({}, "dpm_solver"), ({}, "ddim"), ({"interp_shapes": ((0, 2), (1, 1))}, "dpm_solver")):
        cfg = _config(tmp_path, **kw)
        cfg.sampling.method = method
        cfg.data.meta_path = str(meta)
        cfg.data.extension = "npy"
        with pytest.raises(AssertionError, match="built a model"):
            no_model.uncond_gen_interp(cfg)


def test_command_line_accepts_the_mode():
    import main_diffusion
    path, mode, overrides = main_diffusion.parse_args(
        ["--config=configs/res64.py", "--mode=uncond_gen_interp", "--config.eval.interp_shapes=((0, 1),)",
         "--config.eval.interp_pairs=3"])
    assert mode == "uncond_gen_interp" and path == "configs/res64.py"
    assert ("eval.interp_shapes", ((0, 1),)) in overrides and ("eval.interp_pairs", 3) in overrides


def test_prior_sampling_generator():
    sde = _sde()
    a = sde.prior_sampling((2, 3), generator=torch.Generator().manual_seed(5))
    b = sde.prior_sampling((2, 3), generator=torch.Generator().manual_seed(5))
    torch.manual_seed(5)
    assert torch.equal(a, b) and torch.equal(a, sde.prior_sampling((2, 3)))
