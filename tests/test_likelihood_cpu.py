"""Probability-flow likelihood (diffusion/likelihood.py) without a GPU: the generic path against the reference's own
`get_likelihood_fn` (tests/golden/likelihood_stub.npz, oracle/make_likelihood_golden.py), against a Gaussian whose
log-density is known in closed form, the continuous VP score function, and the command-line plumbing."""
import numpy as np
import pytest
import torch

from helpers import GOLD, load_golden, tiny_config  # noqa: F401
from oracle import likelihood_oracle as lo
from meshdiffusion_b200.diffusion import likelihood, sde_lib
from meshdiffusion_b200.diffusion.models import utils as mutils


def _sde():
    return sde_lib.VPSDE(beta_min=0.1, beta_max=20.0, N=1000, device="cpu")


def test_generic_path_reproduces_reference_golden():
    g = load_golden("likelihood_stub.npz")
    fn = likelihood.get_likelihood_fn(_sde(), lambda x: x, hutchinson_type="Rademacher", rtol=1e-5, atol=1e-5, eps=1e-5)
    bpd, z, nfe = fn(lo.StubScore(seed=0), torch.from_numpy(g["data"]), noise=torch.from_numpy(g["noise"]))
    assert nfe == int(g["nfe"])
    np.testing.assert_allclose(bpd.double().numpy(), g["bpd"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(z.numpy(), g["z"], rtol=1e-12, atol=0)


# residual of the closed-form check, measured: 8.8e-6 (unmasked) and 1.4e-5 (masked) absolute bpd, with nfe 50. It comes
# from stopping at t = eps instead of 0, from the prior mismatch at t = 1 and from rtol / atol = 1e-5.
_GAUSS_TOL = 5e-5


@pytest.mark.parametrize("masked", [False, True])
def test_gaussian_data_bpd_is_known_by_construction(masked):
    sigma = 0.5
    data = lo.stub_data(seed=3)
    mask = None
    if masked:
        mask = (torch.rand(lo.R, lo.R, lo.R, generator=torch.Generator().manual_seed(5)) < 0.4).float()
        data = data * mask
    fn = likelihood.get_likelihood_fn(_sde(), lambda x: x + 8.0, rtol=1e-5, atol=1e-5, eps=1e-5, grid_mask=mask)
    noise = likelihood.hutchinson_noise(data, "Rademacher", generator=torch.Generator().manual_seed(9))
    bpd, z, nfe = fn(lo.GaussianEps(sigma), data, noise=noise)  # inverse_scaler(-1) = 7: zero dequantisation offset
    want = lo.gaussian_bpd(data.numpy(), sigma, None if mask is None else mask.numpy())
    resid = np.abs(bpd.double().numpy() - want).max()
    print(f"gaussian bpd residual ({'masked' if masked else 'unmasked'}): {resid:.2e}, nfe {nfe}")
    assert resid < _GAUSS_TOL
    if masked:
        assert torch.all(z.reshape(lo.B, lo.C, -1)[:, :, mask.reshape(-1) == 0] == 0)


def test_continuous_score_fn_matches_formula():
    sde = _sde()
    model = lo.StubScore(seed=2)
    x = lo.stub_data(seed=4)
    t = torch.tensor([0.3, 0.77])
    got = mutils.get_score_fn(sde, model, train=False, continuous=True)(x, t)
    lmc = -0.25 * t ** 2 * (sde.beta_1 - sde.beta_0) - 0.5 * t * sde.beta_0
    std = torch.sqrt(1.0 - torch.exp(2.0 * lmc))
    want = -model(x, t * (sde.N - 1)) / std[:, None, None, None, None]
    assert torch.equal(got, want)
    # the discrete form is unchanged: the sqrt(1 - alpha_bar) table at labels.long()
    got_d = mutils.get_score_fn(sde, model, train=False, continuous=False)(x, t)
    want_d = -model(x, t * (sde.N - 1)) / sde.sqrt_1m_alphas_cumprod[(t * (sde.N - 1)).long()][:, None, None, None, None]
    assert torch.equal(got_d, want_d)


def test_eval_likelihood_mode_parses():
    import main_diffusion
    import os
    from helpers import ROOT
    _, mode, ov = main_diffusion.parse_args([f"--config={os.path.join(ROOT, 'configs', 'res64.py')}", "--mode=eval_likelihood",
                                             "--config.eval.likelihood_rtol=1e-4"])
    assert mode == "eval_likelihood" and ov == [("eval.likelihood_rtol", 1e-4)]


def test_tf32_differentiable_path_is_refused():
    from meshdiffusion_b200.diffusion.models import ddpm
    net = ddpm.ScoreNet(tiny_config("res64", "tf32"))
    net.eval()
    x = torch.zeros(1, 4, 16, 16, 16, requires_grad=True)
    with pytest.raises(ValueError, match="bf16"):
        net(x, torch.zeros(1))
