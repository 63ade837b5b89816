"""CPU: the DPM-Solver++(2M) sampler (`sampling.method='dpm_solver'`) -- its label grid and step table, and the eager
fp32 update run against an analytic Gaussian model whose exact probability-flow endpoint and marginals are known."""
import math

import numpy as np
import pytest
import torch

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from meshdiffusion_b200.diffusion import sampling, sde_lib

MU, S = 0.3, 0.5
SHAPE = (2, 4, 30, 30, 30)  # 216 000 elements


def _sde():
    return sde_lib.VPSDE(0.1, 20.0, 1000, device="cpu")


def _tables(sde):
    abar = sde.alphas_cumprod.double().cpu().numpy()
    return np.sqrt(abar), np.sqrt(1.0 - abar)


class GaussianEps:
    """Exact noise prediction when every element of x0 is N(MU, S^2) and independent:
    eps*(x, n) = sigma_n (x - alpha_n MU) / (alpha_n^2 S^2 + sigma_n^2), evaluated in float64, returned in float32."""

    def __init__(self, sde):
        self.alpha, self.sigma = _tables(sde)
        self.calls = []

    def __call__(self, x, labels):
        n = int(labels[0].item())
        assert labels.dtype == torch.float32 and torch.all(labels == n), "labels must be one integer per call"
        self.calls.append((n, x.clone()))
        a, s = self.alpha[n], self.sigma[n]
        xd = x.double()
        return (s * (xd - a * MU) / (a * a * S * S + s * s)).float()


def _sampler(sde, K, stochastic=False, mask=None, shape=SHAPE, denoise=True):
    if mask is None:
        mask = torch.ones(1, *shape[2:])
    return sampling.get_dpm_solver_sampler(sde, shape, lambda x: x, n_steps=K, stochastic=stochastic, denoise=denoise,
                                           device="cpu", grid_mask=mask)


def _ode_error(sde, K, seed=0):
    alpha, sigma = _tables(sde)
    torch.manual_seed(seed)
    xT = torch.randn(SHAPE).double()
    torch.manual_seed(seed)  # the sampler draws the same prior
    out, nfe = _sampler(sde, K)(GaussianEps(sde))
    T = sde.N - 1
    exact = alpha[0] * MU + math.sqrt(alpha[0] ** 2 * S * S + sigma[0] ** 2) * (xT - alpha[T] * MU) / math.sqrt(
        alpha[T] ** 2 * S * S + sigma[T] ** 2)
    return (out.double() - exact).abs().max().item(), nfe


def test_label_grid():
    sde = _sde()
    for K in range(2, 101):
        labels, table = sampling.dpm_solver_schedule(sde, K)
        assert labels[0] == sde.N - 1 and labels[-1] == 0
        assert all(a > b for a, b in zip(labels, labels[1:]))
        assert table.shape == (len(labels) - 1, 9) and np.array_equal(table[:, 0], labels[:-1])
        K_eff = len(labels) - 1
        if K <= 37:
            assert K_eff == K, K
        else:
            assert K_eff < K, K
    for bad in (0, 1, -3, 2.5, True):
        with pytest.raises(ValueError):
            sampling.dpm_solver_schedule(sde, bad)


def test_first_step_is_ddim():
    sde = _sde()
    alpha, sigma = _tables(sde)
    g = np.random.default_rng(0)
    x, eps = g.standard_normal(1000), g.standard_normal(1000)
    for K in (2, 16, 25, 50):
        labels, table = sampling.dpm_solver_schedule(sde, K)
        n, label_sigma, inv_alpha, c_x, c_0, c_1, c_z, coef, std = table[0]
        assert c_1 == 0.0 and c_z == 0.0 and n == sde.N - 1
        a, b = labels[0], labels[1]
        assert label_sigma == sigma[a] and coef == alpha[b] and std == sigma[b]
        x0 = (x - label_sigma * eps) * inv_alpha
        dpm = c_x * x + c_0 * x0
        ddim = alpha[b] * (x - sigma[a] * eps) / alpha[a] + sigma[b] * eps
        assert np.abs(dpm - ddim).max() < 1e-12
        assert np.all(table[1:, 5] != 0.0), "every later step is second order"


def test_sde_table_noise():
    sde = _sde()
    _, table = sampling.dpm_solver_schedule(sde, 25, stochastic=True, denoise=True)
    assert np.all(table[:-1, 6] > 0) and table[-1, 6] == 0.0
    _, table = sampling.dpm_solver_schedule(sde, 25, stochastic=True, denoise=False)
    assert np.all(table[:, 6] > 0)
    _, table = sampling.dpm_solver_schedule(sde, 25, stochastic=False)
    assert np.all(table[:, 6] == 0)


def test_ode_against_analytic_gaussian():
    sde = _sde()
    errs = {}
    for K in (16, 25, 32):
        errs[K], nfe = _ode_error(sde, K)
        assert nfe == K
    order = math.log2(errs[16] / errs[32])
    print("ODE max error", errs, "order 16->32 %.2f" % order)
    assert errs[32] < 2.5e-2
    assert order > 1.6
    assert errs[16] > errs[25] > errs[32]


def test_sde_marginal_against_analytic_gaussian():
    sde = _sde()
    alpha, sigma = _tables(sde)
    torch.manual_seed(3)
    out, nfe = _sampler(sde, 50, stochastic=True)(GaussianEps(sde))
    assert nfe == 49
    mean, var = out.double().mean().item(), out.double().var().item()
    exact_var = alpha[0] ** 2 * S * S + sigma[0] ** 2
    print("SDE K=50: mean %.5f (exact %.5f), var %.5f (exact %.5f)" % (mean, alpha[0] * MU, var, exact_var))
    assert abs(mean - alpha[0] * MU) < 5e-3
    assert abs(var / exact_var - 1.0) < 3e-2


def _mask(R, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(1, R, R, R, generator=g) < 0.4).float()


@pytest.mark.parametrize("stochastic", [False, True])
def test_output_vanishes_outside_mask(stochastic):
    sde = _sde()
    R = 12
    mask = _mask(R, 1)
    torch.manual_seed(0)
    out, _ = _sampler(sde, 8, stochastic, mask=mask, shape=(2, 4, R, R, R))(GaussianEps(sde))
    assert torch.isfinite(out).all()
    assert torch.all(out[:, :, mask[0] == 0] == 0)
    assert torch.all(out[:, :, mask[0] == 1] != 0)


@pytest.mark.parametrize("stochastic", [False, True])
@pytest.mark.parametrize("freeze_iters", [None, 600])
def test_conditioning_replaces_channel(monkeypatch, stochastic, freeze_iters):
    """Channel c at pm = 1 holds alpha * partial + sigma * z, with the alpha, sigma of the label the model sees next and the
    per-sample noise drawn for that replacement, before step 0 and after every conditioned step."""
    sde = _sde()
    R, B, c, K = 10, 2, 1, 10
    shape = (B, 4, R, R, R)
    mask = _mask(R, 2)
    g = torch.Generator().manual_seed(4)
    partial = torch.sign(torch.randn(1, 4, R, R, R, generator=g))
    pmask = (torch.rand(1, 4, R, R, R, generator=g) < 0.5).float()
    labels, table = sampling.dpm_solver_schedule(sde, K, stochastic)
    rows = table.astype(np.float32)
    draws = []
    real = torch.randn_like

    def record(t, **kw):
        z = real(t, **kw)
        if tuple(t.shape) == (B, R, R, R):
            draws.append(z.clone())
        return z

    monkeypatch.setattr(torch, "randn_like", record)
    model = GaussianEps(sde)
    torch.manual_seed(5)
    out, nfe = _sampler(sde, K, stochastic, mask=mask, shape=shape)(model, partial=partial, partial_mask=pmask,
                                                                     partial_channel=c, freeze_iters=freeze_iters)
    assert nfe == K and [n for n, _ in model.calls] == labels[:-1]
    limit = sde.N + 10 if freeze_iters is None else freeze_iters
    cond_until = sum(1 for k in range(K - 1) if sde.N - 1 - labels[k] < limit)
    assert 0 < cond_until <= K - 1
    assert len(draws) == 1 + cond_until, "one replacement draw before step 0 and one per conditioned step, no more"
    alpha, sigma = _tables(sde)
    live = (pmask[0, c] == 1) & (mask[0] == 1)
    for k in range(cond_until + 1):
        if k == 0:
            coef, std = float(np.float32(alpha[-1])), float(np.float32(sigma[-1]))
        else:
            coef, std = float(rows[k - 1, 7]), float(rows[k - 1, 8])
        want = partial[:, c] * coef + draws[k] * std
        got = model.calls[k][1][:, c]
        assert torch.equal(got[:, live], want[:, live]), f"step {k}"
        assert torch.all(got[:, mask[0] == 0] == 0)
    assert torch.all(out[:, :, mask[0] == 0] == 0)


def test_eager_entry_keeps_network_x0():
    """The x0 history receives the network's prediction, not the replaced channel."""
    sde = _sde()
    R, B, c = 6, 2, 0
    g = torch.Generator().manual_seed(6)
    x, eps = torch.randn(B, 4, R, R, R, generator=g), torch.randn(B, 4, R, R, R, generator=g)
    mask = torch.ones(R, R, R)
    partial = torch.randn(1, 4, R, R, R, generator=g)
    pmask = torch.ones(1, 4, R, R, R)
    known = sampling._Known(partial, pmask[:, c], [c], B)
    _, table = sampling.dpm_solver_schedule(sde, 10)
    row = sampling._rows32(table)[3]
    hist = torch.randn(B, 4, R, R, R, generator=g)
    z2 = torch.randn(B, 4, R, R, R, generator=g)
    x0 = (x - eps * float(row[2])) * float(row[3])
    xn = sampling._update_eager(eps, x.clone(), hist, mask, row, known=known, known_noise=z2)
    assert torch.equal(hist, x0)
    assert torch.equal(xn[:, c], partial[:, c] * float(row[8]) + z2[:, c] * float(row[9]))


def test_get_sampling_fn_dispatches_dpm_solver():
    from configs import res64
    sde = _sde()
    cfg = res64.get_config()
    cfg.device = "cpu"
    cfg.sampling.method = "dpm_solver"
    R = 8
    shape = (2, 4, R, R, R)
    mask = torch.ones(1, R, R, R)
    for K, sde_form in ((6, False), (40, True)):
        cfg.sampling.dpm_steps, cfg.sampling.dpm_sde = K, sde_form
        fn = sampling.get_sampling_fn(cfg, sde, shape, lambda x: x, 1e-3, grid_mask=mask)
        model = GaussianEps(sde)
        out, nfe = fn(model)
        labels, _ = sampling.dpm_solver_schedule(sde, K)
        assert nfe == len(labels) - 1 == len(model.calls) and out.shape == shape
    del cfg.sampling["dpm_steps"], cfg.sampling["dpm_sde"]
    out, nfe = sampling.get_sampling_fn(cfg, sde, shape, lambda x: x, 1e-3, grid_mask=mask)(GaussianEps(sde))
    assert nfe == 25
    cfg.sampling.dpm_steps = 1
    with pytest.raises(ValueError):
        sampling.get_sampling_fn(cfg, sde, shape, lambda x: x, 1e-3, grid_mask=mask)
