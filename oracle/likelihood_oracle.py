"""ORACLE support for the probability-flow likelihood (diffusion/likelihood.py): small torch score models whose
answers are known, shared by the golden generator (oracle/make_likelihood_golden.py, which feeds them to the unmodified
reference `get_likelihood_fn`) and by the tests (which feed them to ours)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

R, C, B = 4, 4, 2  # stub grid: [B][C][R][R][R]


class StubScore(torch.nn.Module):
    """eps(x, labels) = tanh(conv3d(x, W, 3^3, pad 1) + b * labels / 1000): a dense, non-diagonal Jacobian in x."""

    def __init__(self, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.w = torch.nn.Parameter(torch.randn(C, C, 3, 3, 3, generator=g) * 0.1)
        self.b = torch.nn.Parameter(torch.randn(C, generator=g) * 0.1)

    def forward(self, x, labels):
        h = F.conv3d(x, self.w, padding=1) + self.b[None, :, None, None, None] * (labels / 1000.0)[:, None, None, None, None]
        return torch.tanh(h)


class GaussianEps(torch.nn.Module):
    """The exact eps-prediction for data ~ N(0, sigma^2 I) diffused by the VP-SDE: x_t ~ N(0, (a^2 sigma^2 + s^2) I) with
    (a, s) = marginal_prob(t), score = -x / (a^2 sigma^2 + s^2) = -eps / s. Diagonal Jacobian, so the Rademacher
    Hutchinson estimate of the divergence is exact. Computed in fp64, returned in fp32."""

    def __init__(self, sigma, beta_min=0.1, beta_max=20.0, N=1000):
        super().__init__()
        self.sigma, self.b0, self.b1, self.N = sigma, beta_min, beta_max, N

    def forward(self, x, labels):
        t = labels.double() / (self.N - 1)
        lmc = -0.25 * t ** 2 * (self.b1 - self.b0) - 0.5 * t * self.b0
        a2 = torch.exp(2.0 * lmc)[:, None, None, None, None]
        s2 = 1.0 - a2
        return (torch.sqrt(s2) * x.double() / (a2 * self.sigma ** 2 + s2)).float()


def gaussian_bpd(x, sigma, mask=None):
    """-log N(x; 0, sigma^2 I) / (D ln 2) per sample, over the entries where mask != 0 (all when None)."""
    x = np.asarray(x, np.float64).reshape(x.shape[0], -1)
    keep = np.ones(x.shape[1], bool) if mask is None else np.broadcast_to(np.asarray(mask).reshape(1, -1) != 0,
                                                                         (x.shape[1] // np.asarray(mask).size, np.asarray(mask).size)).reshape(-1)
    xs = x[:, keep]
    D = xs.shape[1]
    logp = -0.5 * D * math.log(2 * math.pi * sigma ** 2) - np.sum(xs ** 2, axis=1) / (2 * sigma ** 2)
    return -logp / (D * math.log(2))


def stub_data(seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, C, R, R, R, generator=g) * 0.5
