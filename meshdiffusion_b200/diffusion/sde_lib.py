"""VP-SDE used by the sampler and the DDPM loss (reference: lib/diffusion/sde_lib.py:176-233).

Host-side plumbing: the tables are tiny (N floats). They are built with the same torch operations, in the same
order and on the same device as the reference does, so per-step coefficients are bit-identical to it.
"""
import numpy as np
import torch


class VPSDE:
    def __init__(self, beta_min=0.1, beta_max=20, N=1000, device=None):
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        self.N = N
        self.beta_0, self.beta_1 = beta_min, beta_max
        self.discrete_betas = torch.linspace(beta_min / N, beta_max / N, N).to(device)
        self.alphas = 1.0 - self.discrete_betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.alphas_cumprod_ext = torch.cat([torch.tensor([1.0 - 1e-4]).to(device), self.alphas_cumprod], dim=0)
        self.sqrt_alphas_cumprod = torch.sqrt(self.alphas_cumprod)
        self.sqrt_1m_alphas_cumprod = torch.sqrt(1.0 - self.alphas_cumprod)

    @property
    def T(self):
        return 1

    def sde(self, x, t):
        beta_t = self.beta_0 + t * (self.beta_1 - self.beta_0)
        return -0.5 * beta_t[:, None, None, None, None] * x, torch.sqrt(beta_t)

    def marginal_prob(self, x, t):
        log_mean_coeff = -0.25 * t ** 2 * (self.beta_1 - self.beta_0) - 0.5 * t * self.beta_0
        return torch.exp(log_mean_coeff[:, None, None, None, None]) * x, torch.sqrt(1.0 - torch.exp(2.0 * log_mean_coeff))

    def prior_sampling(self, shape, generator=None):
        return torch.randn(*shape, generator=generator)

    def prior_logp(self, z):
        n = np.prod(z.shape[1:])
        return -n / 2.0 * np.log(2 * np.pi) - torch.sum(z ** 2, dim=(1, 2, 3, 4)) / 2.0

    def discretize(self, x, t):
        step = (t * (self.N - 1) / self.T).long()
        beta = self.discrete_betas.to(x.device)[step]
        alpha = self.alphas.to(x.device)[step]
        return torch.sqrt(alpha)[:, None, None, None, None] * x - x, torch.sqrt(beta)
