"""Pins diffusion/likelihood.py's generic path against the UNMODIFIED reference `get_likelihood_fn`
(lib/diffusion/likelihood.py:26-113) and writes tests/golden/likelihood_stub.npz.

Run in the authoring container only (needs /root/reference), like oracle/make_golden.py, whose reference import (with the
`ml_collections` stand-in and `Tensor.cuda` neutralised) it reuses:

    python oracle/make_likelihood_golden.py

Exactly ONE thing is substituted: the reference's `get_score_fn` asserts `not continuous` (models/utils.py:183), although
its likelihood.py:61 asks for continuous=True. The substitute is the continuous VP branch
    labels = t (N - 1);  score = -model(x, labels) / std,  std = sde.marginal_prob(0, t)[1]
and is the one diffusion/models/utils.py implements. The score model is oracle/likelihood_oracle.StubScore on CPU fp32.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import likelihood_oracle as lo  # noqa: E402
from oracle.make_golden import GOLD, import_reference  # noqa: E402


def continuous_score_fn(rutils, rsde):
    def get_score_fn(sde, model, train=False, continuous=False, std_scale=True):
        assert continuous and isinstance(sde, rsde.VPSDE) and std_scale
        model_fn = rutils.get_model_fn(model, train=train)

        def score_fn(x, t):
            labels = t * (sde.N - 1)
            score = model_fn(x, labels)
            std = sde.marginal_prob(torch.zeros_like(x), t)[1]
            return -score / std[:, None, None, None, None]

        return score_fn

    return get_score_fn


def main():
    ref = import_reference()
    from lib.diffusion import likelihood as rlik
    rlik.mutils.get_score_fn = continuous_score_fn(ref["rutils"], ref["rsde"])
    sde = ref["rsde"].VPSDE(beta_min=0.1, beta_max=20.0, N=1000)
    model = lo.StubScore(seed=0)
    data = lo.stub_data(seed=1)
    fn = rlik.get_likelihood_fn(sde, lambda x: x, hutchinson_type="Rademacher", rtol=1e-5, atol=1e-5, method="RK45", eps=1e-5)
    torch.manual_seed(7)
    noise = torch.randint_like(data, low=0, high=2).float() * 2 - 1.0  # the draw likelihood_fn makes next
    torch.manual_seed(7)
    bpd, z, nfe = fn(model, data)
    path = os.path.join(GOLD, "likelihood_stub.npz")
    np.savez_compressed(path, data=data.numpy(), noise=noise.numpy(), bpd=bpd.double().numpy(), z=z.numpy(), nfe=np.int64(nfe))
    print(path, "bpd", bpd.tolist(), "nfe", nfe)


if __name__ == "__main__":
    main()
