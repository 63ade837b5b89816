"""Class-conditional score networks and classifier-free guidance, on the CPU: the parameter table, registration order,
checkpoint class counts, the guided eager update, the conditional oracle and an analytic Gaussian gate."""
import numpy as np
import pytest
import torch

from helpers import tiny_config
from oracle import synth, unet_oracle

import class_oracle


def _dpm_sde():
    from meshdiffusion_b200.diffusion import sde_lib
    return sde_lib.VPSDE(0.1, 20.0, 1000, device="cpu")


@pytest.mark.parametrize("name", ["res64", "res128"])
def test_conditional_table_is_unconditional_plus_label_embed(name):
    from meshdiffusion_b200.diffusion.models import ddpm
    cfg = tiny_config(name)
    base = ddpm.arch_from_config(cfg)
    assert base["num_classes"] == 0
    cfg.model.num_classes = 5
    arch = ddpm.arch_from_config(cfg)
    t0, t5 = ddpm.param_table(base), ddpm.param_table(arch)
    assert t5[:-1] == t0
    assert t5[-1] == ("label_embed.weight", (6, 4 * cfg.model.nf))


def test_registration_order_and_zero_init():
    from meshdiffusion_b200.diffusion.models import utils as mutils
    cfg = tiny_config("res64")
    cfg.device = torch.device("cpu")
    torch.manual_seed(0)
    p0 = list(mutils.create_model(cfg).state_dict().items())
    cfg.model.num_classes = 3
    torch.manual_seed(0)
    model = mutils.create_model(cfg)
    p3 = list(model.state_dict().items())
    names = [n for n, _ in model.named_parameters()]
    assert names[-1] == "module.label_embed.weight"
    assert [n for n, _ in p3 if n != "module.label_embed.weight"] == [n for n, _ in p0]
    for (n0, v0), (n3, v3) in zip(p0, p3):
        assert n0 == n3 and torch.equal(v0, v3), n0  # the same draws: the embedding is zero and registered last
    assert torch.equal(model.module.label_embed.weight, torch.zeros(4, 4 * cfg.model.nf))


def test_checkpoint_class_count_mismatch_names_both(tmp_path):
    from meshdiffusion_b200.diffusion import losses
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from meshdiffusion_b200.diffusion.models.ema import ExponentialMovingAverage
    from meshdiffusion_b200.diffusion.utils import restore_checkpoint, save_checkpoint

    def state(k):
        cfg = tiny_config("res64")
        cfg.device = torch.device("cpu")
        cfg.model.num_classes = k
        m = mutils.create_model(cfg)
        return dict(optimizer=losses.get_optimizer(cfg, m.parameters()), model=m,
                    ema=ExponentialMovingAverage(m.parameters(), decay=0.999), step=7)

    path = str(tmp_path / "c.pth")
    save_checkpoint(path, state(2))
    blob = torch.load(path, weights_only=False)
    assert tuple(blob["model"]["module.label_embed.weight"].shape) == (3, 128)
    assert restore_checkpoint(path, state(2), "cpu")["step"] == 7
    for k in (0, 3):
        with pytest.raises(ValueError, match=rf"has 2 classes.*num_classes\) {k}"):
            restore_checkpoint(path, state(k), "cpu")
    with pytest.raises(ValueError, match="has 2 classes"):
        state(0)["model"].load_state_dict(blob["model"], strict=False)


def test_unconditional_model_refuses_class_labels():
    from meshdiffusion_b200.diffusion.models import ddpm
    cfg = tiny_config("res64")
    net = ddpm.ScoreNet(cfg)
    with pytest.raises(ValueError, match="unconditional"):
        net._class_ids(torch.tensor([0]), 1, "cpu")


def test_eager_guided_entry_hand_computed():
    from meshdiffusion_b200.diffusion import sampling
    f = np.float32
    eps_c = torch.tensor([[0.5, -1.25]]).view(1, 1, 2)
    eps_u = torch.tensor([[0.25, 0.75]]).view(1, 1, 2)
    x = torch.tensor([[1.0, -2.0]]).view(1, 1, 2)
    w, sg, ia, cx, c0 = 3.0, 0.5, 2.0, 0.25, 0.75
    row = np.array([0, 10, sg, ia, cx, c0, 0, 0, 0, 0], np.float32)
    h = torch.zeros_like(x)
    out = sampling._update_eager(eps_c, x.clone(), h, torch.ones(1, 1, 2), row, eps_u=eps_u, w=w)
    want = []
    for xv, ec, eu in zip([1.0, -2.0], [0.5, -1.25], [0.25, 0.75]):
        e = f(eu) + f(w) * (f(ec) - f(eu))
        x0 = (f(xv) - f(sg) * e) * f(ia)
        want.append(f(cx) * f(xv) + f(c0) * x0)
    assert out.flatten().tolist() == [float(v) for v in want]   # eps = 1.0 and -5.25: exact in fp32
    assert h.flatten().tolist() == [1.0, 1.25]
    # w = 1 with eps_u is the plain entry on eps_c (eps_u + (eps_c - eps_u) rounds back to eps_c here)
    a = sampling._update_eager(eps_c, x.clone(), torch.zeros_like(x), torch.ones(1, 1, 2), row, eps_u=eps_u, w=1.0)
    b = sampling._update_eager(eps_c, x.clone(), torch.zeros_like(x), torch.ones(1, 1, 2), row)
    assert torch.equal(a, b)


@pytest.mark.parametrize("name", ["res64", "res128"])
def test_conditional_oracle(name):
    from meshdiffusion_b200.diffusion.models import ddpm
    cfg = tiny_config(name)
    arch = unet_oracle.arch_from_config(cfg)
    template = {n: torch.zeros(s) for n, s in ddpm.param_table(ddpm.arch_from_config(cfg))}
    sd = synth.synthetic_state_dict(template, seed=3)
    x, labels = synth.synthetic_inputs(cfg.data.image_size, 3, 4, sd["mask"])
    ref = unet_oracle.unet_forward(sd, arch, x, labels)
    cond = dict(sd, **{"label_embed.weight": torch.zeros(4, 4 * cfg.model.nf)})
    y = torch.tensor([0, 2, 3])
    assert torch.equal(class_oracle.unet_forward(cond, arch, x, labels, y), ref)
    cond["label_embed.weight"] = torch.randn(4, 4 * cfg.model.nf, generator=torch.Generator().manual_seed(1))
    a = class_oracle.unet_forward(cond, arch, x, labels, y)
    assert (a - ref).abs().max() > 1e-3
    # per sample: each row equals the batch-of-one forward at its own class
    for b in range(3):
        one = class_oracle.unet_forward(cond, arch, x[b:b + 1], labels[b:b + 1], y[b:b + 1])
        assert torch.allclose(one, a[b:b + 1], rtol=1e-5, atol=1e-5)
    assert torch.equal(class_oracle.unet_forward(cond, arch, x, labels, None),
                       class_oracle.unet_forward(cond, arch, x, labels, torch.tensor([3, 3, 3])))


class GaussianStub:
    """Exact noise predictions of N(mu_y, I) per class (eps = sigma (x - alpha mu_y)) and, without class_labels, of
    N(0, I) (eps = sigma x). Classifier-free guidance at w then predicts N(w mu_y, I) exactly."""

    def __init__(self, sde, mu):
        self.sde, self.mu = sde, mu

    def __call__(self, x, labels, class_labels=None):
        n = labels.long()
        a = self.sde.sqrt_alphas_cumprod.to(x.device)[n].float().view(-1, 1, 1, 1, 1)
        s = self.sde.sqrt_1m_alphas_cumprod.to(x.device)[n].float().view(-1, 1, 1, 1, 1)
        if class_labels is None:
            return s * x
        mu = self.mu.to(x.device)[torch.as_tensor(class_labels, device=x.device).long()].view(-1, x.shape[1], 1, 1, 1)
        return s * (x - a * mu)


def analytic_gate(device):
    from meshdiffusion_b200.diffusion import sampling
    sde = _dpm_sde()
    mu = torch.tensor([[0.5, -0.25, 0.0, 1.0], [-0.75, 0.5, 0.25, 0.0], [0.0, 0.0, -0.5, 0.5]])
    R, B, w = 16, 6, 2.5
    y = torch.tensor([0, 1, 2, 0, 1, 2])
    torch.manual_seed(0)
    fn = sampling.get_dpm_solver_sampler(sde, (B, 4, R, R, R), lambda v: v, n_steps=25, device=device,
                                         grid_mask=torch.ones(R, R, R, device=device), guidance_scale=w)
    x, nfe = fn(GaussianStub(sde, mu), class_labels=y.to(device))
    assert nfe == 50
    x = x.double().cpu()
    n = R ** 3 * 2  # two samples per class
    for k in range(3):
        s = x[y == k]
        mean = s.mean(dim=(0, 2, 3, 4))
        var = s.var(dim=(0, 2, 3, 4))
        # sampling error of n unit-variance draws (5 sigma) plus the 25-step solver's discretisation error
        assert (mean - w * mu[k].double()).abs().max() < 5 / n ** 0.5 + 5e-3, (k, mean)
        assert (var - 1).abs().max() < 5 * (2 / n) ** 0.5 + 1e-2, (k, var)


def test_analytic_guided_gaussian_cpu():
    analytic_gate("cpu")


def test_guidance_needs_classes_and_pc_refuses_guidance():
    from meshdiffusion_b200.diffusion import sampling
    sde = _dpm_sde()
    stub = GaussianStub(sde, torch.zeros(2, 4))
    fn = sampling.get_dpm_solver_sampler(sde, (1, 4, 4, 4, 4), lambda v: v, n_steps=3, device="cpu",
                                         grid_mask=torch.ones(4, 4, 4), guidance_scale=2.0)
    with pytest.raises(ValueError, match="needs class_labels"):
        fn(stub)
    pc = sampling.get_pc_sampler(sde, (1, 4, 4, 4, 4), sampling.get_predictor("ancestral_sampling"),
                                 sampling.get_corrector("none"), lambda v: v, 0.16, device="cpu",
                                 grid_mask=torch.ones(1, 1, 4, 4, 4))
    with pytest.raises(ValueError, match="guidance_scale = 1"):
        pc(stub, class_labels=torch.tensor([0]), guidance_scale=3.0)


def test_guided_w1_equals_conditional_cpu():
    from meshdiffusion_b200.diffusion import sampling
    sde = _dpm_sde()
    stub = GaussianStub(sde, torch.randn(2, 4, generator=torch.Generator().manual_seed(2)))
    kw = dict(n_steps=5, device="cpu", grid_mask=torch.ones(4, 4, 4))
    x0 = torch.randn(2, 4, 4, 4, 4, generator=torch.Generator().manual_seed(3))
    y = torch.tensor([1, 0])
    a, na = sampling.get_dpm_solver_sampler(sde, (2, 4, 4, 4, 4), lambda v: v, **kw)(stub, x0=x0, class_labels=y)
    b, nb = sampling.get_dpm_solver_sampler(sde, (2, 4, 4, 4, 4), lambda v: v, guidance_scale=1.0, **kw)(
        lambda x, l: stub(x, l, class_labels=y), x0=x0)
    assert torch.equal(a, b) and na == nb == 5
