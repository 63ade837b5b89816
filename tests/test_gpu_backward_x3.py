"""Split-bf16 (bf16x3) training plan on the GPU: the weight-gradient kernel, the data-gradient convolutions, GroupNorm
backward and the whole score-network backward against torch autograd in true fp32 on UNROUNDED fp32 inputs (the
reference trains in fp32: lib/diffusion/losses.py:104-139). Every operand is a (hi, lo) bf16 pair and every product
hi*hi + hi*lo + lo*hi, so the gradients are fp32-class; a single leftover bf16 rounding on a gradient path shows up here
as an error of 1e-3 .. 1e-2.
"""
import pytest
import torch
import torch.nn.functional as F

from helpers import build_model, ddpm_loss, rel_max, tiny_config
from oracle import synth, unet_oracle
from test_gpu_backward import CONV_CASES

pytestmark = pytest.mark.gpu


def _fp32_autograd():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _x3_config(name="res64", dropout=0.0):
    cfg = tiny_config(name, "bf16x3")
    cfg.training.compute_dtype = "bf16x3"
    cfg.model.dropout = dropout
    return cfg


@pytest.mark.parametrize("B,Cin,Cout,R,k,stride", CONV_CASES)
def test_conv3d_backward_x3(B, Cin, Cout, R, k, stride):
    from meshdiffusion_b200 import ops
    _fp32_autograd()
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Cin + R)
    x = torch.randn(B, Cin, R, R, R, device="cuda", generator=g).requires_grad_(True)
    w = (torch.randn(Cout, Cin, k, k, k, device="cuda", generator=g) / (Cin * k ** 3) ** 0.5).requires_grad_(True)
    if stride == 1:
        y = F.conv3d(x, w, None, padding=k // 2)
    else:
        y = F.conv3d(F.pad(x, (0, 1, 0, 1, 0, 1)), w, None, stride=2)
    dy = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(dy)
    want_dx = stride == 1
    dw, dx = ops.conv3d_backward(ops.to_ndhwc(dy, "bf16x3"), ops.to_ndhwc(x.detach(), "bf16x3"), w.detach(), stride=stride,
                                 want_dx=want_dx, precision="bf16x3")
    e_w = rel_max(dw, w.grad)
    msg = f"x3 wgrad B{B} {Cin}->{Cout} R{R} k{k} s{stride}: max {e_w:.3e}"
    if want_dx:
        e_x = rel_max(ops.from_ndhwc(dx, "bf16x3"), x.grad)
        msg += f"; dgrad max {e_x:.3e}"
        assert e_x < 1e-4
    print(msg)
    assert e_w < 1e-4


@pytest.mark.parametrize("C,R,B,silu,with_add", [(128, 16, 2, True, False), (32, 8, 3, True, True), (384, 8, 2, False, True), (1024, 4, 2, True, False)])
def test_groupnorm_act_backward_x3(C, R, B, silu, with_add):
    from meshdiffusion_b200 import ops
    _fp32_autograd()
    g = torch.Generator(device="cuda").manual_seed(C + R)
    x = (torch.randn(B, C, R, R, R, device="cuda", generator=g) * 1.5 + 0.3).requires_grad_(True)
    gamma = (torch.rand(C, device="cuda", generator=g) + 0.5).requires_grad_(True)
    beta = (torch.randn(C, device="cuda", generator=g) * 0.1).requires_grad_(True)
    y = F.group_norm(x, 32, gamma, beta, eps=1e-6)
    if silu:
        y = F.silu(y)
    da = torch.randn(y.shape, device="cuda", generator=g)
    y.backward(da)
    add = torch.randn(x.shape, device="cuda", generator=g) if with_add else None
    xl = ops.to_ndhwc(x.detach(), "bf16x3")
    xd = x.detach().double().permute(0, 2, 3, 4, 1).reshape(B, -1, C)
    stats = torch.stack([xd.sum(1), (xd * xd).sum(1)], dim=-1)
    dx, dg, db = ops.groupnorm_act_backward(xl, stats, gamma.detach(), beta.detach(), ops.to_ndhwc(da, "bf16x3"),
                                            ops.to_ndhwc(add, "bf16x3") if with_add else None, silu=silu, precision="bf16x3")
    ref_dx = x.grad + (add if with_add else 0)
    e = rel_max(ops.from_ndhwc(dx, "bf16x3"), ref_dx)
    eg, eb = rel_max(dg, gamma.grad), rel_max(db, beta.grad)
    print(f"x3 gn bwd C{C} R{R}: dx {e:.3e} dgamma {eg:.3e} dbeta {eb:.3e}")
    assert e < 1e-4 and eg < 1e-4 and eb < 1e-4


def _oracle_grads(cfg, sd, x, labels, noise, mask):
    _fp32_autograd()
    sdg = {k: (v.cuda().clone().requires_grad_(True) if v.dtype == torch.float32 and k not in ("mask", "coords") else v.cuda()) for k, v in sd.items()}
    loss = ddpm_loss(unet_oracle.unet_forward(sdg, unet_oracle.arch_from_config(cfg), x, labels), noise, mask)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in sdg.items() if v.dtype == torch.float32 and v.requires_grad and v.grad is not None}


def _compare(ours, ref):
    """(global rel-L2, (worst tensor, its rel-L2)) over tensors whose reference gradient does not vanish; tensors whose true
    gradient vanishes (pos_layer.weight, the attention key bias) must come out negligible."""
    rows, tot_num, tot_den = [], 0.0, 0.0
    for n, gr in ref.items():
        if n not in ours:
            continue
        num = (ours[n] - gr).double().pow(2).sum().item()
        den = gr.double().pow(2).sum().item()
        tot_num += num; tot_den += den
        rows.append((n, num, den, ours[n].double().pow(2).sum().item()))
    worst = ("", 0.0)
    for n, num, den, mine in rows:
        if den < 1e-10 * tot_den:
            assert mine < 1e-8 * tot_den, f"{n}: gradient should vanish, got norm^2 {mine:.3e} of {tot_den:.3e}"
            continue
        e = (num / den) ** 0.5
        if e > worst[1]:
            worst = (n, e)
    return (tot_num / tot_den) ** 0.5, worst


@pytest.mark.parametrize("name", ["res64", "res128"])
def test_unet_backward_x3_matches_autograd(name):
    cfg = _x3_config(name)
    model, sd = build_model(cfg, "cuda:0", 21)
    net = model.module
    R, B = cfg.data.image_size, 2
    x, labels = synth.synthetic_inputs(R, B, 31, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    noise = torch.randn(x.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    mask = sd["mask"].cuda().view(1, 1, R, R, R)
    ref_loss, ref = _oracle_grads(cfg, sd, x, labels, noise, mask)
    net.train()
    loss = ddpm_loss(model(x, labels), noise, mask)
    loss.backward()
    ours = {n: p.grad for n, p in net.named_parameters() if p.grad is not None}
    glob, worst = _compare(ours, ref)
    dl = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
    print(f"{name} x3: loss rel diff {dl:.3e}; global rel-l2 {glob:.3e}, worst {worst[0]} {worst[1]:.3e}")
    assert dl < 1e-4
    assert glob < 1e-3 and worst[1] < 1e-2


@pytest.mark.parametrize("name", ["res64", "res128"])
def test_unet_backward_x3_matches_reference_golden(name):
    """Engine gradients vs the signatures of the REFERENCE modules' own loss.backward() on CPU fp32, with tolerances 10x
    tighter than the bf16 plan's golden test."""
    import numpy as np
    from helpers import grad_signature, load_golden
    gold = load_golden(f"unet_tiny_{name}_grads.npz")
    cfg = _x3_config(name)
    model, sd = build_model(cfg, "cuda:0", int(gold["state_seed"]))
    net = model.module
    net.train()
    R = cfg.data.image_size
    x, labels = synth.synthetic_inputs(R, 2, int(gold["input_seed"]), sd["mask"])
    noise = torch.randn(x.shape, generator=torch.Generator().manual_seed(int(gold["noise_seed"]))).cuda()
    loss = ddpm_loss(model(x.cuda(), labels.cuda()), noise, sd["mask"].cuda().view(1, 1, R, R, R))
    loss.backward()
    print(f"{name} x3: loss {loss.item():.6f} vs reference {float(gold['loss']):.6f}")
    assert abs(loss.item() - float(gold["loss"])) < 2e-3 * float(gold["loss"])
    tot = float(gold["total_norm"])
    params = dict(net.named_parameters())
    worst = 0.0
    for n, sig in zip(gold["names"], gold["sig"]):
        got = grad_signature(str(n), params[str(n)].grad)
        tol = 4 * (0.005 * sig[0] + 2e-4 * tot)
        assert abs(got[0] - sig[0]) < 0.01 * sig[0] + 2e-4 * tot, f"{n}: norm {got[0]:.4e} vs {sig[0]:.4e}"
        assert np.abs(got[1:] - sig[1:]).max() < tol, f"{n}: projections {got[1:]} vs {sig[1:]}"
        worst = max(worst, np.abs(got[1:] - sig[1:]).max() / tot)
    print(f"{name} x3: {len(gold['names'])} tensors, worst projection error / |g| {worst:.3e}")


def test_res64_full_backward_x3_vs_autograd():
    """Full-size res64 network, B = 1: every gradient tensor against fp32 autograd through the oracle."""
    from helpers import full_config
    cfg = full_config("res64", "bf16x3")
    cfg.training.compute_dtype = "bf16x3"
    cfg.model.dropout = 0.0
    model, sd = build_model(cfg, "cuda:0", 5)
    net = model.module
    net.train()
    R = 64
    x, labels = synth.synthetic_inputs(R, 1, 6, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    noise = torch.randn(x.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    mask = sd["mask"].cuda().view(1, 1, R, R, R)
    loss = ddpm_loss(model(x, labels), noise, mask)
    loss.backward()
    ours = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
    net.release_engine()
    torch.cuda.empty_cache()
    ref_loss, ref = _oracle_grads(cfg, sd, x, labels, noise, mask)
    glob, worst = _compare(ours, ref)
    print(f"res64 full x3: loss {loss.item():.6f} vs {ref_loss.item():.6f}; global rel-l2 {glob:.3e}, worst {worst[0]} {worst[1]:.3e}")
    assert glob < 2e-3


def test_unet_backward_x3_accumulates_and_is_deterministic():
    cfg = _x3_config()
    model, sd = build_model(cfg, "cuda:0", 3)
    net = model.module
    net.train()
    x, labels = synth.synthetic_inputs(16, 2, 8, sd["mask"])
    x, labels = x.cuda(), labels.cuda()

    def run():
        model(x, labels).square().mean().backward()

    run()
    g1 = net._flat_grad.clone()
    for p in net.parameters():
        p.grad = None
    run()
    assert torch.equal(g1, net._flat_grad), "gradients differ run to run"
    run()  # second micro-batch without zero_grad: accumulation
    assert torch.allclose(net._flat_grad, 2 * g1, rtol=1e-5, atol=1e-8)


def test_x3_dropout_gradients_fused_vs_two_pass(monkeypatch):
    """The dropout mask of the split-bf16 forward (norm/act kernel), the two-pass GroupNorm backward and the fused GEMM
    epilogue agree: fused and two-pass engines give the same gradients, which differ from the no-dropout ones."""
    R, B = 16, 2

    def grads(fused, p):
        monkeypatch.setenv("MDB_GNB", "1" if fused else "0")
        torch.manual_seed(1234)  # the dropout seed derives from torch.initial_seed() and a per-model call counter
        model, sd = build_model(_x3_config(dropout=p), "cuda:0", 3)
        net = model.module
        net.train()
        x, labels = synth.synthetic_inputs(R, B, 8, sd["mask"])
        model(x.cuda(), labels.cuda()).square().mean().backward()
        g = net._flat_grad.clone()
        net.release_engine()
        return g

    g_fused, g_two = grads(True, 0.3), grads(False, 0.3)
    g_none = grads(True, 0.0)
    rel = (g_fused - g_two).norm().item() / g_two.norm().item()
    away = (g_fused - g_none).norm().item() / g_none.norm().item()
    print(f"x3 fused vs two-pass under dropout: rel-l2 {rel:.3e}; dropout vs none: {away:.3e}")
    assert rel < 1e-4
    assert away > 5e-2


def test_x3_backward_with_smaller_runtime_batch():
    """An engine planned for 4 and run on 2 gives the gradients of an engine planned for 2."""
    R = 16

    def run(first_batch):
        model, sd = build_model(_x3_config(), "cuda:0", 3)
        net = model.module
        net.train()
        x, labels = synth.synthetic_inputs(R, 4, 8, sd["mask"])
        x, labels = x.cuda(), labels.cuda()
        if first_batch == 4:
            model(x, labels).square().mean().backward()
            for p in net.parameters():
                p.grad = None
        model(x[:2].contiguous(), labels[:2].contiguous()).square().mean().backward()
        g = net._flat_grad.clone()
        net.release_engine()
        return g

    g4, g2 = run(4), run(2)
    rel = (g4 - g2).norm().item() / g2.norm().item()
    print(f"x3 planned-4 vs planned-2 engines on a batch of 2: rel-l2 {rel:.3e}")
    assert rel < 1e-4


def test_x3_loss_curve_tracks_fp32_reference():
    """20 Adam steps on the tiny network, dropout off, same data / labels / noise: the split-bf16 engine tracks fp32
    autograd through the oracle (the bf16 plan's gate is 5e-2)."""
    _fp32_autograd()
    cfg = _x3_config()
    model, sd = build_model(cfg, "cuda:0", 13)
    net = model.module
    net.train()
    R, B, steps = 16, 4, 20
    mask = sd["mask"].cuda().view(1, 1, R, R, R)
    arch = unet_oracle.arch_from_config(cfg)
    ref_sd = {k: (v.cuda().clone().requires_grad_(True) if v.dtype == torch.float32 and k not in ("mask", "coords") else v.cuda()) for k, v in sd.items()}
    ref_params = [v for v in ref_sd.values() if v.requires_grad]
    opt_ref = torch.optim.Adam(ref_params, lr=2e-4, betas=(0.9, 0.999), eps=1e-8)
    opt = torch.optim.Adam([p for p in net.parameters() if p.requires_grad], lr=2e-4, betas=(0.9, 0.999), eps=1e-8)
    g = torch.Generator(device="cuda").manual_seed(4)
    data = (torch.rand(B, 4, R, R, R, device="cuda", generator=g) * 2 - 1) * mask
    ours, theirs = [], []
    for it in range(steps):
        labels = torch.randint(0, 1000, (B,), device="cuda", generator=g).float()
        noise = torch.randn(data.shape, device="cuda", generator=g)
        x = (0.7 * data + 0.7 * noise) * mask
        opt_ref.zero_grad()
        lr_ = ddpm_loss(unet_oracle.unet_forward(ref_sd, arch, x, labels), noise, mask)
        lr_.backward()
        torch.nn.utils.clip_grad_norm_(ref_params, 1.0)
        opt_ref.step()
        opt.zero_grad()
        lo = ddpm_loss(model(x, labels), noise, mask)
        lo.backward()
        torch.nn.utils.clip_grad_norm_([p for p in net.parameters() if p.requires_grad], 1.0)
        opt.step()
        ours.append(lo.item()); theirs.append(lr_.item())
    rel = max(abs(a - b) / abs(b) for a, b in zip(ours, theirs))
    print(f"x3 max relative loss difference over {steps} steps: {rel:.3e}")
    assert rel < 2e-3
    assert theirs[-1] < theirs[0]


def test_x3_trainer_end_to_end(tmp_path, monkeypatch):
    """trainer.train with training.compute_dtype='bf16x3' on the tiny network: the loop runs, writes a checkpoint in the
    usual layout, and the inference engine restores it."""
    import os
    from meshdiffusion_b200.diffusion import trainer
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from meshdiffusion_b200.diffusion.utils import restore_checkpoint
    from meshdiffusion_b200.diffusion.models.ema import ExponentialMovingAverage
    cfg = _x3_config(dropout=0.1)
    cfg.device = torch.device("cuda:0")
    cfg.training.train_dir = wd = os.path.join(tmp_path, "run")
    cfg.data.synthetic = True
    cfg.training.batch_size, cfg.training.n_iters, cfg.training.log_freq = 2, 2, 1
    cfg.training.snapshot_freq_for_preemption, cfg.training.snapshot_freq = 1, 100000
    # the tet grids ship for 64^3 / 128^3 only: the 16^3 test network trains on the full grid with uniform synthetic data
    monkeypatch.setattr(trainer, "load_grid_mask", lambda R, device: torch.ones(R, R, R, device=device))
    monkeypatch.setattr(trainer, "synthetic_grids",
                        lambda batch, R, device, generator=None: torch.rand(batch, 4, R, R, R, device=device, generator=generator) * 2 - 1)
    trainer.train(cfg)
    ck = torch.load(os.path.join(wd, "checkpoints", "checkpoint_2.pth"), map_location="cpu", weights_only=False)
    assert set(ck.keys()) == {"optimizer", "model", "ema", "step"}
    assert all(k.startswith("module.") for k in ck["model"])
    assert all(torch.isfinite(v).all() for v in ck["model"].values() if v.is_floating_point())
    model = mutils.create_model(cfg)
    state = dict(optimizer=torch.optim.Adam(model.parameters()), model=model,
                 ema=ExponentialMovingAverage(model.parameters(), decay=cfg.model.ema_rate), step=0)
    state = restore_checkpoint(os.path.join(wd, "checkpoints", "checkpoint_2.pth"), state, cfg.device, strict=True)
    net = state["model"].module
    for k, v in ck["model"].items():
        assert torch.equal(net.state_dict()[k[len("module."):]].cpu(), v), k
    model.eval()
    x = torch.randn(2, 4, 16, 16, 16, device="cuda")
    with torch.no_grad():
        out = model(x, torch.tensor([10.0, 500.0], device="cuda"))
    assert out.shape == x.shape and torch.isfinite(out).all()
