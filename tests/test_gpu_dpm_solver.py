"""DPM-Solver++(2M) on the GPU: mdb_solver_update bit-exact against the eager fp32 update, its in-kernel Philox noise,
mdb_solver_run bit-exact against the step-by-step public path, the analytic-Gaussian gates through the kernel path, and
`main_diffusion.py --config.sampling.method=dpm_solver` end to end."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, build_model, full_config, tiny_config
from test_dpm_solver_cpu import MU, S, SHAPE, GaussianEps, _tables
from test_gpu_cli import _run

pytestmark = pytest.mark.gpu


def _sde(device="cuda"):
    from meshdiffusion_b200.diffusion import sde_lib
    return sde_lib.VPSDE(0.1, 20.0, 1000, device=device)


@pytest.mark.parametrize("conditional", [False, True])
@pytest.mark.parametrize("kind", ["first_order", "second_order", "sde"])
def test_entry_kernel_matches_eager(kind, conditional):
    from meshdiffusion_b200.diffusion import sampling
    sde = _sde("cpu")
    _, table = sampling.dpm_solver_schedule(sde, 20, stochastic=(kind == "sde"))
    k = 0 if kind == "first_order" else 7
    rows32, entries_c = sampling._rows32(table), sampling._entries_c(table)
    g = torch.Generator().manual_seed(11 + k)
    B, R, c = 3, 16, 2
    x = torch.randn(B, 4, R, R, R, generator=g)
    eps, hist, z = (torch.randn(B, 4, R, R, R, generator=g) for _ in range(3))
    z2 = torch.zeros(B, 4, R, R, R)
    z2[:, c] = torch.randn(B, R, R, R, generator=g)
    mask = (torch.rand(R, R, R, generator=g) < 0.4).float()
    known = known_cpu = None
    if conditional:
        partial = torch.sign(torch.randn(1, 4, R, R, R, generator=g))
        pmask = (torch.rand(B, 4, R, R, R, generator=g) < 0.5).float()
        known_cpu = sampling._Known(partial, pmask[:, c], [c], B)
        known = sampling._Known(partial.cuda(), pmask[:, c].cuda(), [c], B)
    xe, he = x.clone(), hist.clone()
    sampling._update_eager(eps, xe, he, mask, rows32[k], z, known_cpu, z2)
    xg, hg = x.cuda(), hist.cuda()
    sampling._update(eps.cuda(), xg, hg, mask.cuda().reshape(-1), entries_c[k], z.cuda(), known,
                     z2.cuda() if conditional else None)
    assert torch.equal(xg.cpu(), xe), f"{kind}: x differs from the eager update"
    assert torch.equal(hg.cpu(), he), f"{kind}: x0 history differs from the eager update"
    assert torch.all(xe[:, :, mask == 0] == 0)


def test_entry_in_kernel_noise():
    """noise=NULL: z from Philox(seed, element, offset). A step with c_z = 1 and every other coefficient 0 writes z * g."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion import sampling
    B, R = 4, 32
    mask = torch.ones(R, R, R, device="cuda")
    mask[:, :, : R // 2] = 0
    zeros = torch.zeros(B, 4, R, R, R, device="cuda")
    row = _native.SolverEntryC(0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0)

    def draw(seed, step):
        x = zeros.clone()
        sampling._update(zeros, x, torch.empty_like(x), mask.reshape(-1), row, seed=seed, offset=4 * step)
        assert torch.all(x[..., : R // 2] == 0)
        return x[..., R // 2:]

    z0, z1 = draw(1234, 0), draw(1234, 1)
    for z in (z0, z1):
        assert abs(z.mean().item()) < 0.01 and abs(z.var().item() - 1.0) < 0.02
    assert abs((z0 * z1).mean().item()) < 0.01, "noise of consecutive steps is correlated"
    assert torch.equal(draw(1234, 0), z0), "the same (seed, step) must reproduce the same noise"
    assert not torch.equal(draw(1235, 0), z0)


@pytest.mark.parametrize("stochastic", [False, True])
@pytest.mark.parametrize("conditional", [False, True])
@pytest.mark.parametrize("precision", ["bf16", "tf32", "bf16x3"])
@pytest.mark.parametrize("size", ["tiny", "res64"])
def test_device_loop_matches_stepwise(size, precision, conditional, stochastic):
    """mdb_solver_run(seed, step0, n) is bitwise equal to n x [model(x, label) + mdb_solver_update(noise=NULL, seed,
    offset=4*k)] through the public entry points, with and without the replacement of channel 0 of a partial grid."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion import sampling
    cfg = tiny_config("res64", precision) if size == "tiny" else full_config("res64", precision)
    B, n, step0, seed = (3, 5, 2, 77) if size == "tiny" else (2, 3, 6, 78)
    model, sd = build_model(cfg, "cuda:0", 21)
    net = model.module
    R = cfg.data.image_size
    sde = _sde()
    labels, table = sampling.dpm_solver_schedule(sde, 12, stochastic=stochastic)
    entries_c = sampling._entries_c(table)
    mask = sd["mask"].view(-1).cuda().contiguous()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x0 = (torch.randn(B, 4, R, R, R, device="cuda", generator=g) * mask.view(R, R, R)).contiguous()
    h0 = torch.randn(B, 4, R, R, R, device="cuda", generator=g)
    known = None
    if conditional:
        partial = torch.sign(torch.randn(1, 1, R, R, R, device="cuda", generator=g))
        pmask = (torch.rand(1, 1, R, R, R, device="cuda", generator=g) < 0.5).float()
        known = sampling._Known(partial, pmask[:, 0], [0], B)
    until = step0 + n - 1  # the last step runs without the replacement
    with torch.no_grad():
        xa, ha = x0.clone(), h0.clone()
        sampling._native_run(net, xa, ha, mask, entries_c, seed, step0, n, known, until)
        xb, hb = x0.clone(), h0.clone()
        L = _native.lib()
        for k in range(step0, step0 + n):
            eps = model(xb, torch.full((B,), float(labels[k]), device="cuda"))
            ks = known.struct() if (known is not None and k < until) else None
            _native.check(L.mdb_solver_update(_native.ptr(eps), _native.ptr(xb), _native.ptr(hb), _native.ptr(mask),
                                              ctypes.byref(entries_c[k]), R ** 3, 4, B, None, seed, 4 * k,
                                              ctypes.byref(ks) if ks is not None else None, _native.current_stream()))
    assert torch.isfinite(xa).all()
    assert torch.equal(xa, xb) and torch.equal(ha, hb), "mdb_solver_run differs from the step-by-step public path"
    if conditional:
        assert not torch.equal(xa[:, 0], x0[:, 0])


def _gpu_sampler(sde, K, stochastic):
    from meshdiffusion_b200.diffusion import sampling
    return sampling.get_dpm_solver_sampler(sde, SHAPE, lambda x: x, n_steps=K, stochastic=stochastic, device="cuda",
                                           grid_mask=torch.ones(1, *SHAPE[2:], device="cuda"))


def test_analytic_gaussian_through_kernel_path():
    """The CPU gates of the ODE and the SDE, with the analytic model on CUDA: every step runs mdb_solver_update."""
    sde = _sde()
    alpha, sigma = _tables(sde)
    T = sde.N - 1
    errs = {}
    for K in (16, 25, 32):
        torch.manual_seed(0)
        xT = torch.randn(SHAPE).double()
        torch.manual_seed(0)
        out, nfe = _gpu_sampler(sde, K, False)(GaussianEps(sde))
        assert out.is_cuda and nfe == K
        exact = alpha[0] * MU + math.sqrt(alpha[0] ** 2 * S * S + sigma[0] ** 2) * (xT - alpha[T] * MU) / math.sqrt(
            alpha[T] ** 2 * S * S + sigma[T] ** 2)
        errs[K] = (out.cpu().double() - exact).abs().max().item()
    order = math.log2(errs[16] / errs[32])
    print("GPU ODE max error", errs, "order %.2f" % order)
    assert errs[32] < 2.5e-2 and order > 1.6 and errs[16] > errs[25] > errs[32]
    torch.manual_seed(3)
    out, nfe = _gpu_sampler(sde, 50, True)(GaussianEps(sde))
    mean, var = out.double().mean().item(), out.double().var().item()
    exact_var = alpha[0] ** 2 * S * S + sigma[0] ** 2
    print("GPU SDE K=50: mean %.5f var %.5f (exact %.5f %.5f)" % (mean, var, alpha[0] * MU, exact_var))
    assert nfe == 49 and abs(mean - alpha[0] * MU) < 5e-3 and abs(var / exact_var - 1.0) < 3e-2


def test_public_sampler_native_loop_on_score_network():
    """native_rng + a native ScoreNet: the whole loop runs in mdb_solver_run; same seed, same samples; zero off the mask."""
    from meshdiffusion_b200.diffusion import sampling
    cfg = tiny_config("res64", "bf16")
    model, sd = build_model(cfg, "cuda:0", 21)
    R, B = 16, 2
    sde = _sde()
    mask = sd["mask"].view(1, R, R, R).cuda()
    cfg.sampling.method, cfg.sampling.dpm_steps, cfg.sampling.dpm_sde, cfg.sampling.native_rng = "dpm_solver", 6, True, True
    fn = sampling.get_sampling_fn(cfg, sde, (B, 4, R, R, R), lambda x: x, 1e-3, grid_mask=mask)
    outs = []
    for _ in range(2):
        torch.manual_seed(8)
        out, nfe = fn(model)
        outs.append(out)
    assert nfe == 6 and torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])
    assert torch.all(outs[0][:, :, mask[0] == 0] == 0)


def _cli(tmp_path, name, mode, extra):
    out = os.path.join(tmp_path, name)
    _run([f"--config={ROOT}/configs/res64.py", f"--mode={mode}", f"--config.eval.eval_dir={out}",
          f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth", "--config.model.compute_dtype=bf16",
          "--config.sampling.method=dpm_solver", "--config.sampling.dpm_steps=4"] + extra, cwd=str(tmp_path))
    return np.load(os.path.join(out, "0.npy"))


def test_uncond_and_cond_gen_cli(tmp_path):
    from meshdiffusion_b200.geometry import dmtet
    m = dmtet.grid_mask_from_tets(64).numpy()
    sde_args = ["--config.sampling.dpm_sde=True", "--config.sampling.native_rng=True", "--config.eval.batch_size=1"]
    a = _cli(tmp_path, "a", "uncond_gen", sde_args + ["--config.seed=1"])
    b = _cli(tmp_path, "b", "uncond_gen", sde_args + ["--config.seed=1"])
    c = _cli(tmp_path, "c", "uncond_gen", sde_args + ["--config.seed=2"])
    for x in (a, c):
        assert x.shape == (1, 4, 64, 64, 64) and x.dtype == np.float32 and np.isfinite(x).all()
        assert np.all(x[:, :, m == 0] == 0)
    assert np.array_equal(a, b), "same seed, different samples"
    assert not np.array_equal(a, c), "different seeds, same samples"

    verts, _ = dmtet.load_tet_grid(64)
    v = torch.tensor(verts)
    ppath = os.path.join(tmp_path, "dmtet.pt")
    torch.save({"sdf": torch.sign(0.3 - v.norm(dim=1)), "vis": (v[:, 2] > 0).float()}, ppath)
    x = _cli(tmp_path, "cond", "cond_gen", ["--config.eval.batch_size=2", f"--config.eval.partial_dmtet_path={ppath}",
                                            f"--config.eval.tet_path={dmtet.tet_grid_path(64)}",
                                            "--config.eval.freeze_iters=500"])
    assert x.shape == (2, 4, 64, 64, 64) and np.isfinite(x).all()
    assert np.all(x[:, :, m == 0] == 0)
