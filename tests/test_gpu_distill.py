"""GPU: progressive distillation (`--mode=distill`) and the `distilled` sampler.

mdb_distill_step bit-exact against the eager phases, phase 0 against mdb_solver_update, mdb_distill_targets against two
engine forwards and the two kernel calls, the distilled sampler's device loop against its per-step path, a learning check
on a tiny network, and `--mode=distill` end to end with its students through uncond_gen, eval_completion and export."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, build_model, full_config, tiny_config

pytestmark = pytest.mark.gpu


def _sde():
    from meshdiffusion_b200.diffusion import sde_lib
    return sde_lib.VPSDE(0.1, 20.0, 1000, device="cuda")


def _case(B, C, R, seed, K_T=8):
    from meshdiffusion_b200.diffusion import distill
    g = torch.Generator(device="cuda").manual_seed(seed)
    z_s, eps_s, eps_m = (torch.randn(B, C, R, R, R, generator=g, device="cuda") for _ in range(3))
    mask = (torch.rand(R, R, R, generator=g, device="cuda") > 0.3).float()
    return (z_s * mask).contiguous(), eps_s, eps_m, mask, distill.rows_tensor(_sde(), K_T, "cuda")


@pytest.mark.parametrize("B,R,steps", [(5, 7, [3, 0, 2, 3, 1]), (2, 64, [1, 3])])
def test_phases_bit_exact_against_the_eager_path(B, R, steps):
    """Mixed per-sample indices and a partial mask: 7^3 = 343 voxels (not a multiple of 4, under one block pass), and
    res64 at batch 2, where each block strides over its sample's 4 * 64^3 elements several times."""
    from meshdiffusion_b200.diffusion import distill
    C = 4
    z_s, eps_s, eps_m, mask, rows = _case(B, C, R, 1)
    idx = torch.tensor(steps, dtype=torch.int32, device="cuda")
    z_mid, out = torch.empty_like(z_s), torch.empty_like(z_s)
    labels = torch.empty(B, device="cuda")
    distill.distill_step(eps_s, z_s, z_mid, None, mask.reshape(-1), idx, rows, 0, labels)
    want_mid, want_m = distill.distill_step_eager(eps_s.cpu(), z_s.cpu(), None, mask.cpu(), rows.cpu(), idx.cpu(), 0)
    assert torch.equal(z_mid.cpu(), want_mid) and torch.equal(labels.cpu(), want_m)
    distill.distill_step(eps_m, z_s, z_mid, out, mask.reshape(-1), idx, rows, 1, labels)
    want_out, want_s = distill.distill_step_eager(eps_m.cpu(), z_s.cpu(), z_mid.cpu(), mask.cpu(), rows.cpu(), idx.cpu(), 1)
    assert torch.equal(out.cpu(), want_out) and torch.equal(labels.cpu(), want_s)
    if B < 5:
        return
    # an index outside the rows reads none: that sample is NaN, the others are untouched
    bad = torch.tensor([3, 4, 2, -1, 1], dtype=torch.int32, device="cuda")
    out2 = torch.zeros_like(z_s)
    distill.distill_step(eps_m, z_s, z_mid, out2, mask.reshape(-1), bad, rows, 1, labels)
    assert torch.isnan(out2[[1, 3]]).all() and torch.isnan(labels[[1, 3]]).all()
    assert torch.equal(out2[[0, 2, 4]], out[[0, 2, 4]])


def test_wrappers_refuse_operands_the_kernel_would_misread():
    from meshdiffusion_b200.diffusion import distill
    z_s, eps_s, _, mask, rows = _case(2, 4, 5, 3)
    z_mid, labels = torch.empty_like(z_s), torch.empty(2, device="cuda")
    ok = dict(eps=eps_s, z_s=z_s, z_mid=z_mid, out=None, mask_flat=mask.reshape(-1),
              idx=torch.tensor([0, 1], dtype=torch.int32, device="cuda"), rows=rows, phase=0, labels=labels)
    distill.distill_step(**ok)
    for key, bad in (("idx", ok["idx"].long()), ("rows", rows.double()), ("eps", eps_s.transpose(3, 4)),
                     ("z_s", z_s.cpu()), ("labels", torch.empty(3, device="cuda")), ("mask_flat", mask.reshape(-1)[:-1])):
        with pytest.raises(ValueError):
            distill.distill_step(**{**ok, key: bad})


def test_phase0_equals_denoise_entry_with_equal_indices():
    from meshdiffusion_b200.diffusion import distill, sampling
    B, C, R = 3, 4, 9
    z_s, eps_s, _, mask, rows = _case(B, C, R, 2, K_T=16)
    sde = _sde()
    labels = sampling.ddim_grid(sde, 16)
    entries_c = sampling._entries_c(sampling.ddim_table(sde, labels))
    for i in (0, 5, 7):
        idx = torch.full((B,), i, dtype=torch.int32, device="cuda")
        z_mid, lab = torch.empty_like(z_s), torch.empty(B, device="cuda")
        distill.distill_step(eps_s, z_s, z_mid, None, mask.reshape(-1), idx, rows, 0, lab)
        x, hist = z_s.clone(), torch.empty_like(z_s)
        sampling._update(eps_s, x, hist, mask.reshape(-1), entries_c[2 * i])
        assert torch.equal(z_mid, x), f"phase 0 differs from mdb_solver_update at row {i}"
        assert torch.all(lab == labels[2 * i + 1])


def test_distill_targets_equal_two_forwards_and_the_kernels():
    from meshdiffusion_b200.diffusion import distill
    cfg = tiny_config("res64", "bf16x3")
    model, sd = build_model(cfg, "cuda", 5)
    R, B = cfg.data.image_size, 3
    mask = sd["mask"].cuda().reshape(-1).contiguous()
    g = torch.Generator(device="cuda").manual_seed(4)
    z_s = (torch.randn(B, 4, R, R, R, generator=g, device="cuda") * mask.view(R, R, R)).contiguous()
    rows = distill.rows_tensor(_sde(), 8, "cuda")
    idx = torch.tensor([2, 0, 3], dtype=torch.int32, device="cuda")
    labels = rows[idx.long(), 0].contiguous()
    with torch.no_grad():
        got = distill.distill_targets(model.module, z_s, idx, rows, mask, labels.clone())
        lab = labels.clone()
        z_mid, out = torch.empty_like(z_s), torch.empty_like(z_s)
        distill.distill_step(model(z_s, lab).contiguous(), z_s, z_mid, None, mask, idx, rows, 0, lab)
        distill.distill_step(model(z_mid, lab).contiguous(), z_s, z_mid, out, mask, idx, rows, 1, lab)
    assert torch.isfinite(got).all() and torch.equal(got, out)
    assert torch.equal(lab, labels)


def test_distilled_sampler_device_loop_equals_per_step_path():
    from meshdiffusion_b200.diffusion import sampling
    cfg = tiny_config("res64", "bf16x3")
    model, sd = build_model(cfg, "cuda", 6)
    R, B = cfg.data.image_size, 2
    grid_mask = sd["mask"].cuda().view(1, R, R, R)
    x0 = torch.randn(B, 4, R, R, R, generator=torch.Generator(device="cuda").manual_seed(0), device="cuda")
    outs = []
    for native in (True, False):
        fn = sampling.get_distilled_sampler(_sde(), (B, 4, R, R, R), lambda x: x, 4, device="cuda", grid_mask=grid_mask,
                                            native_rng=native)
        out, nfe = fn(model, x0=x0)
        assert nfe == 4
        outs.append(out)
    assert torch.isfinite(outs[0]).all() and torch.equal(outs[0], outs[1])


def _sphere_batches(B, R, seed):
    """Smooth synthetic grids: channel 0 the sign of a sphere of random radius, channels 1-3 small noise."""
    c = (torch.arange(R, device="cuda").float() + 0.5) / R - 0.5
    r = torch.sqrt(c[:, None, None] ** 2 + c[None, :, None] ** 2 + c[None, None, :] ** 2)
    g = torch.Generator(device="cuda").manual_seed(seed)
    while True:
        rad = 0.2 + 0.15 * torch.rand(B, 1, 1, 1, generator=g, device="cuda")
        x = torch.zeros(B, 4, R, R, R, device="cuda")
        x[:, 0] = torch.sign(rad - r)
        x[:, 1:] = 0.1 * torch.randn(B, 3, R, R, R, generator=g, device="cuda")
        yield x, g


def test_one_round_lowers_the_match_error():
    """Tiny network (bf16x3 for both plans), smooth synthetic grids: a teacher first trained for 400 steps with
    `--mode=train`'s step, then one K_T = 4 -> K_S = 2 round of 400 optimiser steps (batch 4, lr 1e-4): the student's
    2-step map moves toward the teacher's 4-step map. (A teacher with random weights is no denoiser: its 2- and 4-step
    maps amplify the first step's error by alpha_500 / alpha_999 ~ 40, and the match error does not measure learning.)"""
    from meshdiffusion_b200.diffusion import distill, trainer
    from meshdiffusion_b200.diffusion.models.ema import ExponentialMovingAverage
    cfg = tiny_config("res64", "bf16x3")
    cfg.training.compute_dtype = "bf16x3"
    cfg.model.dropout = 0.0
    cfg.model.ema_rate = 0.99
    cfg.optim.warmup = 0
    cfg.optim.lr = 2e-4
    teacher, sd = build_model(cfg, "cuda", 7)
    R, B = cfg.data.image_size, 4
    mask = sd["mask"].cuda().view(1, 1, R, R, R)
    sde = _sde()
    torch.manual_seed(0)
    data = _sphere_batches(B, R, 2)
    tstate = dict(model=teacher, optimizer=distill.losses.get_optimizer(cfg, teacher.parameters()),
                  ema=ExponentialMovingAverage(teacher.parameters(), decay=cfg.model.ema_rate), step=0)
    train_step = trainer.make_train_step(cfg, tstate, sde, mask)
    for _ in range(400):
        train_step(tstate, next(data)[0] * mask)
    tstate["ema"].copy_to(teacher.parameters())
    teacher.eval()
    state = distill.student_state(cfg, teacher, 1e-4)
    rows = distill.rows_tensor(sde, 4, "cuda")
    step = distill.make_distill_step(cfg, state, sde, mask, teacher, rows, 1e-4)
    x_match = sde.prior_sampling((B, 4, R, R, R), generator=torch.Generator().manual_seed(1)).cuda() * mask
    before = distill.match_error(teacher, state["ema"], sde, 4, x_match, mask)
    losses = []
    for _ in range(400):
        x, g = next(data)
        idx = torch.randint(0, 2, (B,), generator=g, device="cuda").to(torch.int32)
        losses.append(step(state, x * mask, idx)["loss"].item())
    after = distill.match_error(teacher, state["ema"], sde, 4, x_match, mask)
    print(f"match error before {before}, after {after}; loss first 10 {np.mean(losses[:10]):.4e}, "
          f"last 10 {np.mean(losses[-10:]):.4e}")
    assert np.isfinite(losses).all()
    # H100 80GB HBM3: rms 13.89 -> 6.14 (ratio 0.44), sign agreement 0.899 -> 0.916, loss 1.45e-2 -> 4.82e-3
    assert after["rms"] < 0.7 * before["rms"]
    assert after["sign_agreement"] > before["sign_agreement"] - 0.01


# ---- end to end --------------------------------------------------------------------------------------------------
def _run(args, cwd):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main_diffusion.py")] + args, cwd=cwd, capture_output=True,
                       text=True, timeout=1500)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def test_distill_cli_two_rounds_resume_and_students_in_every_mode(tmp_path):
    from meshdiffusion_b200.diffusion import trainer
    from meshdiffusion_b200.diffusion.utils import save_checkpoint
    from meshdiffusion_b200.geometry import dmtet
    cfg = full_config("res64", "bf16")
    cfg.device = torch.device("cpu")
    teacher = os.path.join(tmp_path, "teacher.pth")
    save_checkpoint(teacher, trainer.build_state(cfg))
    wd = os.path.join(tmp_path, "run")
    base = [f"--config={ROOT}/configs/res64.py", "--config.model.compute_dtype=bf16"]
    distill_args = base + ["--mode=distill", f"--config.training.train_dir={wd}", "--config.data.synthetic=True",
                           "--config.training.batch_size=1", "--config.training.log_freq=1",
                           "--config.training.snapshot_freq_for_preemption=1", f"--config.distill.teacher_ckpt={teacher}",
                           "--config.distill.start_steps=8", "--config.distill.final_steps=2", "--config.distill.iters=3"]
    _run(distill_args, cwd=str(tmp_path))
    out = os.path.join(wd, "distill")
    for K_T, K_S in ((8, 4), (4, 2)):
        info = json.load(open(os.path.join(out, f"steps_{K_S}", "distill.json")))
        assert info["teacher_steps"] == K_T and info["iters_run"] == 3 and np.isfinite(info["final_loss"])
        for when in ("start", "end"):
            assert 0 <= info["match_error"][when]["sign_agreement"] <= 1 and np.isfinite(info["match_error"][when]["rms"])
        ck = torch.load(os.path.join(out, f"steps_{K_S}", "checkpoint.pth"), map_location="cpu", weights_only=False)
        assert set(ck) == {"optimizer", "model", "ema", "step"} and ck["step"] == 3
        assert len(ck["ema"]["shadow_params"]) == 494
    # a run killed in round 2 after its step-2 snapshot: the pre-emption checkpoint holds that state; restart there
    assert json.load(open(os.path.join(out, "progress.json"))) == {"round": 2, "step": 0}
    start = json.load(open(os.path.join(out, "steps_2", "distill.json")))["match_error"]["start"]
    with open(os.path.join(out, "progress.json"), "w") as fh:
        json.dump({"round": 1, "step": 2, "start_match": start}, fh)
    r = _run(distill_args, cwd=str(tmp_path))
    assert "resuming round 2" in r.stderr + r.stdout
    info = json.load(open(os.path.join(out, "steps_2", "distill.json")))
    assert info["iters_run"] == 1 and info["match_error"]["start"] == start
    student = os.path.join(out, "steps_2", "checkpoint.pth")

    samples = os.path.join(tmp_path, "samples")
    _run(base + ["--mode=uncond_gen", f"--config.eval.eval_dir={samples}", f"--config.eval.ckpt_path={student}",
                 "--config.eval.batch_size=2", "--config.sampling.method=distilled", "--config.sampling.distill_steps=2",
                 "--config.sampling.native_rng=True"], cwd=str(tmp_path))
    x = np.load(os.path.join(samples, "0.npy"))
    assert x.shape == (2, 4, 64, 64, 64) and np.isfinite(x).all()
    _run(base + ["--mode=export", f"--config.eval.eval_dir={samples}", "--config.render.res=64",
                 "--config.render.ssaa=1"], cwd=str(tmp_path))
    assert len(os.listdir(os.path.join(samples, "export", "mesh"))) == 2

    grids = trainer.synthetic_grids(1, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(2)).cpu()
    gpath = os.path.join(tmp_path, "grid_0.pt")
    torch.save(grids[0].clone(), gpath)
    meta = os.path.join(tmp_path, "meta.json")
    json.dump([gpath], open(meta, "w"))
    ev = os.path.join(tmp_path, "eval")
    _run(base + [f"--config.data.meta_path={meta}", "--mode=make_partial", f"--config.eval.eval_dir={ev}",
                 "--config.eval.partial_views=(0,)", "--config.eval.partial_res=256"], cwd=str(tmp_path))
    comp = os.path.join(tmp_path, "comp")
    _run(base + [f"--config.data.meta_path={meta}", "--mode=eval_completion", f"--config.eval.ckpt_path={student}",
                 f"--config.eval.tet_path={dmtet.tet_grid_path(64)}", "--config.eval.completion_k=2",
                 "--config.eval.metric_points=256", "--config.sampling.method=distilled",
                 "--config.sampling.distill_steps=2", "--config.eval.batch_size=2", f"--config.eval.eval_dir={comp}",
                 f"--config.eval.partial_dir={ev}/partial"], cwd=str(tmp_path))
    m = json.load(open(os.path.join(comp, "completion", "metrics.json")))
    assert m["settings"]["sampler"] == "distilled" and m["settings"]["distill_steps"] == 2 and m["settings"]["nfe"] == 2
