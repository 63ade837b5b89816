"""CPU: progressive distillation on the halving DDIM grid (`--mode=distill`, `sampling.method='distilled'`).

The grid, the DDIM rows and the distillation rows against the float64 oracle (oracle/distill_oracle.py); the eager fp32
phases (the kernel's bit-exact oracle) against it; an analytic gate on Gaussian data, where every map is a scalar
multiple of z; the settings checks; and the round and resume bookkeeping of the host loop with a stubbed step.
"""
import json
import os

import numpy as np
import pytest
import torch

from helpers import tiny_config
from oracle import distill_oracle as orc


def _sde(N=1000):
    from meshdiffusion_b200.diffusion import sde_lib
    return sde_lib.VPSDE(0.1, 20.0, N, device="cpu")


def _abar(sde):
    return sde.alphas_cumprod.double().numpy()


# ---- grid and tables ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1000, 37])
def test_ddim_grid_endpoints_distinct_and_halving(N):
    from meshdiffusion_b200.diffusion.sampling import ddim_grid
    sde = _sde(N)
    for K in range(2, N):
        l = ddim_grid(sde, K)
        assert len(l) == K + 1 and l[0] == N - 1 and l[-1] == 0
        assert all(a > b for a, b in zip(l, l[1:])), f"labels repeat at K = {K}"
        assert l == orc.grid(N, K)
        if 2 * K <= N - 1:
            assert l == ddim_grid(sde, 2 * K)[::2], f"the {2 * K}-step grid does not halve to the {K}-step one"
    if N == 1000:
        assert ddim_grid(sde, 2) == [999, 500, 0]
        assert ddim_grid(sde, 512)[::64] == ddim_grid(sde, 8)


@pytest.mark.parametrize("K", [1, 0, -4, 1000, 2.0, True, "8"])
def test_ddim_grid_refusals(K):
    from meshdiffusion_b200.diffusion.sampling import ddim_grid
    with pytest.raises(ValueError):
        ddim_grid(_sde(), K)


def test_ddim_table_rows_are_ddim_steps():
    """Each row moves z as alpha_t x0^ + sigma_t eps^ with x0^ = (z - sigma_s eps^) / alpha_s, in float64."""
    from meshdiffusion_b200.diffusion.sampling import ddim_grid, ddim_table
    sde = _sde()
    abar = _abar(sde)
    labels = ddim_grid(sde, 16)
    table = ddim_table(sde, labels)
    assert table.shape == (16, 9) and np.all(table[:, 5] == 0) and np.all(table[:, 6] == 0)
    rng = np.random.default_rng(0)
    z, eps = rng.standard_normal(64), rng.standard_normal(64)
    for k, (lab, sg, inv_a, c_x, c_0, c_1, c_z, coef, std) in enumerate(table):
        s, t = labels[k], labels[k + 1]
        assert lab == s
        assert np.allclose([coef, std], orc.alpha_sigma(abar, t), rtol=1e-15, atol=0)
        got = c_x * z + c_0 * (z - sg * eps) * inv_a
        np.testing.assert_allclose(got, orc.ddim_step(abar, s, t, z, eps), rtol=1e-12, atol=1e-12)


def test_distill_rows_match_the_oracle():
    from meshdiffusion_b200.diffusion.sampling import DISTILL_COLUMNS, distill_rows
    sde = _sde()
    abar = _abar(sde)
    for K_T in (4, 16, 512):
        rows = distill_rows(sde, K_T)
        assert rows.shape == (K_T // 2, len(DISTILL_COLUMNS))
        np.testing.assert_array_equal(rows[:, :3], orc.rows(abar, K_T)[:, :3])
        np.testing.assert_allclose(rows, orc.rows(abar, K_T), rtol=1e-12, atol=1e-13)
    for bad in (3, 1000, 0):
        with pytest.raises(ValueError):
            distill_rows(sde, bad)


def test_one_student_step_with_the_target_lands_on_the_teachers_z_e():
    """For arbitrary teacher predictions, the DDIM step s -> e with eps~ from z_s is the teacher's two steps, to float64
    round-off."""
    from meshdiffusion_b200.diffusion.sampling import ddim_table, distill_rows
    sde = _sde()
    rng = np.random.default_rng(1)
    rows = distill_rows(sde, 32)
    for row in rows:
        s, m, e = (int(v) for v in row[:3])
        sg_s, ia_s, cx_s, c0_s, sg_m, ia_m, cx_m, c0_m, r, inv_d = row[3:]
        z_s, eps_s, eps_m = rng.standard_normal((3, 256))
        z_m = cx_s * z_s + c0_s * (z_s - sg_s * eps_s) * ia_s
        z_e = cx_m * z_m + c0_m * (z_m - sg_m * eps_m) * ia_m
        eps_t = (z_e - r * z_s) * inv_d
        _, sg, inv_a, c_x, c_0, *_ = ddim_table(sde, [s, e])[0]
        student = c_x * z_s + c_0 * (z_s - sg * eps_t) * inv_a
        np.testing.assert_allclose(student, z_e, rtol=0, atol=1e-12 * max(1.0, np.abs(z_e).max()))
        np.testing.assert_allclose(eps_t, orc.teacher_target(_abar(sde), s, m, e, z_s, eps_s, eps_m)[2], rtol=1e-10,
                                   atol=1e-10)


def test_eager_phases_match_the_oracle():
    """The fp32 eager phases (the kernel's bit-exact oracle) with mixed per-sample steps, an unaligned voxel count and a
    partial mask, against the float64 oracle within fp32 round-off; labels m after phase 0 and s after phase 1."""
    from meshdiffusion_b200.diffusion import distill
    sde = _sde()
    abar = _abar(sde)
    K_T = 8
    rows64 = orc.rows(abar, K_T)
    rows = distill.rows_tensor(sde, K_T, "cpu")
    g = torch.Generator().manual_seed(3)
    B, C, R = 5, 4, 7  # 343 voxels
    z_s, eps_s, eps_m = (torch.randn(B, C, R, R, R, generator=g) for _ in range(3))
    mask = (torch.rand(R, R, R, generator=g) > 0.3).float()
    z_s = z_s * mask
    idx = torch.tensor([3, 0, 2, 3, 1], dtype=torch.int32)
    z_mid, lab_m = distill.distill_step_eager(eps_s, z_s, None, mask, rows, idx, 0)
    out, lab_s = distill.distill_step_eager(eps_m, z_s, z_mid, mask, rows, idx, 1)
    assert lab_m.tolist() == [rows64[i, 1] for i in idx.tolist()] and lab_s.tolist() == [rows64[i, 0] for i in idx.tolist()]
    for b, i in enumerate(idx.tolist()):
        s, m, e = (int(v) for v in rows64[i, :3])
        zs, es, em = (t[b].double().numpy() for t in (z_s, eps_s, eps_m))
        want_m = orc.ddim_step(abar, s, m, zs, es) * mask.double().numpy()
        np.testing.assert_allclose(z_mid[b].double().numpy(), want_m, rtol=0, atol=2e-5 * np.abs(want_m).max())
        zm = z_mid[b].double().numpy()  # phase 1 from the fp32 z_mid, as the kernel takes it
        want = orc.target(abar, s, e, zs, orc.ddim_step(abar, m, e, zm, em)) * mask.double().numpy()
        np.testing.assert_allclose(out[b].double().numpy(), want, rtol=0, atol=2e-4 * np.abs(want).max())
    assert torch.all(z_mid[:, :, mask == 0] == 0) and torch.all(out[:, :, mask == 0] == 0)


# ---- analytic gate -----------------------------------------------------------------------------------------------
def _ddim_coef(table_row, eps_coef):
    """z' / z of one DDIM row when eps = eps_coef z."""
    _, sg, inv_a, c_x, c_0, *_ = table_row
    return c_x + c_0 * (1.0 - sg * eps_coef) * inv_a


def test_gaussian_gate_distilled_student_reproduces_the_teacher():
    """x0 ~ N(0, s^2) elementwise: the exact eps at label n is sigma_n z / (alpha_n^2 s^2 + sigma_n^2), so every map is
    z -> k z. The target of an exact teacher is linear in z_s; the K_S-step student that predicts it reproduces the
    2 K_S-step teacher's map to 1e-12; and the 512-step teacher approaches the probability-flow map."""
    from meshdiffusion_b200.diffusion.sampling import ddim_grid, ddim_table, distill_rows
    sde = _sde()
    abar = _abar(sde)
    sd = 0.7

    def exact_eps_coef(n):
        a, s = orc.alpha_sigma(abar, n)
        return s / (a * a * sd * sd + s * s)

    def teacher_map(K):
        labels = ddim_grid(sde, K)
        k = 1.0
        for row, n in zip(ddim_table(sde, labels), labels):
            k *= _ddim_coef(row, exact_eps_coef(n))
        return k

    for K_S in (2, 4, 8, 64):
        rows = distill_rows(sde, 2 * K_S)
        k_student = 1.0
        for row in rows:
            s, m, e = (int(v) for v in row[:3])
            sg_s, ia_s, cx_s, c0_s, sg_m, ia_m, cx_m, c0_m, r, inv_d = row[3:]
            z = np.array([1.0, -2.5, 0.3])
            z_m = cx_s * z + c0_s * (z - sg_s * exact_eps_coef(s) * z) * ia_s
            z_e = cx_m * z_m + c0_m * (z_m - sg_m * exact_eps_coef(m) * z_m) * ia_m
            eps_t = (z_e - r * z) * inv_d
            coef = eps_t / z
            assert np.ptp(coef) <= 1e-13 * np.abs(coef).max(), "the target of an exact teacher is not linear in z_s"
            _, sg, inv_a, c_x, c_0, *_ = ddim_table(sde, [s, e])[0]
            k_student *= c_x + c_0 * (1.0 - sg * coef[0]) * inv_a
        k_teacher = teacher_map(2 * K_S)
        assert abs(k_student - k_teacher) <= 1e-12 * abs(k_teacher), (K_S, k_student, k_teacher)
    a_T, s_T = orc.alpha_sigma(abar, 999)
    a_0, s_0 = orc.alpha_sigma(abar, 0)
    k_flow = np.sqrt(a_0 ** 2 * sd ** 2 + s_0 ** 2) / np.sqrt(a_T ** 2 * sd ** 2 + s_T ** 2)
    errs = {K: abs(teacher_map(K) / k_flow - 1.0) for K in (8, 64, 512)}
    # DDIM is first order: 0.248, 0.0342, 0.00439 at 8, 64, 512 steps (s = 0.7)
    assert errs[512] < errs[64] < errs[8]
    assert errs[512] < 6e-3 and errs[64] / errs[512] > 6, errs


# ---- settings ----------------------------------------------------------------------------------------------------
def _distill_config(**kw):
    cfg = tiny_config()
    from meshdiffusion_b200.compat.install import ensure_ml_collections
    ensure_ml_collections()
    import ml_collections
    cfg.distill = ml_collections.ConfigDict(dict({"teacher_ckpt": "teacher.pth", "iters": 3}, **kw))
    return cfg


def test_settings_rounds_and_defaults():
    from meshdiffusion_b200.diffusion import distill
    st = distill.settings(_distill_config())
    assert (st["start_steps"], st["final_steps"]) == (512, 8)
    assert st["rounds"] == [(512, 256), (256, 128), (128, 64), (64, 32), (32, 16), (16, 8)]
    assert st["lr"] == tiny_config().optim.lr and st["iters"] == 3
    st = distill.settings(_distill_config(start_steps=8, final_steps=2, lr=1e-4))
    assert st["rounds"] == [(8, 4), (4, 2)] and st["lr"] == 1e-4


@pytest.mark.parametrize("kw", [dict(teacher_ckpt="PLACEHOLDER"), dict(teacher_ckpt=""), dict(start_steps=24),
                                dict(start_steps=8, final_steps=8), dict(start_steps=1024), dict(final_steps=1, start_steps=4),
                                dict(start_steps=12, final_steps=4), dict(iters=0), dict(iters=2.5), dict(lr=-1.0),
                                dict(lr=float("nan")), dict(final_steps=True)])
def test_settings_refusals(kw):
    from meshdiffusion_b200.diffusion import distill
    with pytest.raises(ValueError):
        distill.settings(_distill_config(**kw))


def test_distilled_sampler_is_refused_by_edit_and_interp():
    from meshdiffusion_b200.diffusion import edit, interp
    cfg = tiny_config()
    cfg.sampling.method = "distilled"
    with pytest.raises(ValueError, match="distilled"):
        edit.sampler_settings(cfg)
    with pytest.raises(ValueError, match="distilled"):
        interp._method(cfg, False)


def test_completion_takes_the_distilled_sampler():
    from meshdiffusion_b200.diffusion import completion
    cfg = tiny_config()
    cfg.sampling.method = "distilled"
    cfg.sampling.distill_steps = 4
    assert completion.sampler(cfg, 8, 4) == ("distilled", {"distill_steps": 4})


def test_distilled_sampler_cpu_path_is_the_ddim_map():
    """The eager path of the distilled sampler with a linear stand-in network eps = c_n z follows the DDIM rows."""
    from meshdiffusion_b200.diffusion import sampling
    sde = _sde()
    R, B, K = 4, 2, 4
    mask = torch.ones(1, R, R, R)
    fn = sampling.get_distilled_sampler(sde, (B, 4, R, R, R), lambda x: x, K, device="cpu", grid_mask=mask)
    x0 = torch.randn(B, 4, R, R, R, generator=torch.Generator().manual_seed(0))
    model = lambda x, labels: x * 0.5
    out, nfe = fn(model, x0=x0)
    assert nfe == K
    k = 1.0
    labels = sampling.ddim_grid(sde, K)
    for row in sampling.ddim_table(sde, labels):
        k *= _ddim_coef(row, 0.5)
    torch.testing.assert_close(out.double(), x0.double() * k, rtol=1e-5, atol=1e-6)


# ---- host loop ---------------------------------------------------------------------------------------------------
def test_host_loop_rounds_checkpoints_and_resume(tmp_path, monkeypatch):
    """Two rounds 8 -> 4 -> 2 with a stubbed teacher, step and match error (the real ones need the GPU): per-round
    outputs, the micro-step flags, the pre-emption checkpoint and progress.json, and a restart after a kill mid-round that
    resumes at the saved step; the second round's teacher is the first round's student."""
    from meshdiffusion_b200.diffusion import distill, trainer
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from meshdiffusion_b200.diffusion.utils import save_checkpoint
    cfg = _distill_config(start_steps=8, final_steps=2, iters=5)
    cfg.device = torch.device("cpu")
    cfg.data.synthetic = True
    cfg.training.train_dir = str(tmp_path / "run")
    cfg.training.iter_size, cfg.training.batch_size = 2, 2
    cfg.training.snapshot_freq_for_preemption, cfg.training.log_freq = 2, 1
    R = cfg.data.image_size
    st = trainer.build_state(cfg)
    cfg.distill.teacher_ckpt = str(tmp_path / "teacher.pth")
    save_checkpoint(cfg.distill.teacher_ckpt, st)

    monkeypatch.setattr(distill, "load_grid_mask", lambda r, dev: torch.ones(r, r, r))
    monkeypatch.setattr(trainer, "synthetic_grids", lambda b, r, dev, gen=None: torch.zeros(b, 4, r, r, r))
    teachers, calls, kill = [], [], [None]

    def fake_load_teacher(config, path, mask):
        teachers.append(path)
        return mutils.create_model(config)

    def fake_make_distill_step(config, state, sde, mask, teacher, rows, lr):
        assert state["optimizer"].param_groups[0]["lr"] == lr
        K_S = rows.shape[0]

        def step_fn(state, batch, idx, clear_grad=True, update_param=True):
            assert tuple(batch.shape) == (2, 4, R, R, R) and idx.dtype == torch.int32
            assert int(idx.min()) >= 0 and int(idx.max()) < K_S
            if kill[0] is not None and len(calls) == kill[0]:
                raise KeyboardInterrupt
            calls.append((K_S, int(state["step"]), clear_grad, update_param))
            state["step"] += 1
            return {"loss": torch.tensor(0.5)}
        return step_fn

    monkeypatch.setattr(distill, "load_teacher", fake_load_teacher)
    monkeypatch.setattr(distill, "make_distill_step", fake_make_distill_step)
    monkeypatch.setattr(distill, "match_error", lambda *a: {"rms": 1.0, "sign_agreement": 0.5})
    out_dir = os.path.join(cfg.training.train_dir, "distill")

    kill[0] = 2 * 5 + 7  # during round 2, optimiser step 4 (after the step-2 snapshot)
    with pytest.raises(KeyboardInterrupt):
        distill.distill(cfg)
    assert os.path.exists(os.path.join(out_dir, "steps_4", "checkpoint.pth"))
    assert not os.path.exists(os.path.join(out_dir, "steps_2"))
    assert json.load(open(os.path.join(out_dir, "progress.json")))["round"] == 1
    assert json.load(open(os.path.join(out_dir, "progress.json")))["step"] == 2
    assert teachers == [cfg.distill.teacher_ckpt, os.path.join(out_dir, "steps_4", "checkpoint.pth")]
    assert [c[2:] for c in calls[:2]] == [(True, False), (False, True)]
    assert [c[1] for c in calls[:10]] == list(range(10)) and all(c[0] == 4 for c in calls[:10])
    info = json.load(open(os.path.join(out_dir, "steps_4", "distill.json")))
    assert info["teacher_steps"] == 8 and info["student_steps"] == 4 and info["iters"] == 5
    assert info["final_loss"] == 0.5 and info["match_error"]["end"] == {"rms": 1.0, "sign_agreement": 0.5}
    ck = torch.load(os.path.join(out_dir, "steps_4", "checkpoint.pth"), weights_only=False)
    assert set(ck) == {"optimizer", "model", "ema", "step"} and ck["step"] == 10

    # restart: round 2 resumes at optimiser step 2 (micro-step 4) from the pre-emption checkpoint
    calls.clear()
    teachers.clear()
    kill[0] = None
    outs = distill.distill(cfg)
    assert outs == [os.path.join(out_dir, f"steps_{k}", "checkpoint.pth") for k in (4, 2)]
    assert teachers == [os.path.join(out_dir, "steps_4", "checkpoint.pth")]
    assert [c[1] for c in calls] == [4, 5, 6, 7, 8, 9] and all(c[0] == 2 for c in calls)
    info = json.load(open(os.path.join(out_dir, "steps_2", "distill.json")))
    assert info["iters_run"] == 3 and info["match_error"]["start"] == {"rms": 1.0, "sign_agreement": 0.5}
    assert json.load(open(os.path.join(out_dir, "progress.json"))) == {"round": 2, "step": 0}
    # a finished run does nothing more
    calls.clear()
    assert distill.distill(cfg) == outs and calls == []


def test_host_loop_seeds_the_global_generators_with_seed_plus_rank(tmp_path, monkeypatch):
    """The perturbation noise and the student's dropout come from the global generators: distill() seeds them with
    seed + rank, as build_state does for `--mode=train`, so config.seed reaches every draw."""
    from meshdiffusion_b200.diffusion import distill, trainer
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from meshdiffusion_b200.diffusion.utils import save_checkpoint
    monkeypatch.setattr(distill, "load_grid_mask", lambda r, dev: torch.ones(r, r, r))
    monkeypatch.setattr(trainer, "synthetic_grids", lambda b, r, dev, gen=None: torch.zeros(b, 4, r, r, r))
    monkeypatch.setattr(distill, "load_teacher", lambda config, path, mask: mutils.create_model(config))
    monkeypatch.setattr(distill, "match_error", lambda *a: {"rms": 1.0, "sign_agreement": 1.0})
    draws = []

    def fake_make_distill_step(config, state, sde, mask, teacher, rows, lr):
        def step_fn(state, batch, idx, clear_grad=True, update_param=True):
            draws.append((torch.initial_seed(), torch.randn_like(batch).flatten()[:8].clone()))
            state["step"] += 1
            return {"loss": torch.tensor(0.5)}
        return step_fn

    monkeypatch.setattr(distill, "make_distill_step", fake_make_distill_step)

    def run(seed, name):
        cfg = _distill_config(start_steps=4, final_steps=2, iters=1)
        cfg.seed = seed
        cfg.device = torch.device("cpu")
        cfg.data.synthetic = True
        cfg.training.train_dir = str(tmp_path / name)
        cfg.training.iter_size, cfg.training.batch_size = 1, 1
        cfg.distill.teacher_ckpt = str(tmp_path / "teacher.pth")
        if not os.path.exists(cfg.distill.teacher_ckpt):
            save_checkpoint(cfg.distill.teacher_ckpt, trainer.build_state(cfg))
        draws.clear()
        distill.distill(cfg)
        return draws[0]

    a, b, a2 = run(1, "a"), run(2, "b"), run(1, "a2")
    assert a[0] == 1 and b[0] == 2
    assert not torch.equal(a[1], b[1]) and torch.equal(a[1], a2[1])
