"""Shape editing on the GPU: mdb_solver_update bit-exact against the eager fp32 update on RePaint entries (both kinds,
caller and Philox noise, shared and per-sample kept regions), mdb_solver_run bit-exact against the per-entry public path,
resample = 1 on one channel against the conditional solver table, the analytic gate through the kernel path, and
`--mode=edit` end to end followed by `--mode=export`."""
import ctypes
import glob
import json
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, build_model, full_config, tiny_config
from test_edit_cpu import check_gate
from test_gpu_completion import _run

pytestmark = pytest.mark.gpu


def _sde(device="cuda"):
    from meshdiffusion_b200.diffusion import sde_lib
    return sde_lib.VPSDE(0.1, 20.0, 1000, device=device)


def _philox(kind_offset, seed, B, C, R):
    """Philox(seed, element, offset) of every element: a renoise entry with c_x = 0, c_z = 1 and an all-ones mask."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion import sampling
    x = torch.zeros(B, C, R, R, R, device="cuda")
    e = _native.SolverEntryC(1, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0)
    sampling._update(None, x, torch.empty_like(x), torch.ones(R ** 3, device="cuda"), e, seed=seed, offset=kind_offset)
    return x


@pytest.mark.parametrize("per_sample", [False, True])
@pytest.mark.parametrize("philox", [False, True])
@pytest.mark.parametrize("entry", ["first_order", "second_order_sde", "renoise", "last"])
def test_entry_kernel_matches_eager(entry, philox, per_sample):
    from meshdiffusion_b200.diffusion import sampling
    sde = _sde("cpu")
    table, _ = sampling.repaint_schedule(sde, 10, 3, 3, stochastic=True)
    e = {"first_order": 0, "second_order_sde": 1, "renoise": 3, "last": len(table) - 1}[entry]
    rows32, entries_c = table.astype(np.float32), sampling._entries_c(table)
    g = torch.Generator().manual_seed(21 + e)
    B, C, R, seed, offset = 3, 4, 16, 99, 4 * e
    x, eps, hist, z, z2 = (torch.randn(B, C, R, R, R, generator=g) for _ in range(5))
    mask = (torch.rand(R, R, R, generator=g) < 0.6).float()
    nk = B if per_sample else 1
    known = torch.randn(nk, C, R, R, R, generator=g)
    m = (torch.rand(nk, R, R, R, generator=g) < 0.5).float() * mask
    chans = [0, 1, 3]
    if philox:
        z, z2 = _philox(offset, seed, B, C, R).cpu(), _philox(offset + 2, seed, B, C, R).cpu()
    xe, he = x.clone(), hist.clone()
    sampling._update_eager(eps, xe, he, mask, rows32[e], z, sampling._Known(known, m, chans, B), z2)
    xg, hg = x.cuda(), hist.cuda()
    kn = sampling._Known(known.cuda(), m.cuda(), chans, B)
    sampling._update(eps.cuda(), xg, hg, mask.cuda().reshape(-1), entries_c[e], None if philox else z.cuda(), kn,
                     None if philox else z2.cuda(), seed=seed, offset=offset)
    assert torch.equal(xg.cpu(), xe), f"{entry}: x differs from the eager update"
    assert torch.equal(hg.cpu(), he), f"{entry}: x0 history differs from the eager update"
    assert torch.all(xe[:, :, mask == 0] == 0)
    if philox:
        assert abs(z.mean().item()) < 0.02 and abs(z.var().item() - 1.0) < 0.03
        assert abs((z * z2).mean().item()) < 0.02, "the replacement draw must be independent of z"


@pytest.mark.parametrize("size,precision", [("tiny", "bf16x3"), ("res64", "bf16")])
def test_device_loop_matches_per_entry(size, precision):
    """mdb_solver_run(seed, step0, n) on a RePaint table is bitwise equal to n x [model(x, label) on denoise entries +
    mdb_solver_update(noise=NULL, seed, offset=4*e)] through the public entry points."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion import sampling
    cfg = tiny_config("res64", precision) if size == "tiny" else full_config("res64", precision)
    B, step0, n, seed = (4, 2, 9, 31) if size == "tiny" else (2, 3, 6, 32)
    model, sd = build_model(cfg, "cuda:0", 21)
    net = model.module
    R = cfg.data.image_size
    table, _ = sampling.repaint_schedule(_sde(), 8, 2, 3, stochastic=True)
    assert 1 in table[step0:step0 + n, 0]
    entries_c = sampling._entries_c(table)
    mask = sd["mask"].view(-1).cuda().contiguous()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x0 = (torch.randn(B, 4, R, R, R, device="cuda", generator=g) * mask.view(R, R, R)).contiguous()
    h0 = torch.randn(B, 4, R, R, R, device="cuda", generator=g)
    known = torch.randn(B, 4, R, R, R, device="cuda", generator=g)
    keep = (torch.rand(1, R, R, R, device="cuda", generator=g) < 0.5).float() * mask.view(1, R, R, R)
    kn = sampling._Known(known, keep, range(4), B)
    with torch.no_grad():
        xa, ha = x0.clone(), h0.clone()
        sampling._native_run(net, xa, ha, mask, entries_c, seed, step0, n, kn)
        xb, hb = x0.clone(), h0.clone()
        L = _native.lib()
        ks = kn.struct()
        for e in range(step0, step0 + n):
            eps = None if table[e, 0] else model(xb, torch.full((B,), float(entries_c[e].label), device="cuda"))
            _native.check(L.mdb_solver_update(_native.ptr(eps), _native.ptr(xb), _native.ptr(hb), _native.ptr(mask),
                                              ctypes.byref(entries_c[e]), R ** 3, 4, B, None, seed, 4 * e,
                                              ctypes.byref(ks), _native.current_stream()))
    assert torch.isfinite(xa).all()
    assert torch.equal(xa, xb) and torch.equal(ha, hb), "mdb_solver_run differs from the per-entry public path"


@pytest.mark.parametrize("stochastic", [False, True])
def test_resample_one_single_channel_is_the_solver_table(stochastic):
    """resample = 1 with channel set {0}: outside the kept region the output is the conditional solver table's, which
    stops replacing before its last step (same loop, initial x and seed); inside it, the known grid exactly."""
    from meshdiffusion_b200.diffusion import sampling
    cfg = tiny_config("res64", "bf16x3")
    model, sd = build_model(cfg, "cuda:0", 21)
    net = model.module
    R, B, seed, K = cfg.data.image_size, 3, 5, 10
    sde = _sde()
    _, dpm = sampling.dpm_solver_schedule(sde, K, stochastic)
    table, _ = sampling.repaint_schedule(sde, K, 3, 1, stochastic)
    mask = sd["mask"].view(-1).cuda().contiguous()
    g = torch.Generator(device="cuda").manual_seed(seed)
    x0 = (torch.randn(B, 4, R, R, R, device="cuda", generator=g) * mask.view(R, R, R)).contiguous()
    known = torch.sign(torch.randn(B, 4, R, R, R, device="cuda", generator=g))
    keep = (torch.rand(B, 1, R, R, R, device="cuda", generator=g) < 0.5).float() * mask.view(1, 1, R, R, R)
    with torch.no_grad():
        xa = x0.clone()
        kn = sampling._Known(known, keep, [0], B)
        sampling._native_run(net, xa, torch.empty_like(xa), mask, sampling._entries_c(table), seed, known=kn)
        xb = x0.clone()
        sampling._native_run(net, xb, torch.empty_like(xb), mask, sampling._entries_c(dpm), seed, known=kn,
                             replace_until=K - 1)
    kept = keep[:, 0] > 0
    assert torch.equal(xa[:, 1:], xb[:, 1:])
    assert torch.equal(xa[:, 0][~kept], xb[:, 0][~kept])
    assert torch.equal(xa[:, 0][kept], known[:, 0][kept])


def test_analytic_gate_through_kernel_path():
    check_gate("cuda")


def test_edit_cli_then_export(tmp_path):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    grids = synthetic_grids(3, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(4)).cpu()
    src = os.path.join(tmp_path, "shapes.npy")
    np.save(src, grids.numpy().astype(np.float32))
    out = os.path.join(tmp_path, "ev")
    # a small score network at R = 64 (random weights: the checkpoint is missing)
    _run([f"--config={ROOT}/configs/res64.py", "--mode=edit", f"--config.eval.eval_dir={out}",
          f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth", f"--config.eval.edit_source={src}",
          "--config.eval.edit_boxes=((-0.6, -0.6, -0.6, 0.6, 0.0, 0.6), (0.2, 0.2, 0.2, 0.5, 0.5, 0.5))",
          "--config.eval.edit_k=2", "--config.eval.edit_jump=2", "--config.eval.edit_resample=2",
          "--config.eval.batch_size=4", "--config.eval.metric_points=512", "--config.model.compute_dtype=bf16x3",
          "--config.model.nf=32", "--config.model.ch_mult=(1, 2, 2, 2)", "--config.model.num_res_blocks=1",
          "--config.sampling.method=dpm_solver", "--config.sampling.dpm_steps=4", "--config.sampling.native_rng=True"],
         cwd=str(tmp_path))
    d = os.path.join(out, "edit")
    assert sorted(os.listdir(d)) == ["edit.json"] + [f"shapes_{s:04d}.npy" for s in range(3)]
    with open(os.path.join(d, "edit.json")) as fh:
        rep = json.load(fh)
    s = rep["settings"]
    assert s["k"] == 2 and s["jump"] == 2 and s["resample"] == 2 and s["dpm_steps"] == 4 and s["nfe"] == 4 + 2
    assert s["regenerated_vertices"] > 0 and s["kept_voxels"] > 0
    assert [r["source_index"] for r in rep["sources"]] == [0, 1, 2]
    for r in rep["sources"]:
        x = np.load(os.path.join(d, r["file"]))
        assert x.shape == (2, 4, 64, 64, 64) and x.dtype == np.float32 and np.isfinite(x).all()
        assert len(r["variants"]) == 2
        for v in r["variants"]:
            assert v["known_max_abs_diff"] == 0.0
            assert v["regenerated_vertices"] == s["regenerated_vertices"] and 0.0 <= v["sign_flip_share"] <= 1.0
    assert rep["means"]["known_max_abs_diff"] == 0.0
    _run([f"--config={ROOT}/configs/res64.py", "--mode=export", f"--config.eval.eval_dir={d}", "--config.render.res=64",
          "--config.render.ssaa=1"], cwd=str(tmp_path))
    meshes = sorted(os.listdir(os.path.join(d, "export", "mesh")))
    assert meshes == sorted(f"shapes_{s:04d}_{i:06d}.obj" for s in range(3) for i in range(2))
    assert glob.glob(os.path.join(d, "export", "viz", "*.png"))
