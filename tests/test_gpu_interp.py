"""Shape interpolation on the GPU: mdb_slerp_frames against the numpy oracle (sums, weights, bit-exact frames) and the
reference's own `slerp` (golden), its pair-count invariance, sizes and degenerate endpoints; the native inversion loop
bit-exact against the per-step path; the analytic-Gaussian gates through the kernel path; and
`main_diffusion.py --mode=uncond_gen_interp` end to end with noise and with shape endpoints, followed by `--mode=export`."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLD, ROOT, build_model, full_config, tiny_config
from oracle import interp_oracle
from test_gpu_cli import _run
from test_interp_cpu import gaussian_inversion_errors

pytestmark = pytest.mark.gpu

ALPHAS = [f / 7.0 for f in range(8)]


def _slerp(za, zb, alphas=ALPHAS):
    from meshdiffusion_b200.diffusion.interp import slerp_frames
    frames, coef, sums = slerp_frames(za.cuda(), zb.cuda(), alphas)
    torch.cuda.synchronize()
    return frames.cpu(), coef.cpu(), sums.cpu()


def _pairs(P, shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((P,) + shape, generator=g), torch.randn((P,) + shape, generator=g) * 0.5 + 0.1


def _check_against_oracle(za, zb, frames, coef, sums, alphas=ALPHAS):
    for p in range(za.shape[0]):
        a, b = za[p].numpy(), zb[p].numpy()
        want = interp_oracle.slerp_sums(a, b)
        assert np.all(np.abs(sums[p].numpy() - want) <= 1e-12 * np.abs(want).max()), (p, sums[p], want)
        ocoef = interp_oracle.slerp_coef(sums[p].numpy(), alphas)
        assert np.all(np.abs(coef[p].numpy() - ocoef) <= 2e-7 * np.maximum(1.0, np.abs(ocoef))), p
        assert np.array_equal(frames[p].numpy(), interp_oracle.slerp_combine(a, b, coef[p].numpy())), p
        assert torch.equal(frames[p, 0], za[p]) and torch.equal(frames[p, -1], zb[p])
        assert np.array_equal(coef[p, 0].numpy(), [1.0, 0.0]) and np.array_equal(coef[p, -1].numpy(), [0.0, 1.0])


def test_kernel_matches_oracle_and_reference_golden():
    gold = np.load(os.path.join(GOLD, "slerp_reference.npz"))
    za = torch.from_numpy(gold["za"].astype(np.float32))
    zb = torch.from_numpy(gold["zb"].astype(np.float32))
    alphas = [float(a) for a in gold["alphas"]]
    frames, coef, sums = _slerp(za, zb, alphas)
    assert frames.shape == (3, 8, 4, 16, 16, 16) and coef.shape == (3, 8, 2) and sums.dtype == torch.float64
    _check_against_oracle(za, zb, frames, coef, sums, alphas)
    stride = int(gold["stride"])
    for p in range(3):
        got = frames[p].reshape(8, -1)[:, ::stride].numpy()
        want = gold["frames"][p]
        err = np.abs(got - want).max() / np.abs(want).max()
        assert err <= 5e-7, (p, err)


def test_pair_count_invariance():
    za, zb = _pairs(5, (4, 16, 16, 16), 1)
    za[3] *= 1e-3  # a very different scale in the same launch
    frames, coef, sums = _slerp(za, zb)
    _check_against_oracle(za, zb, frames, coef, sums)
    for p in range(5):
        f1, c1, s1 = _slerp(za[p:p + 1], zb[p:p + 1])
        assert torch.equal(f1[0], frames[p]) and torch.equal(c1[0], coef[p]) and torch.equal(s1[0], sums[p]), p


@pytest.mark.parametrize("n", [4 * 16 ** 3 + 3, 4 * 128 ** 3])
def test_sizes(n):
    za, zb = _pairs(2, (n,), 2)
    frames, coef, sums = _slerp(za, zb, [0.0, 0.25, 0.5, 1.0])
    _check_against_oracle(za, zb, frames, coef, sums, [0.0, 0.25, 0.5, 1.0])


def test_frame_count_beyond_one_weight_launch():
    za, zb = _pairs(2, (1000,), 3)
    alphas = [f / 299.0 for f in range(300)]
    frames, coef, sums = _slerp(za, zb, alphas)
    _check_against_oracle(za, zb, frames, coef, sums, alphas)


def test_degenerate_endpoints_lerp():
    a = torch.randn(4, 8, 8, 8, generator=torch.Generator().manual_seed(4))
    alphas = [0.0, 0.3, 0.7, 1.0]
    lerp = np.stack([1.0 - np.array(alphas), np.array(alphas)], 1).astype(np.float32)
    for b in (a.clone(), -a, torch.zeros_like(a)):
        frames, coef, sums = _slerp(a[None], b[None], alphas)
        assert torch.isfinite(frames).all()
        assert np.array_equal(coef[0].numpy(), lerp)
        assert np.array_equal(frames[0].numpy(), interp_oracle.slerp_combine(a.numpy(), b.numpy(), lerp))
    frames, coef, _ = _slerp(torch.zeros_like(a)[None], torch.zeros_like(a)[None], alphas)
    assert torch.all(frames == 0)


def test_entry_point_errors():
    from meshdiffusion_b200 import _native
    L = _native.lib()
    a = torch.zeros(2, 64, device="cuda")
    buf = lambda *s, dt=torch.float32: torch.empty(*s, device="cuda", dtype=dt)  # noqa: E731
    partial, sums = buf(2, L.mdb_slerp_chunks(), 3, dt=torch.float64), buf(2, 3, dt=torch.float64)
    coef, out = buf(2, 4, 2), buf(2, 4, 64)
    al = (ctypes.c_double * 4)(0.0, 0.3, 0.6, 1.0)
    P = _native.ptr
    stream = _native.current_stream()
    cases = [(64, 2, al, 1, P(out)), (64, 0, al, 4, P(out)), (0, 2, al, 4, P(out)), (64, 2, None, 4, P(out)),
             (64, 2, al, 4, None), (64, 2, (ctypes.c_double * 4)(0.0, float("nan"), 0.5, 1.0), 4, P(out))]
    for n, pairs, alphas, frames, o in cases:
        rc = L.mdb_slerp_frames(P(a), P(a), n, pairs, alphas, frames, P(partial), P(sums), P(coef), o, stream)
        assert rc != 0 and L.mdb_last_error().startswith(b"mdb_slerp_frames")
    assert L.mdb_slerp_frames(P(a), P(a), 64, 2, al, 4, P(partial), P(sums), P(coef), P(out), stream) == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("size,precision", [("tiny", "bf16x3"), ("res64", "bf16")])
def test_native_inversion_matches_stepwise(size, precision):
    """The inverter's device-resident loop (mdb_solver_run) is bitwise the per-step path (model + mdb_solver_update)."""
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    cfg = tiny_config("res64", precision) if size == "tiny" else full_config("res64", precision)
    model, sd = build_model(cfg, "cuda:0", 21)
    R, B = cfg.data.image_size, 2
    sde = sde_lib.VPSDE(0.1, 20.0, 1000, device="cuda")
    mask = sd["mask"].view(1, R, R, R).cuda()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.randn(B, 4, R, R, R, device="cuda", generator=g) * 0.5).clamp(-1, 1)
    invert = sampling.get_dpm_solver_inverter(sde, (B, 4, R, R, R), 6, grid_mask=mask, device="cuda")
    za, nfe_a = invert(model, x)
    zb, nfe_b = invert(lambda xx, labels: model(xx, labels), x)  # not a ScoreNet: the per-step path
    assert nfe_a == nfe_b == 6 and torch.isfinite(za).all()
    assert torch.equal(za, zb), "mdb_solver_run differs from the per-step inversion"
    assert torch.all(za[:, :, mask[0] == 0] == 0) and not torch.equal(za, x * mask)


def test_gaussian_inversion_through_kernel_path():
    e25, r25 = gaussian_inversion_errors(25, device="cuda")
    e50, r50 = gaussian_inversion_errors(50, device="cuda")
    print(f"GPU inversion: latent K=25 {e25:.3e}, K=50 {e50:.3e}; round trip K=25 {r25:.3e}, K=50 {r50:.3e}")
    assert e25 <= 1.2e-2 and e50 <= 3e-3 and e25 / e50 >= 3.0
    assert r25 <= 5e-4 and r50 <= 5e-5


def _interp_cli(tmp_path, name, extra):
    out = os.path.join(tmp_path, name)
    _run([f"--config={ROOT}/configs/res64.py", "--mode=uncond_gen_interp", f"--config.eval.eval_dir={out}",
          f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth", "--config.model.compute_dtype=bf16",
          "--config.sampling.method=dpm_solver", "--config.sampling.dpm_steps=3", "--config.eval.batch_size=4"] + extra,
         cwd=str(tmp_path))
    d = os.path.join(out, "interp")
    with open(os.path.join(d, "index.json")) as fh:
        return d, json.load(fh)


def test_cli_noise_endpoints_and_export(tmp_path):
    d, index = _interp_cli(tmp_path, "a", ["--config.eval.interp_pairs=2"])
    assert index["method"] == "dpm_solver" and index["dpm_steps"] == 3 and index["frames"] == 4 and index["pairs"] == 2
    assert set(index["seconds"]) == {"inversion", "slerp", "sampling", "writing"}
    assert [e["file"] for e in index["files"]] == ["pair_0000.npy", "pair_0001.npy"]
    for e in index["files"]:
        x = np.load(os.path.join(d, e["file"]))
        assert x.shape == (4, 4, 64, 64, 64) and x.dtype == np.float32 and np.isfinite(x).all()
        assert e["endpoints"] == "noise" and e["alpha"] == [0.0, 1 / 3, 2 / 3, 1.0]
        assert 60.0 < e["theta_deg"] < 120.0 and all(0.9 < r < 1.1 for r in e["endpoint_rms"])
        assert e["nfe_sampling"] == 3 and e["nfe_inversion"] == 0
    d1, index1 = _interp_cli(tmp_path, "b", ["--config.eval.interp_pairs=1"])
    assert index1["files"][0]["seed"] == index["files"][0]["seed"]
    assert np.array_equal(np.load(os.path.join(d1, "pair_0000.npy")), np.load(os.path.join(d, "pair_0000.npy")))
    dd, index_ddim = _interp_cli(tmp_path, "c", ["--config.sampling.method=ddim"])
    assert index_ddim["method"] == "ddim" and index_ddim["files"][0]["seed"] == index["files"][0]["seed"]
    x = np.load(os.path.join(dd, "pair_0000.npy"))
    assert x.shape == (4, 4, 64, 64, 64) and np.isfinite(x).all()
    _run([f"--config={ROOT}/configs/res64.py", "--mode=export", f"--config.eval.eval_dir={d1}", "--config.render.res=64",
          "--config.render.ssaa=1"], cwd=str(tmp_path))
    meshes = sorted(os.listdir(os.path.join(d1, "export", "mesh")))
    assert meshes == [f"pair_0000_{i:06d}.obj" for i in range(4)]
    assert len(os.listdir(os.path.join(d1, "export", "viz"))) == 4


def test_cli_shape_endpoints(tmp_path):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    grids = synthetic_grids(2, 64, "cpu", generator=torch.Generator().manual_seed(3))
    paths = []
    for k in range(2):
        p = os.path.join(tmp_path, f"grid_{k}.pt")
        torch.save(grids[k].clone(), p)
        paths.append(p)
    meta = os.path.join(tmp_path, "list.json")
    with open(meta, "w") as fh:
        json.dump(paths, fh)
    d, index = _interp_cli(tmp_path, "s", [f"--config.data.meta_path={meta}", "--config.eval.interp_shapes=((0, 1),)"])
    assert index["endpoints"] == "shapes" and len(index["files"]) == 1
    e = index["files"][0]
    assert e["shapes"] == [0, 1] and e["sources"] == paths and e["nfe_inversion"] == 3
    x = np.load(os.path.join(d, e["file"]))
    assert x.shape == (4, 4, 64, 64, 64) and np.isfinite(x).all()
    assert len(e["recon_rel_l2"]) == 2 and all(np.isfinite(e["recon_rel_l2"]))
    print("synthetic-weight reconstruction rel-L2 (K = 3):", e["recon_rel_l2"])
