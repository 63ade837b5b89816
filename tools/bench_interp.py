"""Times shape interpolation (`--mode=uncond_gen_interp`) on synthetic weights:
  * the slerp kernel (mdb_slerp_frames) at 4 * 128^3 elements per endpoint, one pair, F frames: CUDA events over many
    launches after a warm-up, and GB/s over the bytes the call must move (phase 1 reads a and b: 8 B per element; phase 3
    reads them again and writes F frames: 8 + 4 F B per element), against the H100 SXM data-sheet 3.35 TB/s;
  * one noise pair at res64, F frames, K steps, per operand mode, end to end (prior draw, slerp, sampling, copy to the
    host): host clock around a device synchronise;
  * one shape pair (two synthetic grids): inversion of both grids, then decoding the F frames, each timed on its own,
    with the reconstruction rel-L2 of the end frames;
  * the Chamfer distance between consecutive decoded frames (2048 surface points, as --mode=eval_metrics samples them).
    Context only: synthetic weights say nothing about how smooth a trained model's path is.
The card's name, power limit and SM clock are read with nvidia-smi in the same run. Prints one JSON line.

    python tools/bench_interp.py [--frames 8] [--steps 25] [--precisions bf16x3,bf16] [--out path.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}


def _model(precision, device):
    from configs import res64
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth
    cfg = res64.get_config()
    cfg.model.compute_dtype = precision
    cfg.device = device
    model = mutils.create_model(cfg)
    net = model.module
    net.load_state_dict(synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=11))
    model.eval()
    return cfg, model


def _wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def bench_kernel(frames, iters=200):
    """mdb_slerp_frames alone, with every buffer allocated once."""
    import ctypes
    from meshdiffusion_b200 import _native
    L = _native.lib()
    n = 4 * 128 ** 3
    g = torch.Generator(device="cuda").manual_seed(0)
    za = torch.randn(1, n, device="cuda", generator=g)
    zb = torch.randn(1, n, device="cuda", generator=g)
    partial = torch.empty(1, L.mdb_slerp_chunks(), 3, device="cuda", dtype=torch.float64)
    sums = torch.empty(1, 3, device="cuda", dtype=torch.float64)
    coef = torch.empty(1, frames, 2, device="cuda")
    out = torch.empty(1, frames, n, device="cuda")
    alphas = (ctypes.c_double * frames)(*[f / (frames - 1) for f in range(frames)])
    P = _native.ptr
    args = (P(za), P(zb), n, 1, alphas, frames, P(partial), P(sums), P(coef), P(out), _native.current_stream())
    for _ in range(10):
        _native.check(L.mdb_slerp_frames(*args))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        L.mdb_slerp_frames(*args)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    nbytes = (8 + 8 + 4 * frames) * n
    return {"elements": n, "frames": frames, "launches": iters, "ms_per_call": ms, "bytes": nbytes,
            "gb_per_s": nbytes / ms / 1e6, "share_of_3_35_tb_s": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}


def bench_pairs(precision, frames, steps):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    from meshdiffusion_b200.diffusion.interp import _masked_rel_l2, slerp_frames
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import pointcloud
    from meshdiffusion_b200.geometry.dmtet import grid_mask_from_tets
    device = torch.device("cuda:0")
    cfg, model = _model(precision, device)
    R, C = 64, 4
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
    mask = grid_mask_from_tets(R).to(device).view(1, R, R, R)
    sample = sampling.get_dpm_solver_sampler(sde, (frames, C, R, R, R), lambda x: x, n_steps=steps, device=device,
                                             grid_mask=mask)
    invert = sampling.get_dpm_solver_inverter(sde, (2, C, R, R, R), steps, grid_mask=mask, device=device)
    alphas = [f / (frames - 1) for f in range(frames)]

    def noise_pair(p):
        z = sde.prior_sampling((2, C, R, R, R), generator=torch.Generator().manual_seed(p)).to(device)
        fr, _, _ = slerp_frames(z[:1], z[1:], alphas)
        out, _ = sample(model, x0=fr[0])
        return out.cpu()

    noise_pair(0)  # warm-up: engine build, first launches
    _, noise_s = _wall(lambda: noise_pair(1))
    grids = synthetic_grids(2, R, device, generator=torch.Generator(device=device).manual_seed(3)) * mask
    (z, nfe_inv), inv_s = _wall(lambda: invert(model, grids))
    fr, _, _ = slerp_frames(z[:1], z[1:], alphas)
    (dec, nfe), dec_s = _wall(lambda: sample(model, x0=fr[0]))
    recon = [_masked_rel_l2(dec[0], grids[0], mask), _masked_rel_l2(dec[-1], grids[1], mask)]
    pts, empty = pointcloud.grids_to_point_clouds(dec, R, 2048, seed=0)
    cd = pointcloud.chamfer_matrix(pts)
    consecutive = [None if bool(empty[f] or empty[f + 1]) else float(cd[f, f + 1]) for f in range(frames - 1)]
    return {"noise_pair_s": noise_s, "shape_pair": {"inversion_s": inv_s, "nfe_inversion": int(nfe_inv),
                                                   "decoding_s": dec_s, "nfe_decoding": int(nfe),
                                                   "recon_rel_l2": recon},
            "chamfer_consecutive_frames": consecutive, "empty_frames": int(empty.sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--precisions", default="bf16x3,bf16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_interp.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    res = {"card": _card(), "frames": a.frames, "steps": a.steps, "kernel": bench_kernel(a.frames)}
    for p in a.precisions.split(","):
        res[p] = bench_pairs(p, a.frames, a.steps)
    res["card_after"] = _card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
