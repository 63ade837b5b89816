"""Times few-step DPM-Solver++(2M) sampling (`sampling.method='dpm_solver'`) on synthetic weights, per operand mode:
  * one K-step batch through the device-resident loop (mdb_solver_run), ODE and SDE: CUDA events, and a host clock
    around a device synchronise; plus the wall time of the public sampler call (prior draw and copy included);
  * the same number of ancestral steps through mdb_sampler_run (the configured 1000-step sampler's loop), and the
    999-step batch time extrapolated from it;
  * the update kernel alone (mdb_solver_update, second-order step, ODE and SDE with in-kernel Philox noise): time per
    launch and GB/s over the bytes it must move (12 read + 8 written per element, 4 of mask per voxel), against the
    H100 SXM data-sheet 3.35 TB/s.
The card's name, power limit and SM clock are read with nvidia-smi in the same run.

    python tools/bench_dpm_solver.py [--batch 32] [--steps 25] [--precisions bf16x3,bf16] [--out path.json]
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


def _timed(fn):
    """(CUDA-event ms, host-clock ms around a synchronise) of one call."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3


def bench_mode(precision, B, K, device):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    cfg, model = _model(precision, device)
    net = model.module
    R = cfg.data.image_size
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
    mask = net.state_dict()["mask"].view(R, R, R).to(device).contiguous()
    mask_flat = mask.reshape(-1)
    x0 = (torch.randn(B, 4, R, R, R, device=device) * mask).contiguous()
    r = {"precision": precision, "batch": B, "res": R}
    with torch.no_grad():
        # ancestral loop (mdb_sampler_run) over the first K steps of the 1000-step schedule
        ts = torch.linspace(sde.T, 1e-3, sde.N, device=device)
        idx = (ts * (sde.N - 1)).long()
        labels = (ts * (sde.N - 1)).cpu().tolist()
        betas, stds = sde.discrete_betas[idx].cpu().tolist(), sde.sqrt_1m_alphas_cumprod[idx].cpu().tolist()
        x = x0.clone()
        sampling._native_loop(net, x, mask_flat, labels, betas, stds, 2, 1)  # engine set-up on the timed buffers
        x.copy_(x0)
        ev, host = _timed(lambda: sampling._native_loop(net, x, mask_flat, labels, betas, stds, K, 1))
        r["ancestral"] = {"steps": K, "event_ms": ev, "host_ms": host, "ms_per_step": ev / K,
                          "extrapolated_999_steps_s": ev / K * (sde.N - 1) / 1e3}
        for stochastic in (False, True):
            key = "sde" if stochastic else "ode"
            lab, table = sampling.dpm_solver_schedule(sde, K, stochastic)
            entries_c = sampling._entries_c(table)
            x, hist = x0.clone(), torch.empty_like(x0)
            sampling._native_run(net, x, hist, mask_flat, entries_c, 1, 0, 2)
            x.copy_(x0)
            ev, host = _timed(lambda: sampling._native_run(net, x, hist, mask_flat, entries_c, 1))
            cfg.sampling.method, cfg.sampling.dpm_steps, cfg.sampling.dpm_sde = "dpm_solver", K, stochastic
            cfg.sampling.native_rng = True
            fn = sampling.get_sampling_fn(cfg, sde, (B, 4, R, R, R), lambda t: t, 1e-3, grid_mask=mask.view(1, R, R, R))
            nfe = [None]

            def call():
                nfe[0] = fn(model)[1]
            _, public = _timed(call)
            r[f"dpm_{key}"] = {"nfe": nfe[0], "event_ms": ev, "host_ms": host, "public_call_ms": public,
                               "speedup_vs_999_ancestral": r["ancestral"]["extrapolated_999_steps_s"] * 1e3 / host}
            # the update kernel alone, on a second-order step
            eps = torch.randn_like(x0)
            xk, hk = x0.clone(), torch.randn_like(x0)
            for _ in range(3):
                sampling._update(eps, xk, hk, mask_flat, entries_c[3], seed=1, offset=12)
            reps = 200

            def launches():
                for _ in range(reps):
                    sampling._update(eps, xk, hk, mask_flat, entries_c[3], seed=1, offset=12)
            ev, _ = _timed(launches)
            V = R ** 3
            nbytes = B * 4 * V * 20 + V * 4
            us = ev / reps * 1e3
            r[f"update_kernel_{key}"] = {"us": us, "bytes": nbytes, "GB_per_s": nbytes / (us * 1e-6) / 1e9,
                                         "share_of_3.35TB_per_s": nbytes / (us * 1e-6) / HBM_BYTES_PER_S}
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--precisions", default="bf16x3,bf16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dpm_solver needs a GPU"
    device = torch.device("cuda:0")
    res = {"card_before": _card(), "runs": []}
    for p in args.precisions.split(","):
        r = bench_mode(p, args.batch, args.steps, device)
        print(json.dumps(r), flush=True)
        res["runs"].append(r)
    res["card_after"] = _card()
    print(json.dumps(res, indent=2))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=2)


if __name__ == "__main__":
    main()
