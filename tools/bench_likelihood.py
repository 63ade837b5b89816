"""Times the probability-flow likelihood (diffusion/likelihood.py) on synthetic weights.

Per operand mode (bf16x3 and bf16), at the given resolution and batch:
  * one function evaluation of the native path -- training-plan forward + input-only backward (`mdb_unet_backward_input`
    with grads = NULL) + the fused `mdb_pflow_drift_div` -- next to forward + the full backward (parameter gradients
    and dx), so the saving from skipping the parameter gradients is measured, with CUDA events after a warm-up;
  * the NFE and wall seconds (host clock around a device synchronise) of one `likelihood_fn` batch of synthetic grids
    (trainer.synthetic_grids, masked by the tet-grid mask).
The card's name, power limit and SM clock are read with nvidia-smi in the same run.

    python tools/bench_likelihood.py [--config res64] [--batch 8] [--reps 10] [--precisions bf16x3,bf16] [--out path.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}


def _model(config, precision, device):
    from configs import res64, res128
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth
    cfg = (res128 if config == "res128" else res64).get_config()
    cfg.model.compute_dtype = precision
    cfg.training.compute_dtype = precision
    cfg.device = device
    model = mutils.create_model(cfg)
    net = model.module
    net.load_state_dict(synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=11))
    model.eval()
    return cfg, model


def bench_nfe(net, x, labels, h, mask, reps):
    from meshdiffusion_b200 import _native
    L = _native.lib()
    B, C = x.shape[:2]
    V = x[0, 0].numel()
    eng = net._diff_engine(net.precision, B, x.device)
    numel = ctypes.c_longlong()
    _native.check(L.mdb_unet_train_info(eng, None, None, ctypes.byref(numel)))
    grads = torch.zeros(numel.value, device=x.device)
    out, dx, drift = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    div = torch.empty(B, device=x.device, dtype=torch.float64)
    _native.check(L.mdb_unet_set_dropout(eng, 0.0, 0))
    s = _native.current_stream()

    def input_only():
        _native.check(L.mdb_unet_forward(eng, _native.ptr(x), _native.ptr(labels), _native.ptr(out), B, s))
        _native.check(L.mdb_unet_backward_input(eng, _native.ptr(h), _native.ptr(dx), None, 0, B, 0, s))
        _native.check(L.mdb_pflow_drift_div(_native.ptr(x), _native.ptr(out), _native.ptr(h), _native.ptr(dx), _native.ptr(mask),
                                            7.0, 0.5, _native.ptr(drift), _native.ptr(div), B, C, V, s))

    def full():
        _native.check(L.mdb_unet_forward(eng, _native.ptr(x), _native.ptr(labels), _native.ptr(out), B, s))
        _native.check(L.mdb_unet_backward_input(eng, _native.ptr(h), _native.ptr(dx), _native.ptr(grads), numel.value, B, 0, s))

    res = {}
    for name, fn in (("input_only_ms", input_only), ("forward_full_backward_ms", full), ("input_only_ms_repeat", input_only)):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name] = e0.elapsed_time(e1) / reps
    return res


def run(config="res64", batch=8, reps=10, precisions=("bf16x3", "bf16"), rtol=1e-3, atol=1e-3):
    from meshdiffusion_b200.diffusion import likelihood, sde_lib
    from meshdiffusion_b200.diffusion.evaler import load_grid_mask
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    assert torch.cuda.is_available(), "bench_likelihood needs a CUDA device"
    device = torch.device("cuda:0")
    out = {"card": _card(), "config": config, "batch": batch, "reps": reps, "rtol": rtol, "atol": atol, "runs": []}
    for prec in precisions:
        cfg, model = _model(config, prec, device)
        net = model.module
        R = cfg.data.image_size
        mask = load_grid_mask(R, device).view(R, R, R).float()
        gen = torch.Generator(device=device).manual_seed(0)
        data = synthetic_grids(batch, R, device, gen) * mask
        noise = likelihood.hutchinson_noise(data, "Rademacher", generator=torch.Generator(device=device).manual_seed(1)) * mask
        labels = torch.full((batch,), 500.0, device=device)
        r = {"precision": prec}
        r.update(bench_nfe(net, data.contiguous(), labels, noise.contiguous(), mask.contiguous(), reps))
        r["saving_fraction"] = 1.0 - r["input_only_ms"] / r["forward_full_backward_ms"]
        print(json.dumps(r), flush=True)
        sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
        fn = likelihood.get_likelihood_fn(sde, lambda t: t, rtol=rtol, atol=atol, grid_mask=mask)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        bpd, _, nfe = fn(model, data, noise=noise)
        torch.cuda.synchronize()
        r.update(likelihood_seconds=time.perf_counter() - t0, likelihood_nfe=int(nfe), bpd=[float(b) for b in bpd])
        r["seconds_per_nfe"] = r["likelihood_seconds"] / max(1, r["likelihood_nfe"])
        print(json.dumps(r), flush=True)
        out["runs"].append(r)
        net.release_engine()
        del model, net
        torch.cuda.empty_cache()
    out["card_after"] = _card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="res64")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--precisions", default="bf16x3,bf16")
    # synthetic weights make a stiff field (a tiny network needs ~1100 evaluations at 1e-5): the default tolerance keeps
    # one batch to minutes
    ap.add_argument("--rtol", type=float, default=1e-3)
    ap.add_argument("--atol", type=float, default=1e-3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = run(a.config, a.batch, a.reps, tuple(a.precisions.split(",")), a.rtol, a.atol)
    print(json.dumps(res, indent=2))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=2)


if __name__ == "__main__":
    main()
