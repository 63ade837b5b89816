"""Times progressive distillation (`--mode=distill`) and the `distilled` sampler on synthetic weights:
  * mdb_distill_step, each phase, at res64 and batch 16 (mixed per-sample steps of a 512-step teacher): time per launch
    (CUDA events over 200 launches after a warm-up) and GB/s over the bytes each phase must move (phase 0: 12 per
    element, phase 1: 16, plus 4 of mask per voxel), against the H100 SXM data-sheet 3.35 TB/s;
  * one distillation iteration at res64, micro-batch 16 (or the largest of 8, 4, 2, 1 that fits), per operand mode (the same mode for
    the teacher's inference plan and the student's training plan), split into teacher targets (perturb + mdb_distill_targets), student forward +
    loss + backward, and optimiser (clip + FusedAdam + EMA): CUDA events, mean of 5 iterations after 2 warm-ups, and the
    device memory left free with both engines resident;
  * the largest res128 micro-batch (of 8, 4, 2, 1) at which one bf16 iteration runs with both engines resident;
  * uncond_gen sampling at res64, batch 32, bf16x3: `distilled` K = 8 against `dpm_solver` K = 25, alternated twice,
    through the device-resident loop (host clock around a device synchronise).
The card's name, power limit and SM clock are read with nvidia-smi in the same run.

Each micro-batch attempt runs in a fresh process, so one that runs out of memory cannot fail the next.

    python tools/bench_distill.py [--out path.json] [--skip-res128] [--skip-sampling]
"""
import argparse
import gc
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


def _config(res, precision, device):
    from configs import res64, res128
    cfg = (res128 if res == 128 else res64).get_config()
    cfg.model.compute_dtype = precision
    cfg.training.compute_dtype = precision
    cfg.device = device
    return cfg


def _teacher(cfg):
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth
    model = mutils.create_model(cfg)
    net = model.module
    net.load_state_dict(synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=11))
    model.eval()
    return model


def _events(fn, reps=1):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def bench_kernel(device, B=16, R=64):
    from meshdiffusion_b200.diffusion import distill, sde_lib
    sde = sde_lib.VPSDE(0.1, 20.0, 1000, device=device)
    rows = distill.rows_tensor(sde, 512, device)
    V = R ** 3
    z_s, eps = torch.randn(B, 4, R, R, R, device=device), torch.randn(B, 4, R, R, R, device=device)
    z_mid, out = torch.empty_like(z_s), torch.empty_like(z_s)
    mask = (torch.rand(V, device=device) < 0.12).float()
    idx = torch.randint(0, 256, (B,), device=device, dtype=torch.int32)
    labels = torch.empty(B, device=device)
    r = {}
    for phase, per_elem in ((0, 12), (1, 16)):
        fn = lambda: distill.distill_step(eps, z_s, z_mid, out, mask, idx, rows, phase, labels)
        _events(fn, 5)
        us = _events(fn, 200) * 1e3
        nbytes = B * 4 * V * per_elem + V * 4
        r[f"phase{phase}"] = {"us": us, "bytes": nbytes, "GB_per_s": nbytes / (us * 1e-6) / 1e9,
                              "share_of_3.35TB_per_s": nbytes / (us * 1e-6) / HBM_BYTES_PER_S}
    return r


def _iteration_parts(cfg, B, n_warm, n_timed):
    """Per-part CUDA-event ms of distillation iterations (means over n_timed after n_warm), and free memory."""
    from meshdiffusion_b200.diffusion import distill
    teacher = _teacher(cfg)
    models = [teacher]
    try:
        state = distill.student_state(cfg, teacher, 2e-5)
        models.append(state["model"])
        return _iterations(cfg, B, n_warm, n_timed, teacher, state)
    finally:  # also after an out-of-memory error: free both engines before the next attempt
        for m in models:
            m.module.release_engine()
        del models, teacher
        gc.collect()
        torch.cuda.empty_cache()


def _iterations(cfg, B, n_warm, n_timed, teacher, state):
    from meshdiffusion_b200 import train_ops
    from meshdiffusion_b200.diffusion import distill, sde_lib, trainer
    from meshdiffusion_b200.diffusion.models import utils as mutils
    device = cfg.device
    R = cfg.data.image_size
    mask = teacher.module.state_dict()["mask"].view(1, 1, R, R, R).to(device)
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
    rows = distill.rows_tensor(sde, 512, device)
    model, optimizer, ema = state["model"], state["optimizer"], state["ema"]
    optimize_fn = trainer.data_parallel_optimize_fn(cfg, model.module, warmup=0)
    mask_flat = mask.reshape(-1).contiguous()
    mask_sum = float(mask_flat.sum().item())
    sums = {"targets_ms": 0.0, "student_fwd_bwd_ms": 0.0, "optimizer_ms": 0.0}
    batch = torch.randn(B, 4, R, R, R, device=device) * mask
    for it in range(n_warm + n_timed):
        idx = torch.randint(0, 256, (B,), device=device, dtype=torch.int32)
        labels = rows[idx.long(), 0].contiguous()
        t = labels.long()
        box = {}

        def targets():
            z_s = train_ops.ddpm_perturb(batch, torch.randn_like(batch), mask, sde.sqrt_alphas_cumprod[t],
                                         sde.sqrt_1m_alphas_cumprod[t])
            box["z_s"] = z_s
            box["target"] = distill.distill_targets(teacher.module, z_s, idx, rows, mask_flat, labels)

        def fwd_bwd():
            optimizer.zero_grad()
            pred = mutils.get_model_fn(model, train=True)(box["z_s"], labels)
            train_ops.DDPMLossFn.apply(pred, box["target"], mask, mask_sum).backward()

        def opt():
            if optimize_fn(optimizer, model.parameters(), step=state["step"], ema=ema) is not True:
                ema.update(model.parameters())
            state["step"] += 1
        parts = {"targets_ms": _events(targets), "student_fwd_bwd_ms": _events(fwd_bwd), "optimizer_ms": _events(opt)}
        if it >= n_warm:
            for k, v in parts.items():
                sums[k] += v / n_timed
    free, total = torch.cuda.mem_get_info()
    sums["iteration_ms"] = sum(sums.values())
    sums["free_gb_with_both_engines"] = free / 1e9
    sums["total_gb"] = total / 1e9
    return sums


def largest_fit(res, precision, batches, n_warm, n_timed):
    """One record per micro-batch tried, largest first, until one iteration runs with both engines resident. Every
    attempt runs in a process of its own, so memory an out-of-memory attempt left behind cannot fail the next one."""
    out = []
    for B in batches:
        cmd = [sys.executable, os.path.abspath(__file__), "--fit", f"{res},{precision},{B},{n_warm},{n_timed}"]
        p = subprocess.run(cmd, capture_output=True, text=True)
        lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
        r = json.loads(lines[-1]) if lines else {"precision": precision, "res": res, "micro_batch": B, "fits": False,
                                                  "error": (p.stderr or "no output")[-300:]}
        out.append(r)
        print(json.dumps(r), flush=True)
        if r["fits"]:
            break
    return out


def _fit_attempt(spec, device):
    res, precision, B, n_warm, n_timed = spec.split(",")
    r = {"precision": precision, "res": int(res), "micro_batch": int(B)}
    try:
        r.update(_iteration_parts(_config(int(res), precision, device), int(B), int(n_warm), int(n_timed)))
        r["fits"] = True
    except (torch.OutOfMemoryError, RuntimeError) as e:
        r.update(fits=False, error=str(e)[:300])
    print(json.dumps(r), flush=True)


def bench_sampling(device, B=32, rounds=2):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    cfg = _config(64, "bf16x3", device)
    model = _teacher(cfg)
    R = cfg.data.image_size
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
    g = model.module.state_dict()["mask"].view(1, R, R, R).to(device)
    fns = {"distilled_K8": sampling.get_distilled_sampler(sde, (B, 4, R, R, R), lambda x: x, 8, device=device,
                                                         grid_mask=g, native_rng=True),
           "dpm_solver_K25": sampling.get_dpm_solver_sampler(sde, (B, 4, R, R, R), lambda x: x, 25, device=device,
                                                             grid_mask=g, native_rng=True)}
    times = {k: [] for k in fns}
    nfe = {}
    fns["distilled_K8"](model)  # engine build and first launches
    for _ in range(rounds):
        for k, fn in fns.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            nfe[k] = fn(model)[1]
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    model.module.release_engine()
    r = {"batch": B, "precision": "bf16x3", "seconds": times, "nfe": nfe}
    r["speedup"] = min(times["dpm_solver_K25"]) / min(times["distilled_K8"])
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-res128", action="store_true")
    ap.add_argument("--skip-sampling", action="store_true")
    ap.add_argument("--fit", default=None, help=argparse.SUPPRESS)  # one attempt of largest_fit: res,precision,B,warm,timed
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_distill needs a GPU"
    device = torch.device("cuda:0")
    if args.fit:
        return _fit_attempt(args.fit, device)
    res = {"card_before": _card()}
    res["kernel"] = bench_kernel(device)
    print(json.dumps(res["kernel"]), flush=True)
    res["iteration"] = []
    for p in ("bf16", "bf16x3"):
        res["iteration"] += largest_fit(64, p, (16, 8, 4, 2, 1), 2, 5)
    if not args.skip_sampling:
        res["sampling"] = bench_sampling(device)
        print(json.dumps(res["sampling"]), flush=True)
    if not args.skip_res128:
        res["res128_fit"] = largest_fit(128, "bf16", (8, 4, 2, 1), 1, 2)
    res["card_after"] = _card()
    print(json.dumps(res, indent=2))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=2)


if __name__ == "__main__":
    main()
