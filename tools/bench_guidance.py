"""Times classifier-free guidance on a class-conditional res64 network with synthetic weights:
  * the guided solver entry alone (mdb_solver_update_guided, second-order ODE step) against the plain entry
    (mdb_solver_update) at the same shape: time per launch and TB/s over the bytes each must move (guided: eps_c, eps_u,
    x, x0_hist read, x and x0_hist written, fp32, plus the mask; plain: the same without eps_u);
  * one K-step guided dpm_solver batch (mdb_solver_run_guided, w = 3) against the unguided conditional one (w = 1), per
    operand mode: CUDA events around the public sampler call;
  * one bf16 training step (forward + backward, micro-batch 16) of a K = 5 network against K = 0, alternated three
    times (median of 5 steps each), with the spread of the per-round medians.
The card's name, power limit and SM clock are read with nvidia-smi in the same run.

    python tools/bench_guidance.py [--batch 32] [--steps 25] [--precisions bf16x3,bf16] [--out path.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_dpm_solver import HBM_BYTES_PER_S, _card, _timed  # noqa: E402


def _model(precision, num_classes, device, train_precision="bf16"):
    from configs import res64
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth
    cfg = res64.get_config()
    cfg.model.compute_dtype = precision
    cfg.training.compute_dtype = train_precision
    cfg.model.num_classes = num_classes
    cfg.model.dropout = 0.0
    cfg.device = device
    model = mutils.create_model(cfg)
    net = model.module
    sd = synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=11)
    if num_classes:
        sd["label_embed.weight"] = torch.randn(num_classes + 1, 4 * cfg.model.nf, generator=torch.Generator().manual_seed(1))
    net.load_state_dict(sd)
    model.eval()
    return cfg, model


def _median_ms(fn, reps):
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]))


def bench_entry(B, R, reps=50):
    from meshdiffusion_b200.diffusion import sampling
    shape = (B, 4, R, R, R)
    g = torch.Generator(device="cuda").manual_seed(0)
    eps_c, eps_u, x, h = (torch.randn(shape, device="cuda", generator=g) for _ in range(4))
    mask = torch.ones(R ** 3, device="cuda")
    row = np.array([[0, 500, 0.6, 1.3, 0.9, 0.4, -0.2, 0.0, 0.0, 0.0]], np.float32)
    entry = sampling._entries_c(row)[0]
    n = x.numel()
    out = {}
    for name, kw, nbytes in (("plain", {}, 5 * 4 * n + 4 * R ** 3), ("guided", dict(eps_u=eps_u, w=3.0), 6 * 4 * n + 4 * R ** 3)):
        fn = lambda: sampling._update(eps_c, x, h, mask, entry, **kw)  # noqa: E731
        for _ in range(5):
            fn()
        ms = _median_ms(fn, reps)
        out[name] = {"ms": ms, "bytes": nbytes, "tb_per_s": nbytes / ms / 1e9, "share_of_hbm_peak": nbytes / ms / 1e-3 / HBM_BYTES_PER_S}
    return out


def bench_sampler(precision, B, steps, device):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    cfg, model = _model(precision, 5, device)
    R = cfg.data.image_size
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
    y = (torch.arange(B, device=device) % 5).to(torch.int32)
    res = {}
    for w in (1.0, 3.0):
        fn = sampling.get_dpm_solver_sampler(sde, (B, 4, R, R, R), lambda v: v, n_steps=steps, device=device,
                                             grid_mask=torch.ones(R, R, R, device=device), native_rng=True, guidance_scale=w)
        fn(model, class_labels=y)  # warm-up: engine, graphs
        ev, host = _timed(lambda: fn(model, class_labels=y))
        res[f"w{w:g}"] = {"event_ms": ev, "host_ms": host}
    res["ratio_guided_over_unguided"] = res["w3"]["event_ms"] / res["w1"]["event_ms"]
    model.module.release_engine()
    del model
    torch.cuda.empty_cache()
    return res


def bench_train(device, K, B=16, reps=5):
    cfg, model = _model("bf16", K, device)
    net = model.module
    R = cfg.data.image_size
    g = torch.Generator(device=device).manual_seed(0)
    x = torch.randn(B, 4, R, R, R, device=device, generator=g)
    labels = torch.randint(0, 1000, (B,), device=device, generator=g).float()
    y = (torch.arange(B, device=device) % K).to(torch.int32) if K else None

    def step():
        net.train()
        out = model(x, labels) if y is None else model(x, labels, class_labels=y)
        out.square().mean().backward()

    for _ in range(2):
        step()
    ms = _median_ms(step, reps)
    net.release_engine()
    del model
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--precisions", default="bf16x3,bf16")
    ap.add_argument("--out", default=None)
    ap.add_argument("--train-only", action="store_true", help="skip the sampler comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_guidance needs a CUDA device")
    device = torch.device("cuda:0")
    torch.cuda.set_device(device)
    result = {"card": _card(), "batch": args.batch, "steps": args.steps}
    result["entry_res64"] = bench_entry(args.batch, 64)
    if not args.train_only:
        result["sampler"] = {p: bench_sampler(p, args.batch, args.steps, device) for p in args.precisions.split(",")}
    # K = 0 and K = 5 alternated, one engine at a time, so slow drift of the clock or the host falls on both
    runs = {0: [], 5: []}
    for _ in range(3):
        for K in (0, 5):
            runs[K].append(bench_train(device, K))
    result["train_step_bf16_mb16_ms"] = {
        f"K{K}": {"median": float(np.median(v)), "min": min(v), "max": max(v), "runs": v} for K, v in runs.items()}
    result["train_step_bf16_mb16_ms"]["ratio_of_medians"] = float(np.median(runs[5]) / np.median(runs[0]))
    result["card_after"] = _card()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
