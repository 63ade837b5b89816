"""HBM rate of the optimiser-side passes on the real parameter set (res64: 494 trainable tensors, 364 M fp32 values):
clip-coefficient reduction (mdb_grad_clip_coef: reads g), Adam + EMA in one pass (mdb_adam_ema_step: reads p, g, m, v, ema and
writes p, m, v, ema = 36 B per parameter), and the stand-alone EMA update (mdb_ema_update: 12 B per parameter).

    python tools/bench_optimizer.py [--steps 20]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    from configs import res64
    from meshdiffusion_b200 import train_ops
    from meshdiffusion_b200.diffusion.models import ddpm
    from meshdiffusion_b200.diffusion.models.ema import ExponentialMovingAverage
    dev = torch.device("cuda:0")
    table = ddpm.param_table(ddpm.arch_from_config(res64.get_config()))
    g = torch.Generator(device=dev).manual_seed(0)
    params = [torch.nn.Parameter(torch.randn(s, device=dev, generator=g) * 0.05) for n, s in table if n not in ("mask", "coords")]
    flat = torch.randn(sum(p.numel() for p in params), device=dev, generator=g) * 1e-3
    off = 0
    for p in params:  # gradients are views of ONE flat buffer, as the engine hands them out
        p.grad = flat[off:off + p.numel()].view(p.shape)
        off += p.numel()
    n = off
    opt = train_ops.FusedAdam(params, lr=2e-5, betas=(0.9, 0.999), eps=1e-8)
    ema = ExponentialMovingAverage(params, decay=0.9999)
    peak = 3350.0  # GB/s, H100 SXM data sheet (HBM3)
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    res = {}
    for name, fn, bytes_per in (("clip_coef (read g)", lambda: opt.grad_norm_coef(1.0), 4),
                                ("adam+ema one pass", lambda: opt.step(ema=ema), 36),
                                ("clip + adam+ema (the optimiser step)", lambda: (opt.grad_norm_coef(1.0), opt.step(ema=ema)), 40),
                                ("ema alone", lambda: ema.update(params), 12)):
        ms = timed(fn)
        gbs = n * bytes_per / (ms * 1e-3) / 1e9
        res[name] = {"ms": ms, "GBps": gbs, "frac_of_hbm_peak": gbs / peak}
    print(json.dumps({"parameters": n, "tensors": len(params), "hbm_peak_GBps": peak, "includes": "host-side launch overhead of the Python wrapper (pointer-table cache hit)", **res}))


if __name__ == "__main__":
    main()
