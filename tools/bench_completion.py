"""Times shape completion (`--mode=eval_completion`):
  * `mdb_chamfer_pairs` at the mode's size: one launch per group of batch / k partials holding the k ground-truth, the
    k (k - 1) / 2 TMD and the k partial->completion pairs of each, 2048 points per cloud, seeded clouds (the kernel's
    cost does not depend on their content). CUDA events over many launches after a warm-up; pairs per second and the
    share of an FP32 issue bound, point pairs x 8 instructions (3 FADD, 1 FMUL, 2 FFMA, 2 FMNMX) / (132 SMs x 128
    lanes x the SM clock read during the run), the bound tools/bench_pc_metrics.py uses for the Chamfer matrix;
  * one end-to-end run per operand mode on synthetic res64 grids and the network's default (untrained) weights:
    `--mode=make_partial` for `--shapes` shapes from view 0 at 1000^2, then `--mode=eval_completion` with k completions
    per partial by `dpm_solver` at K steps, split into the mode's phases (sampling, meshing and cloud sampling,
    distance kernels, file writes) from its own report; host clock around a device synchronise.
The card's name, power limit and SM clock are read with nvidia-smi in the same run. Prints one JSON line. Completion
quality is not measured: untrained weights say nothing about it.

    python tools/bench_completion.py [--shapes 16] [--k 8] [--batch 32] [--steps 25] [--precisions bf16x3,bf16]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

INSTR_PER_PAIR = 8
H100_SMS, FP32_LANES_PER_SM = 132, 128


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}


def bench_kernel(per_call, k, N=2048, iters=100):
    from meshdiffusion_b200.diffusion.completion import group_pairs
    from meshdiffusion_b200.geometry.pointcloud import chamfer_pairs
    n = per_call
    g = torch.Generator(device="cuda").manual_seed(0)
    clouds = torch.rand(2 * n + n * k, N, 3, device="cuda", generator=g) - 0.5
    pairs, _ = group_pairs(n, k, [True] * n, [True] * (n * k))
    for _ in range(5):
        chamfer_pairs(clouds, pairs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        chamfer_pairs(clouds, pairs)
    e1.record()
    card = _card()  # read while the tail of the window may still run; the clock the bound uses
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    point_pairs = len(pairs) * N * N
    bound_s = point_pairs * INSTR_PER_PAIR / (H100_SMS * FP32_LANES_PER_SM * card["sm_clock_mhz"] * 1e6)
    return {"partials_per_launch": n, "k": k, "points": N, "pairs_per_launch": len(pairs), "launches": iters,
            "ms_per_launch": ms, "pairs_per_s": len(pairs) / (ms * 1e-3), "point_pairs_per_s": point_pairs / (ms * 1e-3),
            "share_of_fp32_issue_bound": bound_s / (ms * 1e-3), "card_during": card}


def _config(tmp, precision, meta, k, batch, steps):
    from configs import res64
    from meshdiffusion_b200.geometry import dmtet
    cfg = res64.get_config()
    cfg.device = torch.device("cuda:0")
    cfg.model.compute_dtype = precision
    cfg.data.meta_path = meta
    cfg.eval.eval_dir = os.path.join(tmp, "eval")
    cfg.eval.ckpt_path = os.path.join(tmp, "missing", "checkpoint.pth")
    cfg.eval.tet_path = dmtet.tet_grid_path(64)
    cfg.eval.batch_size = batch
    cfg.eval.completion_k = k
    cfg.sampling.method = "dpm_solver"
    cfg.sampling.dpm_steps = steps
    return cfg


def bench_end_to_end(shapes, k, batch, steps, precisions):
    from meshdiffusion_b200.diffusion import completion, evaler
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        grids = synthetic_grids(shapes, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(2)).cpu()
        paths = []
        for i in range(shapes):
            paths.append(os.path.join(tmp, f"grid_{i}.pt"))
            torch.save(grids[i].clone(), paths[-1])
        meta = os.path.join(tmp, "meta.json")
        with open(meta, "w") as fh:
            json.dump(paths, fh)
        cfg = _config(tmp, precisions[0], meta, k, batch, steps)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        evaler.make_partial(cfg)
        torch.cuda.synchronize()
        out["make_partial_s"] = time.perf_counter() - t0
        for p in precisions:
            cfg = _config(tmp, p, meta, k, batch, steps)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rep = completion.eval_completion(cfg)
            torch.cuda.synchronize()
            out[p] = {"total_s": time.perf_counter() - t0, "phases_s": rep["seconds"], "nfe": rep["settings"]["nfe"],
                      "partials": rep["means"]["partials"], "samples": rep["means"]["partials"] * k,
                      "empty_completions": rep["means"]["empty_completions"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=16)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--precisions", default="bf16x3,bf16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_completion.py needs a CUDA GPU")
    torch.cuda.set_device(0)
    res = {"card": _card(), "kernel": bench_kernel(a.batch // a.k, a.k),
           "end_to_end": bench_end_to_end(a.shapes, a.k, a.batch, a.steps, a.precisions.split(",")),
           "settings": {"shapes": a.shapes, "k": a.k, "batch": a.batch, "dpm_steps": a.steps}}
    res["card_after"] = _card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
