"""Chamfer-matrix throughput at the size a user of `--mode=eval_metrics` runs, one GPU.

    python tools/bench_pc_metrics.py [--clouds 1000] [--points 2048] [--repeats 3] [--host-pairs 8]

One workload = the 1000 x 1000 cross matrix (generated x reference) plus one 1000-cloud self matrix, 2048 points per
cloud, on seeded clouds (the kernel's cost does not depend on their content). After a warm-up workload, `repeats`
workloads are timed back to back with CUDA events (a multi-second window). The card's name, power limit and SM clock are
read with nvidia-smi while the timed window is running.

Reported: seconds per workload; point-pair evaluations per second; the share of an FP32 issue bound, defined here as
pairs x 8 instructions (3 FADD, 1 FMUL, 2 FFMA, 2 FMNMX per pair) / (132 SMs x 128 lanes x the SM clock read during the
run); and, for context, the per-pair time of the cKDTree oracle on the host over `host-pairs` pairs (which also checks
those entries of the device matrix).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

INSTR_PER_PAIR = 8
H100_SMS, FP32_LANES_PER_SM = 132, 128


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, default=1000)
    ap.add_argument("--points", type=int, default=2048)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-pairs", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pc_metrics needs a CUDA device")
    from meshdiffusion_b200.geometry.pointcloud import chamfer_matrix
    from oracle import pc_metrics_oracle as pco
    dev = torch.device("cuda:0")
    n, N = args.clouds, args.points
    g = torch.Generator(device=dev).manual_seed(0)
    gen = torch.rand(n, N, 3, device=dev, generator=g) - 0.5
    ref = torch.rand(n, N, 3, device=dev, generator=g) - 0.5

    def workload():
        return chamfer_matrix(gen, ref), chamfer_matrix(gen)

    workload()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.repeats):
        cross, self_ = workload()
    e1.record()
    time.sleep(min(1.0, 0.1 * args.repeats))  # read the card while the enqueued window runs
    card = _card()
    torch.cuda.synchronize()
    seconds = e0.elapsed_time(e1) * 1e-3 / args.repeats
    pairs = n * n * N * N + n * (n - 1) // 2 * N * N
    bound_s = pairs * INSTR_PER_PAIR / (H100_SMS * FP32_LANES_PER_SM * card["sm_clock_mhz"] * 1e6)

    # host context: the cKDTree oracle on a sample of the cross pairs, checked against the device entries
    rng = np.random.RandomState(1)
    idx = [(int(i), int(j)) for i, j in zip(rng.randint(0, n, args.host_pairs), rng.randint(0, n, args.host_pairs))]
    gh, rh, ch = gen.cpu().numpy(), ref.cpu().numpy(), cross.cpu().numpy()
    t0 = time.perf_counter()
    host = [pco.chamfer_kdtree(gh[i], rh[j]) for i, j in idx]
    host_per_pair = (time.perf_counter() - t0) / len(idx)
    rel = max(abs(ch[i, j] - h) / h for (i, j), h in zip(idx, host))
    print(json.dumps({
        "metric": "chamfer matrix", "clouds": n, "points": N, "repeats": args.repeats,
        "workload": f"{n}x{n} cross + {n}-cloud self matrix",
        "seconds": seconds, "point_pairs": pairs, "pairs_per_s": pairs / seconds,
        "fp32_issue_bound_s": bound_s, "share_of_fp32_issue_bound": bound_s / seconds,
        "card": card,
        "host_ckdtree_s_per_cloud_pair": host_per_pair, "host_ckdtree_s_for_workload_est": host_per_pair * (n * n + n * (n - 1) // 2),
        "device_vs_ckdtree_max_rel": rel,
        "self_diag_zero": bool((torch.diagonal(self_) == 0).all()),
    }))


if __name__ == "__main__":
    main()
