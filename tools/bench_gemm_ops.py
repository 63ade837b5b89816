"""Per-launch view of the implicit-GEMM kernel in one res64 forward: where the time goes, at what tensor-instruction rate
and at what shared-memory fill rate.

One forward at batch 32 (synthetic weights, seeded input) in the given operand mode, timed per launch with CUDA events
(`ScoreNet.profile`, best of --reps forwards per launch after --warmup forwards). For every GEMM launch it prints the
time, the issued TFLOP/s (executed FLOPs x tensor instructions per product: 1 bf16, 2 tf32, 3 bf16x3, over the time)
and the fill rate (bytes TMA writes into shared memory, from `mdb_unet_gemm_ops`, over the time), then the ten
slowest launches with their operand ring depth (A / B slots from `mdb_unet_gemm_slots`: MDB_MAX_STAGES and MDB_MAX_BSLOTS
cap them). The card's name, power limit and SM clock are read in the same process.

    python tools/bench_gemm_ops.py --precision bf16x3 [--batch 32] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

MMA_PER_PRODUCT = {"bf16": 1.0, "tf32": 2.0, "bf16x3": 3.0}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "nvidia-smi unavailable"


def run(precision, batch=32, warmup=2, reps=3):
    import bench
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_ops needs a GPU")
    dev = torch.device("cuda:0")
    _, model = bench.build_model(precision, batch, dev, 64)
    net = model.module
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(batch, 4, 64, 64, 64, device=dev, generator=g)
    labels = torch.full((batch,), 500.0, device=dev)
    with torch.no_grad():
        for _ in range(warmup):
            model(x, labels)
    torch.cuda.synchronize()
    clock_during = None
    best = {}
    for _ in range(reps):
        for name, ms in net.profile(x, labels):
            best[name] = min(ms, best.get(name, float("inf")))
        clock_during = card()
    ops = net.gemm_ops()
    per = MMA_PER_PRODUCT[precision]
    rows = []
    for (name, flops, fill), (a_slots, b_slots, smem) in zip(ops, net.gemm_slots()):
        ms = best[name]
        rows.append({"name": name, "ms": ms, "flops": flops, "fill_bytes": fill,
                     "issued_tflops": flops * per / (ms * 1e-3) / 1e12, "fill_gbs": fill / (ms * 1e-3) / 1e9,
                     "a_slots": a_slots, "b_slots": b_slots, "smem_bytes": smem})
    forward_ms = sum(best.values())
    gemm_ms = sum(r["ms"] for r in rows)
    net.release_engine()
    return {"precision": precision, "batch": batch, "card": clock_during, "forward_ms": forward_ms, "gemm_ms": gemm_ms,
            "gemm_flops": sum(r["flops"] for r in rows), "gemm_fill_bytes": sum(r["fill_bytes"] for r in rows), "ops": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16x3", choices=list(MMA_PER_PRODUCT))
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write every launch's row here")
    a = ap.parse_args()
    r = run(a.precision, a.batch, a.warmup, a.reps)
    print(f"card (name, power limit, SM clock, max SM clock): {r['card']}")
    print(f"{a.precision} res64 batch {a.batch}: forward {r['forward_ms']:.1f} ms, GEMM launches {r['gemm_ms']:.1f} ms "
          f"({len(r['ops'])} launches, {r['gemm_flops'] / 1e12:.1f} TFLOP, {r['gemm_fill_bytes'] / 1e9:.1f} GB filled)")
    print(f"{'launch':<16}{'ms':>9}{'issued TFLOP/s':>16}{'fill GB/s':>11}{'slots A/B':>11}")
    for o in sorted(r["ops"], key=lambda o: -o["ms"])[:10]:
        slots = f"{o['a_slots']}/{o['b_slots']}"
        print(f"{o['name']:<16}{o['ms']:>9.2f}{o['issued_tflops']:>16.1f}{o['fill_gbs']:>11.0f}{slots:>11}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
