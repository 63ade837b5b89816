"""Per-launch view of the implicit-GEMM kernel in one res64 forward: where the time goes, at what tensor-instruction rate
and at what shared-memory fill rate.

One forward at batch 32 (synthetic weights, seeded input) in the given operand mode, timed per launch with CUDA events
(`ScoreNet.profile`, best of --reps forwards per launch after --warmup forwards). For every GEMM launch it prints the
time, the issued TFLOP/s (executed FLOPs x tensor instructions per product: 1 bf16, 2 tf32, 3 bf16x3, over the time)
and the fill rate (bytes TMA writes into shared memory, from `mdb_unet_gemm_ops`, over the time), then the ten
slowest launches with their operand ring depth (A / B slots from `mdb_unet_gemm_slots`: MDB_MAX_STAGES and MDB_MAX_BSLOTS
cap them), then the per-tile fit of `tile_fits`: launches grouped by tile geometry and entry shape
(`mdb_unet_gemm_tiles`), microseconds per CTA tile against k-steps per tile, whose intercept is the cost per output tile
that does not grow with K. The card's name, power limit and SM clock are read in the same process.

    python tools/bench_gemm_ops.py --precision bf16x3 [--batch 32] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
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
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rows = []
    for (name, flops, fill), (a_slots, b_slots, smem), (work, splits, ksteps, entry_ksteps, block_n) in zip(
            ops, net.gemm_slots(), net.gemm_tiles()):
        ms = best[name]
        rows.append({"name": name, "ms": ms, "flops": flops, "fill_bytes": fill,
                     "issued_tflops": flops * per / (ms * 1e-3) / 1e12, "fill_gbs": fill / (ms * 1e-3) / 1e9,
                     "a_slots": a_slots, "b_slots": b_slots, "smem_bytes": smem,
                     "work_items": work, "ctas": min(work, sms), "splits": splits, "ksteps_per_tile": ksteps / splits,
                     "entry_ksteps": entry_ksteps, "block_n": block_n})
    forward_ms = sum(best.values())
    gemm_ms = sum(r["ms"] for r in rows)
    net.release_engine()
    return {"precision": precision, "batch": batch, "card": clock_during, "forward_ms": forward_ms, "gemm_ms": gemm_ms,
            "gemm_flops": sum(r["flops"] for r in rows), "gemm_fill_bytes": sum(r["fill_bytes"] for r in rows), "ops": rows,
            "tile_fits": tile_fits(rows)}


def tile_fits(rows):
    """Per group of launches with the same tile geometry and entry shape (work items, CTAs, split-K factor, BLOCK_N, most
    k-steps per entry): a least-squares line through (k-steps per tile, microseconds per CTA tile). A CTA tile is the
    launch time over the work items of the busiest CTA (the persistent CTAs take work items round-robin), so the slope is
    the cost of one k-step of a tile and the intercept the cost per tile that does not grow with K (epilogue, tile
    set-up, pipeline fill and drain). Groups whose launches all have the same k-steps per tile have no fit."""
    groups = {}
    for r in rows:
        key = (r["work_items"], r["ctas"], r["splits"], r["block_n"], r["entry_ksteps"])
        groups.setdefault(key, []).append(r)
    fits = []
    for (work, ctas, splits, block_n, entry_ksteps), rs in groups.items():
        per_cta = -(-work // ctas)
        xs = np.array([r["ksteps_per_tile"] for r in rs])
        ys = np.array([r["ms"] * 1e3 / per_cta for r in rs])
        # per k-steps value: launches, mean microseconds per CTA tile, issued TFLOP/s range
        by_k = [{"ksteps": k, "launches": int((xs == k).sum()), "us_per_cta_tile": float(ys[xs == k].mean()),
                 "issued_tflops": [min(r["issued_tflops"] for r in rs if r["ksteps_per_tile"] == k),
                                   max(r["issued_tflops"] for r in rs if r["ksteps_per_tile"] == k)]}
                for k in sorted(set(xs.tolist()))]
        fit = {"work_items": work, "ctas": ctas, "tiles_per_cta": per_cta, "splits": splits, "block_n": block_n,
               "entry_ksteps": entry_ksteps, "launches": len(rs), "ms": sum(r["ms"] for r in rs), "by_ksteps": by_k,
               "us_per_kstep": None, "us_per_tile": None, "rms_us": None}
        if len(by_k) >= 2:
            slope, icept = np.polyfit(xs, ys, 1)
            fit.update(us_per_kstep=float(slope), us_per_tile=float(icept),
                       rms_us=float(np.sqrt(np.mean((ys - (slope * xs + icept)) ** 2))))
        fits.append(fit)
    return sorted(fits, key=lambda f: -f["ms"])


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
    print("per-tile fit (us per CTA tile = slope x k-steps per tile + intercept), one group per tile geometry and entry "
          "shape, slowest group first:")
    print(f"{'work items':>11}{'CTAs':>6}{'tiles/CTA':>10}{'BLOCK_N':>8}{'k/entry':>8}{'launches':>9}{'ms':>9}"
          f"{'us/k-step':>11}{'us/tile':>9}{'rms us':>8}")
    for f in r["tile_fits"]:
        fit = (f"{f['us_per_kstep']:>11.3f}{f['us_per_tile']:>9.1f}{f['rms_us']:>8.1f}" if f["us_per_kstep"] is not None
               else f"{'-':>11}{'-':>9}{'-':>8}")
        print(f"{f['work_items']:>11}{f['ctas']:>6}{f['tiles_per_cta']:>10}{f['block_n']:>8}{f['entry_ksteps']:>8}"
              f"{f['launches']:>9}{f['ms']:>9.1f}{fit}")
        if f["us_per_kstep"] is not None:
            for k in f["by_ksteps"]:
                lo, hi = k["issued_tflops"]
                print(f"{'':>11}  {k['ksteps']:g} k-steps per tile: {k['launches']} launches, "
                      f"{k['us_per_cta_tile']:.1f} us per CTA tile, {lo:.0f}-{hi:.0f} issued TFLOP/s")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
