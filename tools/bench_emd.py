"""EMD-matrix throughput at the size a user of `--mode=eval_metrics --config.eval.metric_emd=True` runs, one GPU.

    python tools/bench_emd.py [--clouds 1000 200] [--points 2048] [--eps 1e-5] [--host-pairs 4] [--out PATH]

One workload = the n x n cross matrix (generated x reference) plus one n-cloud self matrix, 2048 points per cloud. The
auction's cost depends on the clouds (unlike Chamfer's), so they are surface samples of synthetic marching-tet shapes
(oracle.synth, clean and noisy fields), not uniform cubes. Each workload size runs once as a warm-up (a smaller launch of
the same kernel) and once timed with CUDA events; the card's name, power limit and SM clock are read with nvidia-smi while
the timed window runs.

Reported per size: seconds and cloud pairs per second; the largest certified gap; scan elements (cost evaluations) per
pair, counted by the float32 restatement `oracle.emd_oracle.emd_auction` on `host-pairs` of the cross pairs (which also
checks those device entries); the share of an FP32 issue bound, defined as scan elements x the compiled instructions per
element of the bidding loop (read from `cuobjdump -sass` of the library) / (132 SMs x 128 lanes x the SM clock); and, for
context, `scipy.optimize.linear_sum_assignment`'s per-pair host time.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

H100_SMS, FP32_LANES_PER_SM = 132, 128


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}


def instructions_per_element(lib_path):
    """Instructions the bidding scan issues per cost evaluation: the unrolled loop of emd_pair_kernel that evaluates costs
    (MUFU.RSQ) with no barrier, shuffle or fp64 instruction in it (the dual pass is the one with DADD), its instruction
    count over its MUFU.RSQ count. The
    out-of-line slow path of the square root (4 instructions around each CALL, for arguments below 2^-101) is not run."""
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", lib_path], capture_output=True, text=True, timeout=300).stdout
    ins, inside = [], False
    for line in sass.splitlines():
        if "Function :" in line:
            inside = "emd_pair_kernel" in line
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if inside and m:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    best = None
    for k, (addr, op) in enumerate(ins):
        m = re.search(r"BRA (0x[0-9a-f]+)$", op)
        if not m or int(m.group(1), 16) >= addr:
            continue
        body = [o for a, o in ins if int(m.group(1), 16) <= a <= addr]
        rsq = sum("MUFU.RSQ" in o for o in body)
        # the innermost loop: no barrier, shuffle or fp64 instruction inside
        if rsq == 0 or any(re.search(r"\b(BAR|SHFL|DADD|DSETP)\b", o) for o in body):
            continue
        n = len(body) - 4 * sum("CALL" in o for o in body) - sum(o.startswith("NOP") for o in body)
        if best is None or rsq > best[1]:
            best = (n, rsq)
    if best is None:
        raise RuntimeError("bidding loop not found in the SASS of emd_pair_kernel")
    return best[0] / best[1], best


def _clouds(n, N, first_seed):
    """n surface clouds of synthetic marching-tet shapes (res 64), alternating clean and noisy fields."""
    from meshdiffusion_b200.geometry import dmtet
    from meshdiffusion_b200.geometry.pointcloud import sample_surface_points
    from oracle import synth
    verts, idx = dmtet.load_tet_grid(64)
    out = []
    for c0 in range(0, n, 8):
        cases = [(first_seed + k, k % 2 == 1) for k in range(c0, min(n, c0 + 8))]
        sdfs, poss = zip(*[synth.synthetic_dmtet(verts, seed=s, noisy=z, res=64) for s, z in cases])
        mt = dmtet.MarchingTets(idx, verts.shape[0], max_batch=len(cases))
        v, f, _, _, _, off = mt._extract_raw(torch.tensor(np.stack(poss)).cuda(), torch.tensor(np.stack(sdfs)).cuda())
        pts, empty = sample_surface_points(v, f, off[:, 0], off[:, 1], N, seed=first_seed, first_id=c0)
        out.append(pts[~empty])
    return torch.cat(out)


def run(n, N, eps, host_pairs, ipe, lsa_pairs):
    from meshdiffusion_b200.geometry.pointcloud import emd_matrix
    from oracle import emd_oracle as eo
    gen, ref = _clouds(n, N, 0), _clouds(n, N, 100000)
    n_g, n_r = gen.shape[0], ref.shape[0]
    emd_matrix(gen[:8], ref[:8], eps)  # warm-up: module load, smem attribute
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    cross, gcross = emd_matrix(gen, ref, eps)
    self_, gself = emd_matrix(gen, eps=eps)
    e1.record()
    time.sleep(1.0)  # read the card while the enqueued window runs
    card = _card()
    torch.cuda.synchronize()
    seconds = e0.elapsed_time(e1) * 1e-3
    pairs = n_g * n_r + n_g * (n_g - 1) // 2
    rng = np.random.RandomState(1)
    idx = [(int(i), int(j)) for i, j in zip(rng.randint(0, n_g, host_pairs), rng.randint(0, n_r, host_pairs))]
    gh, rh, ch = gen.cpu().numpy(), ref.cpu().numpy(), cross.cpu().numpy()
    scans, dev_vs_host = [], 0.0
    for i, j in idx:
        e, _, s = eo.emd_auction(gh[i], rh[j], eps)
        scans.append(s)
        dev_vs_host = max(dev_vs_host, abs(e - ch[i, j]))
    scan_per_pair = float(np.mean(scans))
    t0 = time.perf_counter()
    lsa = [eo.emd_exact(gh[i], rh[j]) for i, j in idx[:lsa_pairs]]
    lsa_per_pair = (time.perf_counter() - t0) / max(1, len(lsa))
    lsa_excess = max((ch[i, j] - x for (i, j), x in zip(idx, lsa)), default=0.0)
    bound_s = pairs * scan_per_pair * ipe / (H100_SMS * FP32_LANES_PER_SM * card["sm_clock_mhz"] * 1e6)
    return {
        "metric": "emd matrix", "clouds": [n_g, n_r], "points": N, "eps": eps,
        "workload": f"{n_g}x{n_r} cross + {n_g}-cloud self matrix",
        "seconds": seconds, "cloud_pairs": pairs, "pairs_per_s": pairs / seconds,
        "max_gap": max(float(gcross.max()), float(gself.max())),
        "scan_elements_per_pair_est": scan_per_pair, "host_sample_pairs": len(idx),
        "fp32_issue_bound_s": bound_s, "share_of_fp32_issue_bound": bound_s / seconds,
        "card": card,
        "device_vs_auction_restatement_max_abs": dev_vs_host,
        "host_lsa_s_per_pair": lsa_per_pair, "host_lsa_s_for_workload_est": lsa_per_pair * pairs,
        "device_minus_lsa_max": lsa_excess,
        "self_diag_zero": bool((torch.diagonal(self_) == 0).all()),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clouds", type=int, nargs="+", default=[1000, 200])
    ap.add_argument("--points", type=int, default=2048)
    ap.add_argument("--eps", type=float, default=1e-5)
    ap.add_argument("--host-pairs", type=int, default=4)
    ap.add_argument("--lsa-pairs", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_emd needs a CUDA device")
    from meshdiffusion_b200 import _native
    ipe, (n_ins, n_rsq) = instructions_per_element(_native.LIB_PATH)
    for n in args.clouds:
        r = run(n, args.points, args.eps, args.host_pairs, ipe, args.lsa_pairs)
        r["sass_instructions_per_element"] = ipe
        r["sass_loop"] = f"{n_ins} instructions per {n_rsq} cost evaluations"
        line = json.dumps(r)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
