"""Times shape editing (`--mode=edit`: RePaint resampling on the DPM-Solver++(2M) grid) on synthetic weights:
  * the entry kernel alone (mdb_solver_update, in-kernel Philox noise, all four channels replaced): time per launch and
    GB/s over the bytes it must move, against the H100 SXM data-sheet 3.35 TB/s, for a second-order denoise entry
    (x, eps, x0_hist, known read, x and x0_hist written: 24 bytes per element) and a renoise entry (x, known read, x
    written: 12 bytes per element), plus the two masks (8 bytes per voxel);
  * one res64 edit call per operand mode (batch 32, K = 25, jump 5, resample 3 by default): the public sampler call with
    the whole schedule in mdb_solver_run, wall time around a device synchronise, and its network evaluations.
The card's name, power limit and SM clock are read with nvidia-smi in the same run.

    python tools/bench_edit.py [--batch 32] [--steps 25] [--jump 5] [--resample 3] [--precisions bf16x3,bf16] [--out f]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

from bench_dpm_solver import HBM_BYTES_PER_S, _card, _model, _timed  # noqa: E402


def _keep_mask(R, mask, device):
    """The kept region of the benchmark: the grid mask without the voxels of one half of the grid (y < R / 2)."""
    keep = mask.clone()
    keep[:, : R // 2] = 0
    return keep.view(1, R, R, R).contiguous()


def bench_kernel(B, device, R=64, reps=200):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    from meshdiffusion_b200.geometry import dmtet
    sde = sde_lib.VPSDE(0.1, 20.0, 1000, device=device)
    table, _ = sampling.repaint_schedule(sde, 25, 5, 3, stochastic=True)
    entries_c = sampling._entries_c(table)
    mask = dmtet.grid_mask_from_tets(R).to(device)
    mask_flat = mask.reshape(-1).contiguous()
    x0 = torch.randn(B, 4, R, R, R, device=device) * mask
    eps, hist, known = torch.randn_like(x0), torch.randn_like(x0), torch.randn_like(x0)
    kn = sampling._Known(known, _keep_mask(R, mask, device), range(4), B)
    V = R ** 3
    out = {}
    for kind, e, per_elem in (("denoise", 1, 24), ("renoise", int((table[:, 0] == 1).argmax()), 12)):
        assert int(table[e, 0]) == (kind == "renoise") and (kind == "renoise" or table[e, 6] != 0)
        x, h = x0.clone(), hist.clone()

        def launches(n):
            for _ in range(n):
                sampling._update(eps, x, h, mask_flat, entries_c[e], known=kn, seed=1, offset=4 * e)
        launches(3)
        ev, _ = _timed(lambda: launches(reps))
        nbytes = B * 4 * V * per_elem + 2 * V * 4
        us = ev / reps * 1e3
        out[kind] = {"us": us, "bytes": nbytes, "GB_per_s": nbytes / (us * 1e-6) / 1e9,
                     "share_of_3.35TB_per_s": nbytes / (us * 1e-6) / HBM_BYTES_PER_S}
    return {"batch": B, "res": R, **out}


def bench_edit_call(precision, B, K, jump, resample, device):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    from meshdiffusion_b200.geometry import dmtet
    cfg, model = _model(precision, device)
    R = cfg.data.image_size
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device=device)
    mask = dmtet.grid_mask_from_tets(R).to(device)
    known = (torch.randn(B, 4, R, R, R, device=device) * mask).contiguous()
    keep = _keep_mask(R, mask, device)
    fn = sampling.get_repaint_sampler(sde, (B, 4, R, R, R), lambda t: t, n_steps=K, jump=jump, resample=resample,
                                      device=device, grid_mask=mask.view(1, R, R, R), native_rng=True, seed=1)
    res = {}
    fn(model, known, keep, range(4))  # engine set-up and graph capture

    def call():
        res["out"], res["nfe"] = fn(model, known, keep, range(4))
    ev, host = _timed(call)
    kept = keep[0] > 0
    exact = bool(torch.equal(res["out"][:, :, kept], known[:, :, kept]))
    return {"precision": precision, "batch": B, "res": R, "steps": K, "jump": jump, "resample": resample,
            "nfe": res["nfe"], "event_ms": ev, "host_ms": host, "ms_per_nfe": host / res["nfe"], "kept_exact": exact}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--jump", type=int, default=5)
    ap.add_argument("--resample", type=int, default=3)
    ap.add_argument("--precisions", default="bf16x3,bf16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_edit needs a GPU"
    device = torch.device("cuda:0")
    res = {"card_before": _card()}
    with torch.no_grad():
        res["update_kernel"] = bench_kernel(args.batch, device)
        print(json.dumps(res["update_kernel"]), flush=True)
        res["edit_calls"] = []
        for p in args.precisions.split(","):
            r = bench_edit_call(p, args.batch, args.steps, args.jump, args.resample, device)
            print(json.dumps(r), flush=True)
            res["edit_calls"].append(r)
    res["card_after"] = _card()
    print(json.dumps(res, indent=2))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=2)


if __name__ == "__main__":
    main()
