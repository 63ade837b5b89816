"""Light field distance at the size a user of `--mode=eval_metrics --config.eval.metric_lfd=True` runs, one GPU.

    python tools/bench_lfd.py [--shapes 1000] [--out PATH]

Workload: `--shapes` generated + `--shapes` reference shapes, `trainer.synthetic_grids` at res 64 (a sphere with random
deformations near the surface), different generator seeds for the two sets, meshed by marching tets in chunks of 8 as
eval_metrics does. Every timed phase is warmed up on a smaller call of the same kernels first.

Reported:
* descriptors: views per second of `lfd.lfd_descriptors` over both sets (normalization, camera matrices, `mdb_raster_depth`
  and `mdb_lfd_descriptors`; host clock around a device synchronise), and the descriptor kernel alone on 1024 silhouettes
  (CUDA events over 10 launches); empty views and the share of coefficient bytes at 255;
* matrices: the cross matrix and both self matrices (CUDA events), pairs per second, and the share of an integer issue
  bound: per pair 100 x 100 view distances of 12 VABSDIFF4 each plus 6000 alignment sums of 10 adds and a min, over
  132 SMs x 64 INT32 lanes x the SM clock read during the run (full rate assumed for VABSDIFF4);
* end to end: the eval_metrics pipeline on the same grids (meshing, sampling, Chamfer matrices and metrics, plus
  descriptors, LFD matrices and metrics with the flag) without file I/O, host clock around a device synchronise, with
  and without LFD;
* the card's name, power limit and SM clock, read with nvidia-smi while a timed window runs.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

H100_SMS, INT32_LANES_PER_SM = 132, 64
INT_OPS_PER_PAIR = 100 * 100 * 12 + 6000 * (10 + 1)


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in out.split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}


def _batches(n, seed):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    g = torch.Generator(device="cuda").manual_seed(seed)
    for c0 in range(0, n, 8):
        yield synthetic_grids(min(8, n - c0), 64, "cuda", generator=g)


def _sync_clock():
    torch.cuda.synchronize()
    return time.perf_counter()


def run(n):
    from meshdiffusion_b200.diffusion import gen_metrics
    from meshdiffusion_b200.geometry import lfd
    from meshdiffusion_b200.geometry.pointcloud import grids_to_meshes
    out = {"shapes": n, "views_per_shape": 100, "res": lfd.LFD_RES}
    meshes = {s: [grids_to_meshes(g, 64) for g in _batches(n, s)] for s in (0, 1)}
    lfd.lfd_descriptors(*meshes[0][0])  # warm-up
    t0 = _sync_clock()
    desc, empty = {}, 0
    for s in (0, 1):
        parts = [lfd.lfd_descriptors(*m) for m in meshes[s]]
        desc[s] = torch.cat([d for d, _ in parts])
        empty += int(sum(e.sum() for _, e in parts))
    seconds = _sync_clock() - t0
    views = 2 * n * 100
    coefs = torch.cat([desc[0], desc[1]])[..., :lfd.COEFS]
    out["descriptors"] = {"seconds": seconds, "views_per_s": views / seconds, "empty_views": empty,
                          "saturated_share": float((coefs == 255).sum()) / coefs.numel(),
                          "saturated_zernike": float((coefs[..., :35] == 255).sum()) / coefs[..., :35].numel(),
                          "saturated_fourier": float((coefs[..., 35:] == 255).sum()) / coefs[..., 35:].numel()}
    # the descriptor kernel alone, on the face ids of one rasterizer call
    from meshdiffusion_b200.geometry import singleview
    verts, faces, vo, fo = meshes[0][0]
    c, s = lfd.normalization(verts, vo)
    B = len(vo) - 1
    mvp = torch.from_numpy(lfd.camera_mvps(c, s).reshape(-1, 16)).cuda()
    jm = torch.arange(B, dtype=torch.int32, device="cuda").repeat_interleave(100)
    _, face_id = singleview._raster_packed(verts, faces, torch.from_numpy(vo[:-1].copy()).cuda(), torch.from_numpy(fo).cuda(),
                                           jm, mvp, lfd.LFD_RES)
    face_id = face_id.repeat(2, 1, 1)[:1024].contiguous()
    lfd.silhouette_descriptors(face_id)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        lfd.silhouette_descriptors(face_id)
    e1.record()
    torch.cuda.synchronize()
    k_s = e0.elapsed_time(e1) * 1e-3 / 10
    out["descriptor_kernel"] = {"images": 1024, "seconds": k_s, "images_per_s": 1024 / k_s}

    g, r = desc[0], desc[1]
    lfd.lfd_matrix(g[:16], r[:16])  # warm-up
    torch.cuda.synchronize()
    e0.record()
    lfd.lfd_matrix(g, r)
    lfd.lfd_matrix(g)
    lfd.lfd_matrix(r)
    e1.record()
    time.sleep(0.5)  # read the card while the enqueued window runs
    card = _card()
    torch.cuda.synchronize()
    m_s = e0.elapsed_time(e1) * 1e-3
    pairs = n * n + 2 * (n * (n - 1) // 2)
    bound = pairs * INT_OPS_PER_PAIR / (H100_SMS * INT32_LANES_PER_SM * card["sm_clock_mhz"] * 1e6)
    out["matrices"] = {"pairs": pairs, "seconds": m_s, "pairs_per_s": pairs / m_s, "int_ops_per_pair": INT_OPS_PER_PAIR,
                       "int_issue_bound_s": bound, "share_of_int_bound": bound / m_s}

    def pipeline(light_fields):
        t = _sync_clock()
        gen, _, glf = gen_metrics._clouds(_batches(n, 0), 64, 2048, 42, "cuda", light_fields)
        ref, _, rlf = gen_metrics._clouds(_batches(n, 1), 64, 2048, 42, "cuda", light_fields)
        m = gen_metrics.generation_metrics(gen, ref)
        if light_fields:
            m.update(gen_metrics.lfd_metrics(glf[0], rlf[0]))
        return _sync_clock() - t, m

    pipeline(False)  # warm-up of the Chamfer path at full size
    t_cd, m_cd = pipeline(False)
    t_lfd, m_lfd = pipeline(True)
    assert all(m_lfd[k] == m_cd[k] for k in ("mmd_cd", "cov_cd", "1nna_cd"))
    out["end_to_end"] = {"seconds_without_lfd": t_cd, "seconds_with_lfd": t_lfd,
                         "metrics": {k: m_lfd[k] for k in ("mmd_cd", "cov_cd", "1nna_cd", "mmd_lfd", "cov_lfd", "1nna_lfd")}}
    out["card"] = card
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lfd needs a CUDA GPU")
    res = run(a.shapes)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
