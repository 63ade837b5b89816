"""`--mode=uncond_gen_interp`: shape interpolation (the reference's `uncond_gen_interp`, lib/diffusion/evaler.py:73-130,
which the reference never made reachable).

Each pair of endpoints in latent space is slerped into F = `eval.batch_size` frames with alpha_f = f / (F - 1), and
the frames are decoded by a deterministic sampler, so every frame is a fixed function of its starting latent and the
frames form a path:
  * noise endpoints (default): `eval.interp_pairs` pairs (default 1); pair p draws both endpoints from
    `sde.prior_sampling` with a CPU generator seeded `seed * 1000003 + p`, unmasked as in the reference, so a pair is
    the same on every rank and for any world size;
  * shape endpoints: `eval.interp_shapes = ((i, j), ...)`, index pairs into the shapes `data.meta_path` /
    `data.filter_meta_path` select, loaded as `--mode=eval_likelihood` loads them and masked. Each pair's two grids are
    mapped to their latents by the DPM-Solver++(2M) ODE run backwards (`sampling.get_dpm_solver_inverter`) with the
    sampler's own `sampling.dpm_steps`, so frames 0 and F - 1 reconstruct the inputs up to discretisation error.

The sampler is `sampling.method = 'dpm_solver'` with `dpm_sde = False`, or `'ddim'` (noise endpoints only). Writes
`<eval_dir>/interp/pair_<p:04d>.npy` (float32 [F, 4, R, R, R]) and `index.json` (`index_<rank>.json` per rank under
torchrun, where rank r takes the pairs p = r (mod world size)). `--mode=export` with `eval.eval_dir=<eval_dir>/interp`
meshes and renders the frames.
"""
import ctypes
import json
import logging
import math
import os
import time

import numpy as np
import torch

from .. import _native
from . import sampling
from .evaler import _rank, _setup, load_grid_mask
from .trainer import _path_or_none
from .utils import restore_checkpoint

TIMING_KEYS = ("seconds",)


def slerp_frames(za, zb, alphas):
    """Spherical interpolation through mdb_slerp_frames. za, zb: CUDA tensors of one shape [P, ...] (P endpoint pairs,
    any trailing shape; the whole tensor of each pair enters the angle, no mask); alphas: F numbers. Returns
    (frames [P, F, ...] float32, coef [P, F, 2] float32 = (w_a, w_b) per frame, sums [P, 3] float64 = (a.b, a.a, b.b))."""
    if za.shape != zb.shape or za.dim() < 2:
        raise ValueError(f"slerp_frames: endpoints must have one shape [P, ...], got {tuple(za.shape)} and {tuple(zb.shape)}")
    if not (za.is_cuda and zb.is_cuda):
        raise ValueError("slerp_frames: the endpoints must be CUDA tensors")
    alphas = [float(a) for a in alphas]
    P, F = za.shape[0], len(alphas)
    n = za[0].numel()
    a = za.detach().to(torch.float32).reshape(P, n).contiguous()
    b = zb.detach().to(device=a.device, dtype=torch.float32).reshape(P, n).contiguous()
    L = _native.lib()
    partial = torch.empty(P, L.mdb_slerp_chunks(), 3, device=a.device, dtype=torch.float64)
    sums = torch.empty(P, 3, device=a.device, dtype=torch.float64)
    coef = torch.empty(P, F, 2, device=a.device, dtype=torch.float32)
    out = torch.empty((P, F) + tuple(za.shape[1:]), device=a.device, dtype=torch.float32)
    _native.check(L.mdb_slerp_frames(_native.ptr(a), _native.ptr(b), n, P, (ctypes.c_double * F)(*alphas), F,
                                     _native.ptr(partial), _native.ptr(sums), _native.ptr(coef), _native.ptr(out), _native.current_stream()))
    return out, coef, sums


def _frames(ev):
    F = ev.batch_size
    if isinstance(F, bool) or not isinstance(F, (int, np.integer)) or F < 2:
        raise ValueError(f"uncond_gen_interp: eval.batch_size is the number of frames per pair and must be an integer >= 2, "
                         f"got {F!r}")
    return int(F)


def _method(config, shape_endpoints):
    method = str(config.sampling.method).lower()
    if method == "dpm_solver":
        if config.sampling.get("dpm_sde", False):
            raise ValueError("uncond_gen_interp: sampling.dpm_sde=True draws fresh noise per frame, so the frames would not "
                             "form a path; use the ODE form (dpm_sde=False)")
        K = config.sampling.get("dpm_steps", 25)
        if isinstance(K, bool) or int(K) != K or K < 2:
            raise ValueError(f"sampling.dpm_steps must be an integer >= 2, got {K!r}")
        return method, int(K)
    if method == "distilled":
        raise ValueError("uncond_gen_interp: sampling.method='distilled' is not supported: interpolation and inversion "
                         "run the dpm_solver ODE; use the teacher's checkpoint with sampling.method='dpm_solver'")
    if method == "ddim":
        if shape_endpoints:
            raise ValueError("uncond_gen_interp: shape endpoints need sampling.method='dpm_solver' (the inversion runs "
                             "its ODE backwards)")
        return method, None
    raise ValueError(f"uncond_gen_interp: sampling.method={method!r} draws fresh noise per frame, so the frames would not "
                     "form a path; use 'dpm_solver' (dpm_sde=False) or 'ddim'")


def _shape_pairs(spec):
    if spec is None or spec in ("", "PLACEHOLDER") or (isinstance(spec, (tuple, list)) and len(spec) == 0):
        return None
    try:
        pairs = [tuple(int(v) for v in p) for p in spec]
    except (TypeError, ValueError):
        raise ValueError(f"uncond_gen_interp: eval.interp_shapes must be index pairs ((i, j), ...), got {spec!r}") from None
    if any(len(p) != 2 for p in pairs):
        raise ValueError(f"uncond_gen_interp: eval.interp_shapes must be index pairs ((i, j), ...), got {spec!r}")
    return pairs


def _n_pairs(ev):
    n = ev.get("interp_pairs", 1)
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 1:
        raise ValueError(f"uncond_gen_interp: eval.interp_pairs must be an integer >= 1, got {n!r}")
    return int(n)


def _dataset(config, mask):
    from ..dataset.shapenet_dmtet_dataset import ShapeNetDMTetDataset
    return ShapeNetDMTetDataset(config.data.meta_path, mask.cpu(), deform_scale=config.model.get("deform_scale", 1.0),
                                aug=False, filter_meta_path=_path_or_none(config.data.get("filter_meta_path", None)),
                                normalize_sdf=config.data.get("normalize_sdf", True),
                                extension=config.data.get("extension", "pt"))


def _sync(device):
    if torch.device(device).type == "cuda":
        torch.cuda.synchronize(device)


def _masked_rel_l2(x, ref, mask):
    d = ((x - ref) * mask).double().pow(2).sum().sqrt()
    r = (ref * mask).double().pow(2).sum().sqrt()
    return float(d / r) if float(r) > 0 else float("nan")


def uncond_gen_interp(config):
    """Writes the frames of this rank's pairs and its index; returns the index. Every argument is checked (ValueError)
    before a network is built."""
    from .classes import refuse_conditional
    refuse_conditional(config, "uncond_gen_interp")
    ev = config.eval
    F = _frames(ev)
    shapes = _shape_pairs(ev.get("interp_shapes", None))
    method, K = _method(config, shapes is not None)
    device = config.device
    R, C = config.data.image_size, config.data.num_channels
    seed = int(config.get("seed", 42))
    rank, world = _rank(), int(os.environ.get("WORLD_SIZE", "1"))
    mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    ds = None
    if shapes is not None:
        ds = _dataset(config, mask)
        for i, j in shapes:
            if not (0 <= i < len(ds) and 0 <= j < len(ds)):
                raise ValueError(f"uncond_gen_interp: shape pair ({i}, {j}) is out of range: {config.data.meta_path} "
                                 f"selects {len(ds)} shapes")
        n_pairs = len(shapes)
    else:
        n_pairs = _n_pairs(ev)

    out_dir = os.path.join(ev.eval_dir, "interp")
    os.makedirs(out_dir, exist_ok=True)
    torch.manual_seed(seed)  # the same network on every rank and in every run when no checkpoint is found
    score_model, ema, state, sde = _setup(config)
    shape = (F, C, R, R, R)
    sampling_fn = sampling.get_sampling_fn(config, sde, shape, lambda x: x, 1e-3, grid_mask=mask.view(1, R, R, R))
    state = restore_checkpoint(ev.ckpt_path, state, device=device)
    ema.copy_to(score_model.parameters())
    score_model.eval()
    invert = (sampling.get_dpm_solver_inverter(sde, (2, C, R, R, R), K, grid_mask=mask.view(1, R, R, R), device=device)
              if shapes is not None else None)
    alphas = [f / (F - 1) for f in range(F)]
    n = C * R ** 3
    secs = dict(inversion=0.0, slerp=0.0, sampling=0.0, writing=0.0)
    index = []
    for p in range(rank, n_pairs, world):
        t0 = time.perf_counter()
        entry = {"file": f"pair_{p:04d}.npy", "pair": p}
        if shapes is None:
            gen = torch.Generator(device="cpu").manual_seed(seed * 1000003 + p)
            z = sde.prior_sampling((2, C, R, R, R), generator=gen).to(device)
            entry.update(endpoints="noise", seed=seed * 1000003 + p, nfe_inversion=0)
        else:
            i, j = shapes[p]
            grids = torch.stack([ds[i], ds[j]]).to(device) * mask
            z, nfe_inv = invert(score_model, grids)
            _sync(device)
            entry.update(endpoints="shapes", shapes=[i, j], sources=[ds.fpath_list[i].rstrip(), ds.fpath_list[j].rstrip()],
                         nfe_inversion=int(nfe_inv))
        t1 = time.perf_counter()
        frames, coef, sums = slerp_frames(z[:1], z[1:], alphas)
        ab, aa, bb = (float(v) for v in sums[0].cpu())
        t2 = time.perf_counter()
        samples, nfe = sampling_fn(score_model, x0=frames[0])
        samples = samples.float().cpu().numpy()  # synchronises
        t3 = time.perf_counter()
        np.save(os.path.join(out_dir, entry["file"]), samples)
        t4 = time.perf_counter()
        theta = (math.degrees(math.acos(max(-1.0, min(1.0, ab / math.sqrt(aa * bb))))) if aa > 0 and bb > 0 else None)
        entry.update(alpha=alphas, theta_deg=theta, endpoint_rms=[math.sqrt(aa / n), math.sqrt(bb / n)],
                     coef=coef[0].cpu().tolist(), nfe_sampling=int(nfe))
        if shapes is not None:
            x = torch.from_numpy(samples)
            g = grids.cpu()
            m = mask[0].cpu()
            entry["recon_rel_l2"] = [_masked_rel_l2(x[0], g[0], m), _masked_rel_l2(x[-1], g[1], m)]
        index.append(entry)
        for key, dt in zip(("inversion", "slerp", "sampling", "writing"), (t1 - t0, t2 - t1, t3 - t2, t4 - t3)):
            secs[key] += dt
        logging.info("uncond_gen_interp: rank %d, pair %d -> %s (theta %s deg)", rank, p, entry["file"],
                     "n/a" if theta is None else f"{theta:.3f}")
    out = {"method": method, "dpm_steps": K, "frames": F, "pairs": n_pairs, "resolution": R, "seed": seed,
           "endpoints": "noise" if shapes is None else "shapes", "seconds": secs, "files": index}
    with open(os.path.join(out_dir, "index.json" if world == 1 else f"index_{rank}.json"), "w") as fh:
        json.dump(out, fh, indent=1)
    return out
