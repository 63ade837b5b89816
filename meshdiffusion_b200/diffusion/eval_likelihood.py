"""`--mode=eval_likelihood`: negative log-likelihood (bits/dim) of held-out shapes under the probability-flow ODE.

Sample-quality metrics (`--mode=eval_metrics`) compare generated shapes with a reference split; they say nothing about
how well the model fits shapes it was not trained on. Test-split bpd is that complementary number, and the natural way
to compare checkpoints of one run. The shapes of `data.meta_path` (filtered by `data.filter_meta_path`) go through the
item transform the trainer feeds the model, without augmentation and masked by the grid mask, and
`diffusion/likelihood.py` integrates them in the masked convention. One process; writes `<eval_dir>/likelihood.json`.
"""
import json
import logging
import os
import time

import numpy as np
import torch

from . import likelihood
from .evaler import _setup, load_grid_mask
from .trainer import _path_or_none
from .utils import restore_checkpoint

TIMING_KEYS = ("seconds",)


def eval_likelihood(config):
    """Writes `<eval_dir>/likelihood.json` and returns its content."""
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise SystemExit("--mode=eval_likelihood runs in one process; start it with python, not torchrun")
    from ..dataset.shapenet_dmtet_dataset import ShapeNetDMTetDataset
    device = config.device
    R = config.data.image_size
    seed = int(config.get("seed", 42))
    ev = config.eval
    hutchinson = str(ev.get("likelihood_hutchinson", "Rademacher"))
    rtol, atol = float(ev.get("likelihood_rtol", 1e-5)), float(ev.get("likelihood_atol", 1e-5))
    eps = float(ev.get("likelihood_eps", 1e-5))
    max_shapes = ev.get("likelihood_max_shapes", None)
    eval_dir = ev.eval_dir
    os.makedirs(eval_dir, exist_ok=True)

    score_model, ema, state, sde = _setup(config)
    state = restore_checkpoint(ev.ckpt_path, state, device=device)
    ema.copy_to(score_model.parameters())
    score_model.eval()
    net = score_model.module
    mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    ds = ShapeNetDMTetDataset(config.data.meta_path, mask.cpu(), deform_scale=config.model.get("deform_scale", 1.0), aug=False,
                              filter_meta_path=_path_or_none(config.data.get("filter_meta_path", None)),
                              normalize_sdf=config.data.get("normalize_sdf", True), extension=config.data.get("extension", "pt"))
    n = len(ds) if max_shapes is None else min(len(ds), int(max_shapes))
    if n == 0:
        raise ValueError(f"the shape list {config.data.meta_path} selects no shapes")
    fn = likelihood.get_likelihood_fn(sde, lambda x: x, hutchinson_type=hutchinson, rtol=rtol, atol=atol, eps=eps,
                                      grid_mask=mask.view(R, R, R))
    bs = int(ev.batch_size)
    bpd, nfe = [], []
    torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    for k, i in enumerate(range(0, n, bs)):
        data = torch.stack([ds[j] for j in range(i, min(i + bs, n))]).to(device) * mask
        gen = torch.Generator(device="cpu").manual_seed(seed * 1000003 + k)
        noise = likelihood.hutchinson_noise(data.cpu(), hutchinson, generator=gen).to(device)
        b, _, f = fn(score_model, data, noise=noise)
        bpd.extend(float(v) for v in b)
        nfe.append(int(f))
        logging.info("eval_likelihood: batch %d (%d shapes): mean bpd %.6f, %d function evaluations", k, data.shape[0],
                     float(np.mean(b.numpy())), f)
    torch.cuda.synchronize(device)
    seconds = time.perf_counter() - t0
    arr = np.asarray(bpd, np.float64)
    out = dict(bpd=bpd, nfe=nfe, bpd_mean=float(arr.mean()),
               bpd_stderr=float(arr.std(ddof=1) / np.sqrt(arr.size)) if arr.size > 1 else float("nan"),
               n_shapes=int(arr.size), dims=int(config.data.num_channels * int(mask.sum().item())),
               convention=likelihood.MASKED_CONVENTION, hutchinson=hutchinson, rtol=rtol, atol=atol, eps=eps, seed=seed,
               compute_dtype=net.precision, seconds=seconds)
    path = os.path.join(eval_dir, "likelihood.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=2)
    logging.info("eval_likelihood: %d shapes, mean bpd %.6f +- %.6f -> %s", arr.size, out["bpd_mean"], out["bpd_stderr"], path)
    return out
