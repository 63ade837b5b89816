"""`--mode=distill`: progressive distillation (Salimans & Ho, "Progressive Distillation for Fast Sampling of Diffusion
Models", ICLR 2022) of a trained checkpoint into few-step students for `sampling.method='distilled'`.

Each round trains a student to match two DDIM steps of its teacher with one step of its own, on the halving DDIM grid
(sampling.ddim_grid), so each round halves the number of steps: round r goes from K_T = start_steps / 2^(r-1) teacher
steps to K_S = K_T / 2 student steps, until K_S = final_steps. The teacher of round 1 is the EMA of
`distill.teacher_ckpt`; the teacher of every later round is the EMA of the round before. The student has the teacher's
architecture and starts from its weights, with a fresh FusedAdam (`distill.lr`, default `optim.lr`, no warm-up) and an
EMA that starts at those weights.

A micro-step draws a batch (`data.*` as `--mode=train` reads it), a student step i ~ U{0 .. K_S - 1} per sample and
z_s = perturb(x0, eps) at label s = l_{2i} (mdb_ddpm_perturb), computes the target eps~ on the teacher's inference engine
(mdb_distill_targets: forward, DDIM step s -> m, forward, DDIM step m -> e and the target) and takes the student's
`--mode=train` step on (z_s, s) against eps~: the same DDPMLossFn, clipping, FusedAdam, EMA and micro-batching
(`training.iter_size`), through losses.get_update_fn. Under torchrun every rank makes its own targets, gradients go
through the bucketed all-reduce and rank 0 alone writes.

Outputs under `<training.train_dir>/distill/`:
  steps_<K_S>/checkpoint.pth  the student, in the four-key checkpoint layout every mode and the reference load;
  steps_<K_S>/distill.json    teacher steps and checkpoint, iterations, final loss, seconds, and the match error;
  checkpoint-meta.pth, progress.json  the pre-emption checkpoint of the running round and (round, step), written every
                              `training.snapshot_freq_for_preemption` optimiser steps; a restarted run resumes there.
The match error compares the teacher's K_T-step and the student's K_S-step DDIM maps from one fixed, seeded prior batch
(both through mdb_solver_run): the masked RMS difference and the channel-0 sign agreement on grid-mask voxels, at the
start and the end of every round.
"""
import json
import logging
import os
import time

import numpy as np
import torch

from .. import _native, train_ops
from . import losses, sampling, sde_lib, trainer
from .evaler import load_grid_mask
from .models import utils as mutils
from .models.ema import ExponentialMovingAverage
from .utils import restore_checkpoint, save_checkpoint

MATCH_SEED_OFFSET = 7919  # the match error's prior batch: torch CPU generator seeded seed + this, the same every round


def _int(v):
    return not isinstance(v, bool) and isinstance(v, (int, np.integer))


def settings(config):
    """The distillation settings of `config.distill`, checked: teacher_ckpt, start_steps, final_steps, iters, lr and the
    rounds [(K_T, K_S)]. Raises ValueError for a malformed setting."""
    d = config.get("distill", None)
    if d is None:
        raise ValueError("--mode=distill needs the distill.* settings (at least distill.teacher_ckpt)")
    ckpt = d.get("teacher_ckpt", None)
    if not isinstance(ckpt, str) or ckpt in ("", "PLACEHOLDER"):
        raise ValueError("distill.teacher_ckpt must name the teacher's checkpoint")
    start, final = d.get("start_steps", 512), d.get("final_steps", 8)
    N = int(config.model.num_scales)
    if not _int(final) or final < 2:
        raise ValueError(f"distill.final_steps must be an integer >= 2, got {final!r}")
    if not _int(start) or start > N - 1:
        raise ValueError(f"distill.start_steps must be an integer <= N - 1 = {N - 1}, got {start!r}")
    ratio = start // final
    if start % final or ratio < 2 or ratio & (ratio - 1):
        raise ValueError(f"distill.start_steps must be final_steps * 2^R with R >= 1, got {start} and {final}")
    iters = d.get("iters", None)
    if not _int(iters) or iters < 1:
        raise ValueError(f"distill.iters (optimiser steps per round) must be an integer >= 1, got {iters!r}")
    lr = d.get("lr", None)
    lr = float(config.optim.lr) if lr is None else lr
    if isinstance(lr, bool) or not isinstance(lr, (int, float)) or not np.isfinite(lr) or lr <= 0:
        raise ValueError(f"distill.lr must be a positive number, got {lr!r}")
    rounds, k = [], int(start)
    while k > final:
        rounds.append((k, k // 2))
        k //= 2
    return {"teacher_ckpt": ckpt, "start_steps": int(start), "final_steps": int(final), "iters": int(iters),
            "lr": float(lr), "rounds": rounds}


# ---- the kernels -------------------------------------------------------------------------------------------------
def rows_tensor(sde, K_T, device):
    """sampling.distill_rows as the float32 mdb_distill_row array [K_T / 2, 13] on `device`."""
    return torch.tensor(sampling.distill_rows(sde, K_T).astype(np.float32), device=device)


def _check_operands(z_s, idx, rows, mask_flat, labels, **fp32):
    """The kernels read raw pointers: refuse tensors they would misread (wrong dtype, device, layout or size)."""
    B, V = z_s.shape[0], z_s[0, 0].numel()
    want = {"z_s": (z_s, z_s.shape), "mask": (mask_flat, (V,)), "labels": (labels, (B,)), **fp32}
    for name, (t, shape) in want.items():
        if t is None:
            continue
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
            raise ValueError(f"distill: {name} must be a contiguous float32 CUDA tensor of shape {tuple(shape)}")
    if not idx.is_cuda or idx.dtype != torch.int32 or not idx.is_contiguous() or tuple(idx.shape) != (B,):
        raise ValueError(f"distill: the step indices must be a contiguous int32 CUDA tensor of shape ({B},)")
    if (not rows.is_cuda or rows.dtype != torch.float32 or not rows.is_contiguous() or rows.dim() != 2
            or rows.shape[1] != len(sampling.DISTILL_COLUMNS)):
        raise ValueError(f"distill: rows must be a contiguous float32 CUDA tensor [n, {len(sampling.DISTILL_COLUMNS)}]")


def distill_step(eps, z_s, z_mid, out, mask_flat, idx, rows, phase, labels):
    """One phase of mdb_distill_step on CUDA tensors: phase 0 writes z_mid, phase 1 out; both write labels [B]."""
    L = _native.lib()
    B, C = z_s.shape[0], z_s.shape[1]
    _check_operands(z_s, idx, rows, mask_flat, labels, eps=(eps, z_s.shape), z_mid=(z_mid, z_s.shape),
                    out=(out, z_s.shape))
    _native.check(L.mdb_distill_step(_native.ptr(eps), _native.ptr(z_s), _native.ptr(z_mid), _native.ptr(out),
                                     _native.ptr(mask_flat), _native.ptr(idx), _native.ptr(rows), rows.shape[0], int(phase),
                                     _native.ptr(labels), z_s[0, 0].numel(), C, B, _native.current_stream()))


def distill_step_eager(eps, z_s, z_mid, mask, rows, idx, phase):
    """One phase in torch fp32 ops with mdb_distill_step's operation order (each product and sum rounded on its own), so
    it is the kernel's bit-exact oracle. rows: float32 [n, 13]; idx int [B]; mask broadcasts over z. Returns (z_mid for
    phase 0 / eps~ for phase 1, labels [B])."""
    w = rows[idx.long()]
    col = lambda name: w[:, sampling.DISTILL_COLUMNS.index(name)].view(-1, 1, 1, 1, 1)
    if phase == 0:
        x0 = (z_s - eps * col("sigma_s")) * col("inv_alpha_s")
        return (z_s * col("c_x_s") + x0 * col("c_0_s")) * mask, w[:, 1].clone()
    x0 = (z_mid - eps * col("sigma_m")) * col("inv_alpha_m")
    z_e = (z_mid * col("c_x_m") + x0 * col("c_0_m")) * mask
    return (z_e - z_s * col("r")) * col("inv_d") * mask, w[:, 0].clone()


def distill_targets(net, z_s, idx, rows, mask_flat, labels):
    """eps~ [B, C, R, R, R] of a native ScoreNet teacher (mdb_distill_targets); labels [B] hold the rows' label_s."""
    L = _native.lib()
    B = z_s.shape[0]
    _check_operands(z_s, idx, rows, mask_flat, labels)
    R, C = net.arch["image_size"], net.arch["num_channels"]
    if tuple(z_s.shape[1:]) != (C, R, R, R):
        raise ValueError(f"distill: z_s has shape {tuple(z_s.shape)}, the teacher takes [B, {C}, {R}, {R}, {R}]")
    net._ensure_engine(B, z_s.device)
    net.sync_parameters()
    out, z_mid, eps_buf = torch.empty_like(z_s), torch.empty_like(z_s), torch.empty_like(z_s)
    _native.check(L.mdb_distill_targets(net._handle, _native.ptr(z_s), _native.ptr(idx), _native.ptr(rows), rows.shape[0],
                                        _native.ptr(mask_flat), _native.ptr(out), _native.ptr(labels), _native.ptr(z_mid),
                                        _native.ptr(eps_buf), B, _native.current_stream()))
    return out


# ---- models ------------------------------------------------------------------------------------------------------
def load_teacher(config, path, mask):
    """A ScoreNet holding the EMA weights of the checkpoint at `path`, in eval mode (only its inference engine runs)."""
    if not os.path.exists(path):
        raise FileNotFoundError(f"distill: the teacher checkpoint {path} does not exist")
    blob = torch.load(path, map_location="cpu", weights_only=False)  # the optimiser moments stay on the host
    model = mutils.create_model(config)
    model.load_state_dict(blob["model"], strict=False)  # as restore_checkpoint loads it
    ema = ExponentialMovingAverage(model.parameters(), decay=config.model.ema_rate)
    ema.load_state_dict(blob["ema"])
    ema.copy_to(model.parameters())
    model.module.mask.data[:] = mask
    model.eval()
    return model


def student_state(config, teacher, lr):
    """The training state of a student initialised from the teacher's weights: fresh FusedAdam at `lr`, EMA at those
    weights, step 0."""
    model = mutils.create_model(config)
    model.load_state_dict(teacher.state_dict())
    optimizer = losses.get_optimizer(config, model.parameters())
    for group in optimizer.param_groups:
        group["lr"] = lr
    ema = ExponentialMovingAverage(model.parameters(), decay=config.model.ema_rate)
    return dict(optimizer=optimizer, model=model, ema=ema, step=0)


def make_distill_step(config, state, sde, mask, teacher, rows, lr):
    """`step_fn(state, batch, idx, clear_grad, update_param)` -> {"loss"}: perturb at the rows' label_s, the teacher's
    targets, and the student's `--mode=train` step against them."""
    net = state["model"].module
    update = losses.get_update_fn(trainer.data_parallel_optimize_fn(config, net, lr=lr, warmup=0))
    mask_flat = mask.reshape(-1).float().contiguous()
    mask_sum = float(mask_flat.sum().item())
    sqrt_ac, sqrt_1mac = sde.sqrt_alphas_cumprod.to(mask.device), sde.sqrt_1m_alphas_cumprod.to(mask.device)

    def step_fn(state, batch, idx, clear_grad=True, update_param=True):
        net.reduce_in_backward = bool(update_param)  # gradients are exchanged once per optimiser step
        labels = rows[idx.long(), 0].contiguous()
        t = labels.long()
        z_s = train_ops.ddpm_perturb(batch, torch.randn_like(batch), mask, sqrt_ac[t], sqrt_1mac[t])
        target = distill_targets(teacher.module, z_s, idx, rows, mask_flat, labels)
        model, optimizer = state["model"], state["optimizer"]
        if clear_grad:
            optimizer.zero_grad()
        pred = mutils.get_model_fn(model, train=True)(z_s, labels)
        loss = train_ops.DDPMLossFn.apply(pred, target, mask, mask_sum)
        update(state, loss, update_param)
        return {"loss": loss}

    return step_fn


def match_error(teacher, ema, sde, K_T, x_T, mask):
    """Teacher (K_T DDIM steps) against the student's EMA (K_T / 2 steps) from the same prior x_T, both through
    mdb_solver_run on the teacher's engine: {"rms": masked RMS difference, "sign_agreement": share of grid-mask voxels
    where channel 0 has the same sign}."""
    shape = tuple(x_T.shape)
    g = mask.reshape(shape[2:])
    run = lambda K: sampling.get_distilled_sampler(sde, shape, lambda x: x, K, device=x_T.device, grid_mask=g,
                                                   native_rng=True)(teacher, x0=x_T)[0]
    a = run(K_T)
    ema.store(teacher.parameters())
    ema.copy_to(teacher.parameters())
    try:
        b = run(K_T // 2)
    finally:
        ema.restore(teacher.parameters())
    m = g.bool()
    n = float(m.sum().item()) * shape[0]
    rms = ((a - b).double().square() * g).sum().item() / (n * shape[1])
    sign = (torch.sign(a[:, 0]) == torch.sign(b[:, 0]))[:, m].double().sum().item() / n
    return {"rms": rms ** 0.5, "sign_agreement": sign}


# ---- the mode ----------------------------------------------------------------------------------------------------
def _read_progress(out_dir):
    path = os.path.join(out_dir, "progress.json")
    if not os.path.exists(path):
        return {"round": 0, "step": 0}
    with open(path) as fh:
        return json.load(fh)


def _write_json(path, obj):
    tmp = path + ".tmp"
    with open(tmp, "w") as fh:
        json.dump(obj, fh, indent=1)
    os.replace(tmp, path)


def distill(config):
    """Runs (or resumes) every round; returns the paths of the students' checkpoints."""
    from .classes import refuse_conditional
    refuse_conditional(config, "distill")
    st = settings(config)
    if config.training.sde.lower() != "vpsde":
        raise NotImplementedError(f"SDE {config.training.sde} unknown.")
    device = config.device
    rank, world = trainer._init_distributed(device)
    seed = int(config.get("seed", 42))
    # as build_state seeds `--mode=train`: the perturbation noise and the student's dropout differ per rank and follow
    # config.seed
    torch.manual_seed(seed + rank)
    if config.training.batch_size % world != 0:
        raise ValueError(f"training.batch_size {config.training.batch_size} is not divisible by the {world} ranks")
    local_batch = config.training.batch_size // world
    out_dir = os.path.join(config.training.train_dir, "distill")
    os.makedirs(out_dir, exist_ok=True)
    meta = os.path.join(out_dir, "checkpoint-meta.pth")
    sde = sde_lib.VPSDE(beta_min=config.model.beta_min, beta_max=config.model.beta_max, N=config.model.num_scales,
                        device=device)
    R, C = config.data.image_size, config.data.num_channels
    mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    next_batch = trainer.batch_source(config, mask, local_batch, rank, world)
    gen = torch.Generator(device=device).manual_seed(seed + rank)
    prior_gen = torch.Generator().manual_seed(seed + MATCH_SEED_OFFSET)
    x_match = sde.prior_sampling((local_batch, C, R, R, R), generator=prior_gen).to(device) * mask
    iter_size, freq = config.training.iter_size, config.training.snapshot_freq_for_preemption
    progress = _read_progress(out_dir)
    outputs = []
    for r, (K_T, K_S) in enumerate(st["rounds"]):
        student_dir = os.path.join(out_dir, f"steps_{K_S}")
        if r < progress["round"]:
            outputs.append(os.path.join(student_dir, "checkpoint.pth"))
            continue
        teacher_path = st["teacher_ckpt"] if r == 0 else os.path.join(out_dir, f"steps_{K_T}", "checkpoint.pth")
        teacher = load_teacher(config, teacher_path, mask)
        state = student_state(config, teacher, st["lr"])
        first = 0
        if r == progress["round"] and progress["step"] > 0:
            restore_checkpoint(meta, state, device, strict=True)
            first, start_match = int(progress["step"]), progress["start_match"]
            logging.info("distill: resuming round %d (%d -> %d steps) at step %d", r + 1, K_T, K_S, first)
        else:
            start_match = match_error(teacher, state["ema"], sde, K_T, x_match, mask) if rank == 0 else None
        trainer.sync_replicas(state)
        rows = rows_tensor(sde, K_T, device)
        step_fn = make_distill_step(config, state, sde, mask, teacher, rows, st["lr"])
        if rank == 0:
            logging.info("distill: round %d, %d -> %d steps, start match error %s", r + 1, K_T, K_S, start_match)
        t0, loss = time.perf_counter(), float("nan")
        for it in range(first, st["iters"]):
            total = 0.0
            for inner in range(iter_size):
                batch = next_batch(gen)
                idx = torch.randint(0, K_S, (local_batch,), generator=gen, device=gen.device).to(device, torch.int32)
                out = step_fn(state, batch, idx, clear_grad=(inner == 0), update_param=(inner == iter_size - 1))
                total += out["loss"].item()
            loss = total / iter_size
            done = it + 1
            if rank == 0 and done % config.training.log_freq == 0:
                logging.info("distill: round %d, step %d, distill_loss: %.5e", r + 1, done, loss)
            if rank == 0 and done % freq == 0 and done < st["iters"]:
                save_checkpoint(meta, state)
                _write_json(os.path.join(out_dir, "progress.json"),
                            {"round": r, "step": done, "start_match": start_match})
        seconds = time.perf_counter() - t0
        end_match = match_error(teacher, state["ema"], sde, K_T, x_match, mask) if rank == 0 else None
        ckpt = os.path.join(student_dir, "checkpoint.pth")
        if rank == 0:
            save_checkpoint(ckpt, state)
            _write_json(os.path.join(student_dir, "distill.json"), {
                "teacher_steps": K_T, "student_steps": K_S, "teacher_ckpt": teacher_path, "iters": st["iters"],
                "iters_run": st["iters"] - first, "iter_size": iter_size, "batch_size": config.training.batch_size,
                "lr": st["lr"], "final_loss": loss, "seconds": seconds,
                "match_error": {"start": start_match, "end": end_match}})
            _write_json(os.path.join(out_dir, "progress.json"), {"round": r + 1, "step": 0})
            logging.info("distill: round %d done, final loss %.5e, end match error %s", r + 1, loss, end_match)
        if world > 1:
            import torch.distributed as dist
            dist.barrier()  # the next round's teacher is the checkpoint rank 0 just wrote
        outputs.append(ckpt)
        for m in (teacher, state["model"]):
            if hasattr(m, "module"):
                m.module.release_engine()
        del teacher, state, step_fn
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()
    return outputs
