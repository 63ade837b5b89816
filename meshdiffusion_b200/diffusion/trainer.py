"""`--mode=train` driver (reference: lib/diffusion/trainer.py:18-130).

Host loop with the reference's structure: model / EMA / Adam, auto-resume from `checkpoints-meta/checkpoint.pth`,
grid mask written into `score_model.module.mask`, micro-batching through `training.iter_size`, logging every
`log_freq`, pre-emption checkpoint every `snapshot_freq_for_preemption`, numbered checkpoints every `snapshot_freq`.

Forward AND backward of the score network run inside the sm_90a engine (bf16 operands, fp32 master weights /
gradients / Adam / EMA); `loss.backward()` reaches it through one autograd node (models/ddpm.py); the loss arithmetic,
clipping, Adam and the EMA run in the library's optimiser-side kernels (train_ops.py). Data parallelism is one process
per GPU (torchrun), replacing the reference's nn.DataParallel (models/utils.py:95): replicas start from identical
weights, every rank steps on batch_size / world grids, and the flat fp32 gradient buffer is averaged over NCCL once per
optimiser step in buckets that start reducing on a side stream as soon as the backward pass has finished with them.
`config.data.synthetic = True` trains on on-device synthetic DMTet grids (sphere SDF on the tet vertices + random
near-surface deformation, SURVEY section 8d-3) instead of the dataset.
"""
import logging
import os

import torch

from . import losses, sde_lib
from .evaler import load_grid_mask
from .models import utils as mutils
from .models.ema import ExponentialMovingAverage
from .utils import restore_checkpoint, save_checkpoint


def synthetic_grids(batch, resolution, device, generator=None):
    """[B,4,R,R,R] in [-1,1]: channel 0 = sign(0.3 - |v|) on tet vertices, channels 1-3 = U(-0.5,0.5) near the surface."""
    from ..geometry.dmtet import grid_coords_of_tet_vertices, load_tet_grid
    verts, _ = load_tet_grid(resolution)
    v = torch.tensor(verts, device=device)
    c = grid_coords_of_tet_vertices(v.cpu()).to(device)
    r = v.norm(dim=1)
    sdf = torch.sign(0.3 - r)
    near = (r - 0.3).abs() < (1.0 / resolution)
    x = torch.zeros(batch, 4, resolution, resolution, resolution, device=device)
    x[:, 0, c[:, 0], c[:, 1], c[:, 2]] = sdf
    d = (torch.rand(batch, 3, v.shape[0], device=device, generator=generator) - 0.5) * near.float()
    x[:, 1:, c[:, 0], c[:, 1], c[:, 2]] = d
    return x


def _path_or_none(p):
    """The stock configs carry the literal "PLACEHOLDER" for unset paths (configs/res64.py): no filter list then."""
    return None if p in (None, "", "PLACEHOLDER") else p


def _init_distributed(device):
    """(rank, world): joins the NCCL group when launched under torchrun, else (0, 1)."""
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        dist.init_process_group("nccl" if torch.device(device).type == "cuda" else "gloo")
    return (dist.get_rank(), dist.get_world_size()) if dist.is_initialized() else (0, 1)


def build_state(config, rank=0, world=1):
    """Model / EMA / optimiser / step counter of trainer.py:36-42. Every rank builds the SAME initial weights (the global
    generator is seeded with config.seed before the model is created and re-seeded with seed + rank afterwards, so labels,
    noise and dropout differ per rank), and rank 0's parameters, buffers and EMA are broadcast on top, so replicas that only
    exchange gradients stay identical."""
    seed = int(config.get("seed", 42))
    torch.manual_seed(seed)
    score_model = mutils.create_model(config)
    ema = ExponentialMovingAverage(score_model.parameters(), decay=config.model.ema_rate)
    optimizer = losses.get_optimizer(config, score_model.parameters())
    torch.manual_seed(seed + rank)
    state = dict(optimizer=optimizer, model=score_model, ema=ema, step=0)
    return state


def sync_replicas(state):
    """Broadcasts rank 0's parameters, buffers and EMA shadow (after create_model / restore_checkpoint)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return
    with torch.no_grad():
        for t in list(state["model"].parameters()) + list(state["model"].buffers()) + list(state["ema"].shadow_params):
            dist.broadcast(t.data, src=0)


def make_train_step(config, state, sde, mask):
    """`train_step_fn(state, batch, clear_grad, update_param)` exactly as train() uses it: losses.get_step_fn around an
    optimize_fn that first completes the data-parallel gradient mean (a wait when the backward pass already overlapped the
    bucketed all-reduce, see ScoreNet.reduce_in_backward) and then runs warm-up + clip + FusedAdam (+ EMA)."""
    net = state["model"].module
    base_optimize_fn = losses.optimization_manager(config)

    def optimize_fn(optimizer, params, step, **kw):
        net.allreduce_grads()  # no-op on one GPU
        return base_optimize_fn(optimizer, params, step=step, **kw)

    step_fn = losses.get_step_fn(sde, train=True, optimize_fn=optimize_fn, mask=mask, loss_type=config.training.loss_type)

    def train_step_fn(state, batch, clear_grad=True, update_param=True):
        net.reduce_in_backward = bool(update_param)  # gradients are exchanged once per optimiser step
        return step_fn(state, batch, clear_grad=clear_grad, update_param=update_param)

    return train_step_fn


def train(config):
    workdir = config.training.train_dir
    os.makedirs(workdir, exist_ok=True)
    device = config.device
    rank, world = _init_distributed(device)
    state = build_state(config, rank, world)
    score_model = state["model"]

    checkpoint_dir = os.path.join(workdir, "checkpoints")
    checkpoint_meta_dir = os.path.join(workdir, "checkpoints-meta", "checkpoint.pth")
    os.makedirs(checkpoint_dir, exist_ok=True)
    os.makedirs(os.path.dirname(checkpoint_meta_dir), exist_ok=True)
    state = restore_checkpoint(checkpoint_meta_dir, state, device)
    initial_step = int(state["step"])

    R = config.data.image_size
    mask = load_grid_mask(R, device).view(1, 1, R, R, R)
    score_model.module.mask.data[:] = mask
    sync_replicas(state)

    if config.training.sde.lower() != "vpsde":
        raise NotImplementedError(f"SDE {config.training.sde} unknown.")
    sde = sde_lib.VPSDE(beta_min=config.model.beta_min, beta_max=config.model.beta_max, N=config.model.num_scales,
                        device=device)
    train_step_fn = make_train_step(config, state, sde, mask)

    # `training.batch_size` is the GLOBAL batch, as it is for the reference's nn.DataParallel (which scatters one batch
    # over the visible GPUs): every rank steps on batch_size / world grids
    if config.training.batch_size % world != 0:
        raise ValueError(f"training.batch_size {config.training.batch_size} is not divisible by the {world} ranks")
    local_batch = config.training.batch_size // world

    synthetic = bool(config.data.get("synthetic", False))
    data_iter = train_loader = sampler = None
    epoch = 0
    if not synthetic:
        # trainer.py:64-75 of the reference: JSON list of per-shape grids, shuffled DataLoader; under torchrun every rank
        # reads its own shard (DistributedSampler) instead of nn.DataParallel scattering one batch
        from ..dataset.shapenet_dmtet_dataset import ShapeNetDMTetDataset
        dataset = ShapeNetDMTetDataset(config.data.meta_path, deform_scale=config.model.get("deform_scale", 1.0), aug=True,
                                       grid_mask=mask.cpu(), filter_meta_path=_path_or_none(config.data.get("filter_meta_path", None)),
                                       normalize_sdf=config.data.get("normalize_sdf", True),
                                       extension=config.data.get("extension", "pt"))
        if world > 1:
            sampler = torch.utils.data.distributed.DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=True,
                                                                      seed=int(config.get("seed", 42)))
        train_loader = torch.utils.data.DataLoader(dataset, batch_size=local_batch, shuffle=sampler is None,
                                                   sampler=sampler, num_workers=config.data.get("num_workers", 0), pin_memory=True)
        data_iter = iter(train_loader)

    def next_batch(gen):
        nonlocal data_iter, epoch
        if synthetic:
            return synthetic_grids(local_batch, R, device, gen) * mask
        try:
            batch = next(data_iter)
        except StopIteration:
            epoch += 1
            if sampler is not None:
                sampler.set_epoch(epoch)  # a new shuffle every epoch
            data_iter = iter(train_loader)
            batch = next(data_iter)
        return batch.to(device, non_blocking=True)

    iter_size = config.training.iter_size
    num_train_steps = config.training.n_iters
    gen = torch.Generator(device=device).manual_seed(int(config.get("seed", 42)) + rank)
    if rank == 0:
        logging.info("Training operand mode: %s (training.compute_dtype).", score_model.module.train_precision)
    logging.info("Starting training loop at step %d.", initial_step // iter_size)
    for step in range(initial_step // iter_size, num_train_steps + 1):
        tmp_loss = 0.0
        for inner in range(iter_size):
            batch = next_batch(gen)
            loss = train_step_fn(state, batch, clear_grad=(inner == 0), update_param=(inner == iter_size - 1))["loss"]
            tmp_loss += loss.item()
        tmp_loss /= iter_size
        if step % config.training.log_freq == 0 and rank == 0:
            logging.info("step: %d, training_loss: %.5e", step, tmp_loss)
        if rank != 0:
            continue  # replicas start identical and apply the same averaged gradients: rank 0 alone writes checkpoints
        if step != 0 and step % config.training.snapshot_freq_for_preemption == 0:
            save_checkpoint(checkpoint_meta_dir, state)
        if step != 0 and step % config.training.snapshot_freq == 0 or step == num_train_steps:
            save_checkpoint(os.path.join(checkpoint_dir, f"checkpoint_{step}.pth"), state)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
