"""The reference arm of bench.py: the UNMODIFIED MeshDiffusion modules from baseline/_ref (lib/diffusion/models/ddpm_res64.py,
sde_lib.py, sampling.py, configs/res64.py) driven through the reference's own public API -- mutils.create_model,
sampling.get_sampling_fn -> pc_sampler -- on the host cores (`--impl reference`) or, as the stock-PyTorch-GPU baseline of
the bench line, on the same GPU. Nothing of this repository's package is imported here.

Run-time patches applied from the outside (SURVEY 8c), none of which touches the reference's arithmetic:
  * `ml_collections` is not installed: a minimal attribute-dict stand-in is put in sys.modules for configs/*.py;
  * on a GPU-less host `torch.Tensor.cuda` is the identity (sde_lib.py:189,192 hard-code .cuda() for the beta tables);
  * `tqdm.trange` inside sampling.py is bounded to the requested number of iterations of the N=1000 schedule (the loop
    body, the schedule and every coefficient are untouched; num_scales=10 would push beta above 1, SURVEY 8c-5);
  * the checkpoint is synthetic: the reference's own initialisers, with its zero-initialised layers (Conv_1, NIN_3, head)
    re-drawn with the reference's default_init(1.0), so activations are O(1) and no denormals distort the CPU timing.
"""
import os
import sys
import time
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "_ref")


class _ConfigDict(dict):
    """Just enough of ml_collections.ConfigDict for configs/default_configs.py: attribute access on nested dicts."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v


def available():
    return os.path.exists(os.path.join(REF, "lib", "diffusion", "sampling.py"))


def load(device):
    """Imports the reference modules and returns (modules, config) for res64 on `device`."""
    if not available():
        raise RuntimeError("baseline/_ref is missing: run `python baseline/install_reference.py` where /root/reference exists")
    if "ml_collections" not in sys.modules:
        mod = types.ModuleType("ml_collections")
        mod.ConfigDict = _ConfigDict
        sys.modules["ml_collections"] = mod
    if torch.device(device).type == "cpu":
        torch.Tensor.cuda = lambda self, *a, **k: self
    # the reference's top-level packages are called `lib` and `configs`: give them a clean import context
    for name in [m for m in sys.modules if m == "configs" or m.startswith("configs.") or m == "lib" or m.startswith("lib.")]:
        del sys.modules[name]
    # ... and keep this repository's own `configs` package (a regular package beats the reference's namespace packages
    # wherever it sits on sys.path) out of the way while the reference's modules are imported
    repo_root = os.path.dirname(HERE)
    saved = list(sys.path)
    sys.path[:] = [REF] + [q for q in saved if os.path.abspath(q or os.getcwd()) != repo_root]
    try:
        from lib.diffusion.models import ddpm_res64, layers, utils as mutils  # noqa: F401
        from lib.diffusion import sde_lib, sampling
        from configs import res64 as cfg64
    finally:
        sys.path[:] = saved
    assert os.path.abspath(cfg64.__file__).startswith(os.path.abspath(REF)), "the reference's configs must come from baseline/_ref"
    config = cfg64.get_config()
    config.device = torch.device(device)
    return dict(mutils=mutils, layers=layers, sde_lib=sde_lib, sampling=sampling), config


def build(device, seed=0):
    ref, config = load(device)
    torch.manual_seed(seed)
    # models/utils.py:88-96 with the reference's own `use_parallel=False` switch: nn.DataParallel would claim every visible GPU
    # (and refuses a CPU-resident module on a GPU box); one device is what both arms measure
    model = ref["mutils"].create_model(config, use_parallel=False).to(config.device)
    net = model
    init = ref["layers"].default_init(1.0)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if name.endswith("Conv_1.weight") or name.endswith("NIN_3.W") or (p.dim() == 5 and p.shape[0] == config.data.num_channels):
                p.copy_(init(tuple(p.shape)).to(p.device))
        mask = torch.load(os.path.join(REF, "data", "grid_mask_64.pt"), map_location=config.device).to(config.device).float()
        net.mask.data[:] = mask.view(1, 1, 64, 64, 64)  # trainer.py:59-63
    model.eval()
    sde = ref["sde_lib"].VPSDE(beta_min=config.model.beta_min, beta_max=config.model.beta_max, N=config.model.num_scales)
    return ref, config, model, sde, mask.view(1, 64, 64, 64)


def run_steps(ref, config, model, sde, mask, batch, n_iters):
    """`n_iters` iterations of the reference's pc_sampler loop (uncond branch) at `batch`; returns wall seconds."""
    sampling = ref["sampling"]
    shape = (batch, config.data.num_channels, config.data.image_size, config.data.image_size, config.data.image_size)
    fn = sampling.get_sampling_fn(config, sde, shape, lambda x: x, 1e-3, grid_mask=mask)
    real = sampling.tqdm.trange
    sampling.tqdm.trange = lambda n, *a, **k: range(min(n, n_iters))
    try:
        if config.device.type == "cuda":
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        out, _ = fn(model)
        if config.device.type == "cuda":
            torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    finally:
        sampling.tqdm.trange = real
    assert torch.isfinite(out).all()
    return dt


def gpu_baseline(batch=8, steps=3, warmup=1, device="cuda:0"):
    """Stock PyTorch on the same GPU: the reference modules as they ship (cuDNN convolutions with TF32 allowed -- torch's
    default), then with TF32 disabled (true fp32, the arithmetic the 1e-3 parity contract is written against) and under
    bf16 autocast. sample-steps/s each."""
    ref, config, model, sde, mask = build(device)
    out = {"batch": batch, "steps": steps, "impl": "unmodified reference modules (baseline/_ref) through get_sampling_fn/pc_sampler, stock torch"}
    modes = [("tf32_default", True, None), ("fp32_strict", False, None), ("bf16_autocast", True, torch.bfloat16)]
    for name, tf32, autocast in modes:
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        try:
            ctx = torch.autocast("cuda", dtype=autocast) if autocast is not None else torch.autocast("cuda", enabled=False)
            with ctx:
                run_steps(ref, config, model, sde, mask, batch, warmup)
                dt = run_steps(ref, config, model, sde, mask, batch, steps)
            out[name] = {"value": batch * steps / dt, "unit": "sample-steps/s", "ms_per_step": dt / steps * 1e3}
        except Exception as ex:  # e.g. out of memory at this batch: report, never fail the bench line
            out[name] = {"error": str(ex)[:160]}
            torch.cuda.empty_cache()
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    return out
