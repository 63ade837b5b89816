"""Shared helpers for the parity tests."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import synth  # noqa: E402


def tiny_config(name="res64", precision="tf32"):
    from configs import res64, res128
    cfg = (res128 if name == "res128" else res64).get_config()
    synth.apply_tiny(cfg, name)
    cfg.model.compute_dtype = precision
    return cfg


def full_config(name="res64", precision="tf32"):
    from configs import res64, res128
    cfg = (res128 if name == "res128" else res64).get_config()
    cfg.model.compute_dtype = precision
    return cfg


def build_model(cfg, device, state_seed):
    """Score network with the deterministic synthetic weights the golden vectors were generated with."""
    from meshdiffusion_b200.diffusion.models import utils as mutils
    cfg.device = torch.device(device)
    model = mutils.create_model(cfg)
    net = model.module
    sd = synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=state_seed)
    net.load_state_dict(sd)
    model.eval()  # inference engine; the training tests switch to .train() explicitly
    return model, sd


def rel_max(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


def rel_l2(a, b):
    return ((a - b).double().pow(2).sum().sqrt() / b.double().pow(2).sum().sqrt()).item()


def load_golden(name):
    return np.load(os.path.join(GOLD, name))


def ddpm_loss(pred, noise, mask):
    """lib/diffusion/losses.py:69-78 (l2, masked)."""
    losses = torch.square(pred - noise) * mask
    losses = losses.reshape(losses.shape[0], -1).mean(dim=-1)
    return torch.mean(losses) / mask.sum() * mask.numel()


def grad_signature(name, g, seed=1234):
    """Same (norm, 4 random projections) signature as oracle/make_golden.py::grad_signature."""
    gen = torch.Generator().manual_seed(seed + sum(ord(c) for c in name))
    r = torch.randn(4, g.numel(), generator=gen, dtype=torch.float64)
    gd = g.detach().double().reshape(-1).cpu()
    return np.concatenate([[gd.norm().item()], (r @ gd).numpy()])


def engine_report(cfg, batch, precision, training, dry=True):
    """What a score-network engine (or with dry=True its GPU-less plan) answers without running: mdb_unet_info, every
    mdb_unet_gemm_ops row and, for a training plan, mdb_unet_train_info and mdb_unet_grad_ready of every parameter."""
    import ctypes
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(cfg), batch, precision, training=training)
    h = ctypes.c_void_p()
    _native.check((L.mdb_unet_create_dry if dry else L.mdb_unet_create)(ctypes.byref(c), ctypes.byref(h)))
    try:
        fl, ar, ng, ns = ctypes.c_double(), ctypes.c_longlong(), ctypes.c_int(), ctypes.c_int()
        _native.check(L.mdb_unet_info(h, ctypes.byref(fl), ctypes.byref(ar), ctypes.byref(ng), ctypes.byref(ns)))
        r = {"flops": fl.value, "arena": ar.value, "n_gemm": ng.value, "n_steps": ns.value, "gemm_ops": []}
        for i in range(ng.value):
            name, f, fb = ctypes.c_char_p(), ctypes.c_double(), ctypes.c_double()
            _native.check(L.mdb_unet_gemm_ops(h, i, ctypes.byref(name), ctypes.byref(f), ctypes.byref(fb)))
            r["gemm_ops"].append((name.value.decode(), f.value, fb.value))
        if training:
            bf, nb, nu = ctypes.c_double(), ctypes.c_int(), ctypes.c_longlong()
            _native.check(L.mdb_unet_train_info(h, ctypes.byref(bf), ctypes.byref(nb), ctypes.byref(nu)))
            r.update(bwd_flops=bf.value, n_bwd_steps=nb.value, numel=nu.value, grad_ready={})
            for i in range(L.mdb_unet_num_params(h)):
                name, step = ctypes.c_char_p(), ctypes.c_int()
                _native.check(L.mdb_unet_param_info(h, i, ctypes.byref(name), None, None, None))
                _native.check(L.mdb_unet_grad_ready(h, name.value, ctypes.byref(step)))
                r["grad_ready"][name.value.decode()] = step.value
        return r
    finally:
        L.mdb_unet_destroy(h)
