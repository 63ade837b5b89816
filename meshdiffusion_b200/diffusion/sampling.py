"""Predictor-corrector sampling for the VP-SDE score model.

Interface mirror of the reference's lib/diffusion/sampling.py: predictor / corrector registries (:33-80),
`get_sampling_fn` (:83-132), `get_pc_sampler` -> `pc_sampler(model, partial, partial_mask, partial_channel,
freeze_iters)` (:357-487). The configured pair (ancestral_sampling + none, configs/res64.py:22-23) runs on a fused
path: one native U-Net evaluation and ONE fused update kernel per step (score scaling, ancestral mean / noise and
both grid-mask multiplies), with the state resident in HBM and no host synchronisation inside the loop. Other
registered predictors / correctors use the same native network through `get_score_fn` with a few torch
elementwise ops around it. `method='dpm_solver'` (no working reference counterpart) is the few-step DPM-Solver++(2M)
sampler at the end of this file; `get_dpm_solver_inverter` runs its ODE form backwards (a grid's latent, for
`--mode=uncond_gen_interp`). `method='distilled'` is the DDIM ODE on the halving grid of a progressively distilled
student (`--mode=distill`), through the same solver code.
"""
import abc
import contextlib
import ctypes
import functools

import numpy as np
import torch

from .. import _native
from . import sde_lib
from .models import utils as mutils

_PREDICTORS = {}
_CORRECTORS = {}


def register_predictor(cls=None, *, name=None):
    def _add(c):
        key = name if name is not None else c.__name__
        if key in _PREDICTORS:
            raise ValueError(f"Already registered model with name: {key}")
        _PREDICTORS[key] = c
        return c
    return _add if cls is None else _add(cls)


def register_corrector(cls=None, *, name=None):
    def _add(c):
        key = name if name is not None else c.__name__
        if key in _CORRECTORS:
            raise ValueError(f"Already registered model with name: {key}")
        _CORRECTORS[key] = c
        return c
    return _add if cls is None else _add(cls)


def get_predictor(name):
    return _PREDICTORS[name]


def get_corrector(name):
    return _CORRECTORS[name]


def get_sampling_fn(config, sde, shape, inverse_scaler, eps, grid_mask=None, return_traj=False):
    method = config.sampling.method.lower()
    if method == "pc":
        return get_pc_sampler(
            sde=sde, shape=shape,
            predictor=get_predictor(config.sampling.predictor.lower()),
            corrector=get_corrector(config.sampling.corrector.lower()),
            inverse_scaler=inverse_scaler, snr=config.sampling.snr, n_steps=config.sampling.n_steps_each,
            probability_flow=config.sampling.probability_flow, continuous=config.training.continuous,
            denoise=config.sampling.noise_removal, eps=eps, device=config.device, grid_mask=grid_mask,
            return_traj=return_traj,
            max_iters=config.sampling.get("max_iters", None), native_rng=config.sampling.get("native_rng", False),
            seed=config.get("seed", 42), guidance_scale=config.sampling.get("guidance_scale", 1.0))
    if method == "ddim":
        return get_ddim_sampler(sde=sde, shape=shape, predictor=get_predictor("ddim"), inverse_scaler=inverse_scaler,
                                n_steps=config.sampling.n_steps_each, denoise=config.sampling.noise_removal, eps=eps,
                                device=config.device, grid_mask=grid_mask,
                                guidance_scale=config.sampling.get("guidance_scale", 1.0))
    if method == "dpm_solver":
        return get_dpm_solver_sampler(sde=sde, shape=shape, inverse_scaler=inverse_scaler,
                                      n_steps=config.sampling.get("dpm_steps", 25),
                                      stochastic=config.sampling.get("dpm_sde", False),
                                      denoise=config.sampling.noise_removal, device=config.device, grid_mask=grid_mask,
                                      native_rng=config.sampling.get("native_rng", False), seed=config.get("seed", 42),
                                      guidance_scale=config.sampling.get("guidance_scale", 1.0))
    if method == "distilled":
        return get_distilled_sampler(sde=sde, shape=shape, inverse_scaler=inverse_scaler,
                                     n_steps=config.sampling.get("distill_steps", 8), device=config.device,
                                     grid_mask=grid_mask, native_rng=config.sampling.get("native_rng", False),
                                     seed=config.get("seed", 42), guidance_scale=config.sampling.get("guidance_scale", 1.0))
    raise ValueError(f"Sampler name {method} unknown.")


# ------------------------------------------------------------------------------------------------------------------
class Predictor(abc.ABC):
    def __init__(self, sde, score_fn, probability_flow=False):
        self.sde, self.score_fn, self.probability_flow = sde, score_fn, probability_flow

    @abc.abstractmethod
    def update_fn(self, x, t):
        ...


class Corrector(abc.ABC):
    def __init__(self, sde, score_fn, snr, n_steps):
        self.sde, self.score_fn, self.snr, self.n_steps = sde, score_fn, snr, n_steps

    @abc.abstractmethod
    def update_fn(self, x, t):
        ...


def _bcast(v):
    return v[:, None, None, None, None]


def _reverse_sde(sde, score_fn, x, t, probability_flow):
    """Drift / diffusion of the reverse-time SDE (sde_lib.py:100-107)."""
    drift, diffusion = sde.sde(x, t)
    score = score_fn(x, t)
    drift = drift - _bcast(diffusion) ** 2 * score * (0.5 if probability_flow else 1.0)
    return drift, (torch.zeros_like(diffusion) if probability_flow else diffusion)


def _reverse_discretize(sde, score_fn, x, t, probability_flow):
    """sde_lib.py:109-111."""
    f, G = sde.discretize(x, t)
    rev_f = f - _bcast(G) ** 2 * score_fn(x, t) * (0.5 if probability_flow else 1.0)
    return rev_f, (torch.zeros_like(G) if probability_flow else G)


@register_predictor(name="euler_maruyama")
class EulerMaruyamaPredictor(Predictor):
    def update_fn(self, x, t):
        dt = -1.0 / self.sde.N
        z = torch.randn_like(x)
        drift, diffusion = _reverse_sde(self.sde, self.score_fn, x, t, self.probability_flow)
        x_mean = x + drift * dt
        return x_mean + _bcast(diffusion) * np.sqrt(-dt) * z, x_mean


@register_predictor(name="reverse_diffusion")
class ReverseDiffusionPredictor(Predictor):
    def update_fn(self, x, t):
        f, G = _reverse_discretize(self.sde, self.score_fn, x, t, self.probability_flow)
        z = torch.randn_like(x)
        x_mean = x - f
        return x_mean + _bcast(G) * z, x_mean


@register_predictor(name="ancestral_sampling")
class AncestralSamplingPredictor(Predictor):
    def __init__(self, sde, score_fn, probability_flow=False):
        super().__init__(sde, score_fn, probability_flow)
        if not isinstance(sde, sde_lib.VPSDE):
            raise NotImplementedError(f"SDE class {sde.__class__.__name__} not yet supported.")
        assert not probability_flow, "Probability flow not supported by ancestral sampling"

    def update_fn(self, x, t):
        sde = self.sde
        beta = sde.discrete_betas.to(t.device)[(t * (sde.N - 1) / sde.T).long()]
        score = self.score_fn(x, t)
        x_mean = (x + _bcast(beta) * score) / _bcast(torch.sqrt(1.0 - beta))
        return x_mean + _bcast(torch.sqrt(beta)) * torch.randn_like(x), x_mean


@register_predictor(name="none")
class NonePredictor(Predictor):
    def __init__(self, sde, score_fn, probability_flow=False):
        pass

    def update_fn(self, x, t):
        return x, x


@register_corrector(name="langevin")
class LangevinCorrector(Corrector):
    def update_fn(self, x, t):
        sde = self.sde
        alpha = sde.alphas.to(t.device)[(t * (sde.N - 1) / sde.T).long()]
        x_mean = x
        for _ in range(self.n_steps):
            grad = self.score_fn(x, t)
            noise = torch.randn_like(x)
            grad_norm = torch.norm(grad.reshape(grad.shape[0], -1), dim=-1).mean()
            noise_norm = torch.norm(noise.reshape(noise.shape[0], -1), dim=-1).mean()
            step = (self.snr * noise_norm / grad_norm) ** 2 * 2 * alpha
            x_mean = x + _bcast(step) * grad
            x = x_mean + _bcast(torch.sqrt(step * 2)) * noise
        return x, x_mean


@register_corrector(name="ald")
class AnnealedLangevinDynamics(Corrector):
    def update_fn(self, x, t):
        sde = self.sde
        alpha = sde.alphas.to(t.device)[(t * (sde.N - 1) / sde.T).long()]
        std = sde.marginal_prob(x, t)[1]
        x_mean = x
        for _ in range(self.n_steps):
            grad = self.score_fn(x, t)
            noise = torch.randn_like(x)
            step = (self.snr * std) ** 2 * 2 * alpha
            x_mean = x + _bcast(step) * grad
            x = x_mean + noise * _bcast(torch.sqrt(step * 2))
        return x, x_mean


@register_corrector(name="none")
class NoneCorrector(Corrector):
    def __init__(self, sde, score_fn, snr, n_steps):
        pass

    def update_fn(self, x, t):
        return x, x


# ------------------------------------------------------------------------------------------------------------------
def _native_net(model):
    from .models.ddpm import ScoreNet
    inner = getattr(model, "module", model)
    return inner if isinstance(inner, ScoreNet) else None


class _Cond:
    """Replacement conditioning of the partial branch (sampling.py:453-467 of the reference) in the form the update kernel
    takes it: channel `c` of `partial` / `partial_mask` (batch 1 = one grid shared by all samples, or one per sample) and
    the per-step marginal_prob scalars, computed with the reference's torch ops so they are bit-identical."""

    def __init__(self, sde, partial, partial_mask, c, timesteps, B):
        V = partial[0, 0].numel()
        self.c = int(c)
        self.partial = partial[:, c].to(torch.float32).contiguous()
        self.pmask = partial_mask[:, c].to(torch.float32).contiguous()
        for t in (self.partial, self.pmask):
            if t.shape[0] not in (1, B):
                raise ValueError("partial / partial_mask must have batch 1 or the sampling batch")
        self.pb = V if self.partial.shape[0] == B and B > 1 else 0
        self.mb = V if self.pmask.shape[0] == B and B > 1 else 0
        lmc = -0.25 * timesteps ** 2 * (sde.beta_1 - sde.beta_0) - 0.5 * timesteps * sde.beta_0  # sde_lib.py:211
        self.coefs = torch.exp(lmc).cpu().tolist()
        self.stds = torch.sqrt(1.0 - torch.exp(2.0 * lmc)).cpu().tolist()

    def struct(self, i=None, noise=None):
        s = _native.SamplerCondC()
        s.partial, s.partial_bstride = self.partial.data_ptr(), self.pb
        s.partial_mask, s.mask_bstride = self.pmask.data_ptr(), self.mb
        s.channel = self.c
        if i is not None:
            s.mean_coef, s.std = self.coefs[i], self.stds[i]
        s.noise = noise.data_ptr() if noise is not None else None
        return s


def _fused_update(eps, x, noise, mask_flat, beta, std, cond=None):
    """x, x_mean <- ancestral update (+ replacement conditioning when `cond` is given), in place on x; one kernel."""
    L = _native.lib()
    x_mean = torch.empty_like(x)
    B, C = x.shape[0], x.shape[1]
    V = x[0, 0].numel()
    _native.check(L.mdb_sampler_update(_native.ptr(eps), _native.ptr(x), _native.ptr(x_mean), _native.ptr(noise),
                                       _native.ptr(mask_flat), beta, std, V, C, B, 0, 0,
                                       ctypes.byref(cond) if cond is not None else None, _native.current_stream()))
    return x, x_mean


def _rank():
    import os
    return int(os.environ.get("RANK", "0"))


def get_pc_sampler(sde, shape, predictor, corrector, inverse_scaler, snr, n_steps=1, probability_flow=False,
                   continuous=False, denoise=True, eps=1e-3, device="cuda", grid_mask=None, return_traj=False,
                   max_iters=None, native_rng=False, seed=42, guidance_scale=1.0):
    """Returns `pc_sampler(model, partial=None, partial_mask=None, partial_channel=0, freeze_iters=None)`.

    `max_iters` truncates the loop to its first iterations of the N-step schedule (used by the plumbing config;
    setting num_scales=10 instead would push beta above 1). `native_rng` draws the per-step noise inside the update
    kernel (Philox keyed by seed + rank, element index and step) and runs the whole loop inside the library -- the
    unconditional branch and the partial (`cond_gen`) branch alike.
    """
    fused = predictor is AncestralSamplingPredictor and corrector is NoneCorrector and not probability_flow

    def generic_step(model, x, vec_t):
        score_fn = mutils.get_score_fn(sde, model, train=False, continuous=continuous)
        c = NoneCorrector(sde, score_fn, snr, n_steps) if corrector is None else corrector(sde, score_fn, snr, n_steps)
        x, x_mean = c.update_fn(x, vec_t)
        x, x_mean = x * grid_mask, x_mean * grid_mask
        p = NonePredictor(sde, score_fn, probability_flow) if predictor is None else predictor(sde, score_fn, probability_flow)
        x, x_mean = p.update_fn(x, vec_t)
        return x * grid_mask, x_mean * grid_mask

    def compute_xzero(model, x, t, mask):
        step = (t * (sde.N - 1) / sde.T).long()
        a1, a2 = sde.sqrt_alphas_cumprod[step], sde.sqrt_1m_alphas_cumprod[step]
        eps_pred = model(x, t * torch.ones(shape[0], device=x.device))
        return ((x - a2 * eps_pred) / a1).clamp(-1, 1) * mask

    def pc_sampler(model, partial=None, partial_mask=None, partial_channel=0, freeze_iters=None, class_labels=None,
                   guidance_scale=guidance_scale):
        with _conditioned(model, class_labels, guidance_scale, "pc") as model, torch.no_grad():
            if freeze_iters is None:
                freeze_iters = sde.N + 10
            c = partial_channel
            timesteps = torch.linspace(sde.T, eps, sde.N, device=device)
            x = sde.prior_sampling(shape).to(device)
            assert x.dim() == 5
            x = x * grid_mask
            B = shape[0]
            net = _native_net(model)
            binary_mask = bool(((grid_mask == 0) | (grid_mask == 1)).all())
            use_fused = fused and net is not None and binary_mask and x.is_cuda
            if use_fused:
                # per-step scalars, gathered once (no host sync inside the loop)
                idx = (timesteps * (sde.N - 1) / sde.T).long()
                betas = sde.discrete_betas.to(device)[idx].cpu().tolist()
                stds = sde.sqrt_1m_alphas_cumprod.to(device)[(timesteps * (sde.N - 1)).long()].cpu().tolist()
                labels_all = (timesteps * (sde.N - 1)).cpu().tolist()
                mask_flat = grid_mask.to(device=device, dtype=torch.float32).reshape(-1).contiguous()
                assert mask_flat.numel() == x[0, 0].numel()
                x = x.contiguous()
            traj = []
            if use_fused:
                net._ensure_engine(B, x.device)
            # nobody edits the weights inside the loop: skip per-step change detection
            with net.frozen() if use_fused else contextlib.nullcontext():
                return _run(model, net, x, use_fused, partial, partial_mask, c, freeze_iters, timesteps, B, traj,
                            betas if use_fused else None, stds if use_fused else None,
                            labels_all if use_fused else None, mask_flat if use_fused else None)

    def _run(model, net, x, use_fused, partial, partial_mask, c, freeze_iters, timesteps, B, traj, betas, stds,
             labels_all, mask_flat):
        def step(x, i, cond=None):
            vec_t = torch.ones(B, device=device) * timesteps[i]
            if not use_fused:
                return generic_step(model, x, vec_t)
            eps_out = model(x, vec_t * (sde.N - 1))
            z = torch.randn_like(x)
            z2 = torch.randn_like(x[:, c]).contiguous() if cond is not None else None  # same draw order as the reference
            return _fused_update(eps_out, x, z, mask_flat, betas[i], stds[i], cond.struct(i, z2) if cond is not None else None)

        if partial is not None:
            assert partial.dim() == 5
            vec_t = torch.ones(B, device=device) * timesteps[0]
            x[:, c] = partial[:, c] * grid_mask[:, c]
            pmean, pstd = sde.marginal_prob(x, vec_t)
            # NB: (B,1,1,1,1) * (B,D,H,W) broadcasts to (B,B,D,H,W) in the reference (sampling.py:436-440)
            sampled = pmean[:, c] + pstd[:, None, None, None, None] * torch.randn_like(pmean[:, c])
            x[:, c] = (x[:, c] * (1 - partial_mask[:, c]) + sampled[:, c] * partial_mask[:, c]) * grid_mask[:, c]
            x_mean = x
            total = sde.N if max_iters is None else min(max_iters, sde.N)
            cond_until = min(freeze_iters, sde.N - 1)
            if use_fused:
                # the replacement + re-noising runs inside the update kernel (one launch per step); with native_rng the
                # whole loop runs inside the library
                cond = _Cond(sde, partial, partial_mask, c, timesteps, B)
                x = x.contiguous()
                if native_rng and not return_traj:
                    x_mean = _native_loop(net, x, mask_flat, labels_all, betas, stds, total, seed + _rank(), 0, cond, cond_until)
                else:
                    for i in range(total):
                        x, x_mean = step(x, i, cond if i < cond_until else None)
                total = 0
            for i in range(total):
                x, x_mean = step(x, i)
                if i != sde.N - 1 and i < freeze_iters:
                    keep, pm = 1 - partial_mask[:, c], partial_mask[:, c]
                    x[:, c] = (x[:, c] * keep + partial[:, c] * pm) * grid_mask[:, c]
                    x_mean[:, c] = (x_mean[:, c] * keep + partial[:, c] * pm) * grid_mask[:, c]
                    vec_t = torch.ones(B, device=device) * timesteps[i]
                    pmean, pstd = sde.marginal_prob(x, vec_t)
                    sampled = pmean[:, c] + pstd[:, None, None, None] * torch.randn_like(pmean[:, c])
                    x[:, c] = (x[:, c] * keep + sampled * pm) * grid_mask[:, c]
                    x_mean[:, c] = x[:, c]
        else:
            total = sde.N - 1 if max_iters is None else min(max_iters, sde.N - 1)
            if use_fused and native_rng and not return_traj:
                x_mean = _native_loop(net, x, mask_flat, labels_all, betas, stds, total, seed + _rank())
            else:
                x_mean = x
                for i in range(total):
                    x, x_mean = step(x, i)
                    if return_traj and i >= 700 and i % 10 == 0:
                        traj.append(compute_xzero(model, x, timesteps[i], grid_mask))
        if return_traj:
            return traj, sde.N * (n_steps + 1)
        return inverse_scaler(x_mean if denoise else x), sde.N * (n_steps + 1)

    return pc_sampler


@contextlib.contextmanager
def _conditioned(model, class_labels, guidance_scale, name):
    """The pc and ddim samplers condition on class_labels without guidance: yields the model to call."""
    if float(guidance_scale) != 1.0:
        raise ValueError(f"the {name} sampler supports class conditioning without guidance only (guidance_scale = 1, "
                         f"got {guidance_scale}); use sampling.method='dpm_solver' or 'distilled' for guidance")
    if class_labels is None:
        yield model
        return
    net = _native_net(model)
    if net is None:
        yield functools.partial(model, class_labels=class_labels)
        return
    with net.conditioned(class_labels):
        yield model


def _native_loop(net, x, mask_flat, labels, betas, stds, total, seed, step0=0, cond=None, cond_until=0):
    """Steps step0 .. step0+total-1 of the loop inside the library (mdb_sampler_run): no Python between steps. The
    schedule lists are indexed by the GLOBAL step; `cond` (a _Cond) switches on the partial branch's replacement
    conditioning for the steps below `cond_until`."""
    L = _native.lib()
    B = x.shape[0]
    net._ensure_engine(B, x.device)
    net.sync_parameters()
    net._set_classes(net._handle, net._class_ids(net._bound_classes, B, x.device), B)
    x_mean = torch.empty_like(x)
    eps_buf = torch.empty_like(x)
    labels_buf = torch.empty(B, device=x.device, dtype=torch.float32)
    arr = lambda v: (ctypes.c_float * total)(*v[step0:step0 + total])
    cs = cond.struct() if cond is not None else None
    _native.check(L.mdb_sampler_run(net._handle, _native.ptr(x), _native.ptr(x_mean), _native.ptr(mask_flat), arr(labels),
                                    arr(betas), arr(stds), total, B, int(seed), _native.ptr(eps_buf),
                                    _native.ptr(labels_buf), int(step0), ctypes.byref(cs) if cs is not None else None,
                                    arr(cond.coefs) if cond is not None else None, arr(cond.stds) if cond is not None else None,
                                    int(cond_until), _native.current_stream()))
    return x_mean


# ------------------------------------------------------------------------------------------------------------------
# DDIM (deterministic) sampling. The reference registers a 'ddim' predictor (sampling.py:249-257) on top of
# RSDE.discretize_ddim (sde_lib.py:113-140) and ships get_ddim_sampler (sampling.py:500-570), whose last line raises a
# NameError (`encode` is undefined). The update below is the same fp64 arithmetic; the sampler is the working version.
@register_predictor(name="ddim")
class DDIMPredictor(Predictor):
    def update_fn(self, x, t, tprev=None):
        sde = self.sde
        step = (t * (sde.N - 1) / sde.T).long()
        step_prev = (tprev * (sde.N - 1) / sde.T).long()
        eps = self.score_fn(x.float(), t.float())  # std_scale=False: the raw noise prediction
        a1 = _bcast(sde.sqrt_alphas_cumprod.to(x.device)[step])
        a2 = _bcast(sde.sqrt_1m_alphas_cumprod.to(x.device)[step])
        a1p = _bcast(sde.sqrt_alphas_cumprod.to(x.device)[step_prev])
        a2p = _bcast(sde.sqrt_1m_alphas_cumprod.to(x.device)[step_prev])
        r1 = a1p.double() / a1.double()
        r2 = a2p.double() / a2.double()
        x0_scaled = x.double() - a2.double() * eps.double()
        noise_part = x - x0_scaled
        x0_pred = x0_scaled / a1
        x_new = r1 * x + (-r1 + r2) * noise_part.double()
        return x_new, x0_pred


def get_ddim_sampler(sde, shape, predictor, inverse_scaler, n_steps=1, denoise=False, eps=1e-3, device="cuda",
                     grid_mask=None, guidance_scale=1.0):
    def ddim_sampler(model, schedule="quad", num_steps=100, x0=None, partial=None, partial_mask=None, partial_channel=0,
                     class_labels=None, guidance_scale=guidance_scale):
        with _conditioned(model, class_labels, guidance_scale, "ddim") as model, torch.no_grad():
            x = (x0 if x0 is not None else sde.prior_sampling(shape).to(device)) * grid_mask
            c = partial_channel
            if partial is not None:
                x[:, c] = x[:, c] * (1 - partial_mask) + partial * partial_mask
            if schedule == "uniform":
                seq = list(range(0, sde.N, sde.N // num_steps))
            elif schedule == "quad":
                seq = [int(s) for s in np.linspace(0, np.sqrt(sde.N * 0.8), 100) ** 2]
            else:
                raise ValueError(f"unknown DDIM schedule {schedule}")
            timesteps = torch.tensor(seq) / sde.N
            score_fn = mutils.get_score_fn(sde, model, train=False, continuous=False, std_scale=False)
            pred = (predictor or DDIMPredictor)(sde, score_fn, False)
            x0_pred = x
            for i in reversed(range(1, len(timesteps))):
                vec_t = torch.ones(shape[0], device=device) * timesteps[i].to(device)
                vec_tprev = torch.ones(shape[0], device=device) * timesteps[i - 1].to(device)
                x, x0_pred = pred.update_fn(x, vec_t, vec_tprev)
                x, x0_pred = (x * grid_mask).float(), (x0_pred * grid_mask).float()
                if partial is not None:
                    x[:, c] = x[:, c] * (1 - partial_mask) + partial * partial_mask
                    x0_pred[:, c] = x0_pred[:, c] * (1 - partial_mask) + partial * partial_mask
            return inverse_scaler(x0_pred * grid_mask if denoise else x * grid_mask), sde.N * (n_steps + 1)

    return ddim_sampler


# ------------------------------------------------------------------------------------------------------------------
# DPM-Solver++(2M) (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion Probabilistic Models"),
# in its ODE form and in the SDE form of k-diffusion's sample_dpmpp_2m_sde: a second-order multistep exponential
# integrator in log-SNR time on the same noise prediction as the samplers above, one network evaluation per step, so a
# sample costs ~25 evaluations instead of 999.
def _vp_arrays(sde):
    """float64 alpha_n = sqrt(alphas_cumprod[n]), sigma_n = sqrt(1 - alphas_cumprod[n]) and lambda_n = log(alpha_n / sigma_n)."""
    abar = sde.alphas_cumprod.detach().to("cpu", torch.float64).numpy()
    alpha, sigma = np.sqrt(abar), np.sqrt(1.0 - abar)
    return alpha, sigma, np.log(alpha) - np.log(sigma)


def dpm_solver_schedule(sde, n_steps, stochastic=False, denoise=True):
    """Label grid and step table of DPM-Solver++(2M) with `n_steps` (K) log-SNR intervals.

    With alpha_n = sqrt(alphas_cumprod[n]), sigma_n = sqrt(1 - alphas_cumprod[n]) and lambda_n = log alpha_n - log sigma_n
    (float64), the labels are the ones whose lambda is nearest each of K + 1 equally spaced targets from lambda_{N-1} to
    lambda_0, repeats dropped: labels[0] = N - 1, labels[-1] = 0, K_eff = len(labels) - 1 network evaluations (K_eff < K
    only when two targets share a label, near label 0). Row k of the table (float64, the fields of mdb_solver_entry after
    `kind`: label, sigma, inv_alpha, c_x, c_0, c_1, c_z, known_coef, known_std) moves x from labels[k] to labels[k + 1]:
    x' = c_x x + c_0 x0_k + c_1 x0_{k-1} + c_z z with x0_k = (x - sigma eps) inv_alpha. Step 0 is first order (c_1 = 0);
    with `denoise` the last SDE step adds no noise. Returns (labels, table)."""
    if isinstance(n_steps, bool) or int(n_steps) != n_steps or n_steps < 2:
        raise ValueError(f"sampling.dpm_steps must be an integer >= 2, got {n_steps!r}")
    K = int(n_steps)
    alpha, sigma, lam = _vp_arrays(sde)
    N = alpha.shape[0]
    targets = lam[N - 1] + np.arange(K + 1) * ((lam[0] - lam[N - 1]) / K)
    labels = []
    for t in targets:
        n = int(np.argmin(np.abs(lam - t)))
        if not labels or n != labels[-1]:
            labels.append(n)
    assert labels[0] == N - 1 and labels[-1] == 0 and all(a > b for a, b in zip(labels, labels[1:]))
    return labels, _solver_table(alpha, sigma, lam, labels, stochastic, denoise)


def _solver_table(alpha, sigma, lam, labels, stochastic=False, denoise=True):
    """float64 step table of DPM-Solver++(2M) along `labels` (any direction): row k moves x from labels[k] to
    labels[k + 1] with h = lambda_t - lambda_s; row 0 is first order."""
    K_eff = len(labels) - 1
    table = np.zeros((K_eff, 9), dtype=np.float64)
    h_prev = None
    for k in range(K_eff):
        s, t = labels[k], labels[k + 1]
        h = lam[t] - lam[s]
        if stochastic:
            c_x = sigma[t] / sigma[s] * np.exp(-h)
            b = -alpha[t] * np.expm1(-2.0 * h)
            c_z = 0.0 if (denoise and k == K_eff - 1) else sigma[t] * np.sqrt(-np.expm1(-2.0 * h))
        else:
            c_x, b, c_z = sigma[t] / sigma[s], -alpha[t] * np.expm1(-h), 0.0
        if h_prev is None:
            c_0, c_1 = b, 0.0
        else:
            r = h_prev / h
            c_0, c_1 = b * (1.0 + 1.0 / (2.0 * r)), -b / (2.0 * r)
        table[k] = (s, sigma[s], 1.0 / alpha[s], c_x, c_0, c_1, c_z, alpha[t], sigma[t])
        h_prev = h
    return table


def dpm_solver_inversion_schedule(sde, n_steps):
    """Labels and step table of the inverse map: the ODE form of DPM-Solver++(2M) run backwards over the labels of
    `dpm_solver_schedule(sde, n_steps)`, from label 0 to N - 1. The rows use the same float64 formula with h < 0; row 0
    is first order and c_z = 0 (the cond fields are not used). K_eff network evaluations map a grid at label 0 (what the
    sampler returns) to the latent at label N - 1 that the sampler with the same K maps back to it, up to the
    discretisation error of both directions. Returns (labels, table)."""
    labels, _ = dpm_solver_schedule(sde, n_steps)
    labels = labels[::-1]
    alpha, sigma, lam = _vp_arrays(sde)
    return labels, _solver_table(alpha, sigma, lam, labels)


# ------------------------------------------------------------------------------------------------------------------
# Progressive distillation (Salimans & Ho, "Progressive Distillation for Fast Sampling of Diffusion Models", ICLR 2022) on
# the halving DDIM grid: a student with K steps learns two DDIM steps of its 2K-step teacher per step of its own.
DISTILL_COLUMNS = ("label_s", "label_m", "label_e", "sigma_s", "inv_alpha_s", "c_x_s", "c_0_s",
                   "sigma_m", "inv_alpha_m", "c_x_m", "c_0_m", "r", "inv_d")


def ddim_grid(sde, K):
    """The K-step DDIM label grid l_i = round((N - 1)(1 - i / K)), i = 0 .. K, rounded half up in integer arithmetic:
    l_0 = N - 1, l_K = 0, and the grid halves exactly (l^(K)_i = l^(2K)_{2i}). K must lie in [2, N - 1]; a finer grid
    would repeat labels."""
    N = sde.N
    if isinstance(K, bool) or not isinstance(K, (int, np.integer)) or not 2 <= K <= N - 1:
        raise ValueError(f"the DDIM grid needs an integer number of steps in [2, N - 1 = {N - 1}], got {K!r}")
    K = int(K)
    return [((N - 1) * (K - i) * 2 + K) // (2 * K) for i in range(K + 1)]


def ddim_table(sde, labels):
    """float64 first-order ODE rows (dpm_solver_schedule's columns) along `labels`: row k is _solver_table's first-order
    step labels[k] -> labels[k + 1], i.e. DDIM (c_1 = 0, c_z = 0, known_coef / known_std = alpha, sigma of labels[k + 1])."""
    if len(labels) < 2:
        raise ValueError("ddim_table needs at least two labels")
    alpha, sigma, lam = _vp_arrays(sde)
    return np.stack([_solver_table(alpha, sigma, lam, labels[k:k + 2])[0] for k in range(len(labels) - 1)])


def distill_rows(sde, K_T):
    """float64 rows [K_T / 2, 13] (DISTILL_COLUMNS, mdb_distill_row field order) of a round whose teacher takes K_T steps
    on ddim_grid(sde, K_T). Row i: labels s = l_{2i}, m = l_{2i+1}, e = l_{2i+2}; the (sigma, inv_alpha, c_x, c_0) of the
    teacher's DDIM steps s -> m and m -> e (ddim_table's rows 2i and 2i + 1); r = alpha_e / alpha_s and
    inv_d = 1 / (sigma_e - alpha_e sigma_s / alpha_s), so that eps~ = (z_e - r z_s) inv_d is the noise prediction whose
    single DDIM step from z_s lands on z_e."""
    if isinstance(K_T, bool) or not isinstance(K_T, (int, np.integer)) or K_T % 2:
        raise ValueError(f"a distillation round needs an even number of teacher steps, got {K_T!r}")
    labels = ddim_grid(sde, K_T)
    table = ddim_table(sde, labels)
    alpha, sigma, _ = _vp_arrays(sde)
    rows = np.zeros((K_T // 2, len(DISTILL_COLUMNS)), dtype=np.float64)
    for i in range(K_T // 2):
        s, m, e = labels[2 * i:2 * i + 3]
        a, b = table[2 * i], table[2 * i + 1]
        rows[i] = (s, m, e, *a[1:5], *b[1:5], alpha[e] / alpha[s], 1.0 / (sigma[e] - alpha[e] * sigma[s] / alpha[s]))
    return rows


# ------------------------------------------------------------------------------------------------------------------
# RePaint resampling (Lugmayr et al., "RePaint: Inpainting using Denoising Diffusion Probabilistic Models", CVPR 2022) on
# the DPM-Solver++(2M) label grid, for shape editing: the kept region is replaced on every step, and every block of
# `jump` solver steps is redone `resample` times, jumping back to the block's first label by forward diffusion in
# between, so the network sees the kept and the regenerated region together at every noise level of the block.
REPAINT_COLUMNS = ("kind", "label", "sigma", "inv_alpha", "c_x", "c_0", "c_1", "c_z", "known_coef", "known_std")


def repaint_schedule(sde, n_steps, jump, resample, stochastic=False, denoise=True):
    """Entry table of RePaint resampling over the labels of `dpm_solver_schedule(sde, n_steps, stochastic, denoise)`.

    The K_eff solver steps are cut into blocks of `jump` steps. Every block but the last runs `resample` times, with a
    renoise entry from the block's last label lo back to its first label hi between two runs; the last block runs once.
    Rows (float64, mdb_solver_entry field order, REPAINT_COLUMNS):
      denoise (kind 0): the solver step's row (label, sigma, inv_alpha, c_x, c_0, c_1, c_z, alpha, sigma of the label it
        lands on); the first step of a repeated run is first order (c_1 = 0), since the x0 history belongs to the
        abandoned run;
      renoise (kind 1): (1, hi, 0, 0, a, 0, 0, s, alpha_hi, sigma_hi) with a = alpha_hi / alpha_lo, s = sqrt(1 - a^2).
    The last row's replacement pair is (1, 0), so the kept region of the output equals the known grid. With resample = 1
    the rows are dpm_solver_schedule's. Returns (table, number of network evaluations = denoise rows)."""
    for name, v in (("jump", jump), ("resample", resample)):
        if isinstance(v, bool) or int(v) != v or v < 1:
            raise ValueError(f"repaint: {name} must be an integer >= 1, got {v!r}")
    jump, resample = int(jump), int(resample)
    labels, table = dpm_solver_schedule(sde, n_steps, stochastic, denoise)
    alpha, sigma, lam = _vp_arrays(sde)
    K = len(labels) - 1
    rows = []
    for b0 in range(0, K, jump):
        b1 = min(b0 + jump, K)
        runs = 1 if b1 == K else resample
        for r in range(runs):
            for k in range(b0, b1):
                row = table[k]
                if r > 0 and k == b0:  # first order; never the last step, so the sub-table's noise term is the table's
                    row = _solver_table(alpha, sigma, lam, labels[b0:b0 + 2], stochastic, denoise=False)[0]
                rows.append(np.concatenate([[0.0], row]))
            if r < runs - 1:
                lo, hi = labels[b1], labels[b0]
                a = alpha[hi] / alpha[lo]
                rows.append(np.array([1.0, hi, 0.0, 0.0, a, 0.0, 0.0, np.sqrt(1.0 - a * a), alpha[hi], sigma[hi]]))
    out = np.stack(rows)
    out[-1, 8:10] = (1.0, 0.0)
    return out, int((out[:, 0] == 0).sum())


# ------------------------------------------------------------------------------------------------------------------
# Every table above -- DPM-Solver++(2M)'s and its inverse's (9 columns, all denoise entries), the distilled student's DDIM
# rows and RePaint's (REPAINT_COLUMNS) -- runs through one update kernel (mdb_solver_update) and one device loop
# (mdb_solver_run); _update_eager is the kernel's bit-exact CPU oracle.
def _rows32(table):
    """The table as float32 REPAINT_COLUMNS rows: a 9-column solver table gets kind 0 (denoise) on every row."""
    rows = np.asarray(table, dtype=np.float64)
    if rows.shape[1] == len(REPAINT_COLUMNS) - 1:
        rows = np.concatenate([np.zeros((len(rows), 1)), rows], axis=1)
    return rows.astype(np.float32)


def _entries_c(table):
    """The table (a 9-column solver table or REPAINT_COLUMNS) as the float32 mdb_solver_entry array the library takes."""
    rows = _rows32(table)
    arr = (_native.SolverEntryC * len(rows))()
    for i, r in enumerate(rows):
        arr[i] = _native.SolverEntryC(int(r[0]), *(float(v) for v in r[1:]))
    return arr


class _Known:
    """The kept region in the form the update kernel takes it: `known` fp32 [1 or B, C, R, R, R] (what the output must
    hold there), `mask` fp32 [1 or B, R, R, R] (1 = kept voxel; 1 / B samples = shared / per sample) and the replaced
    channels. The per-entry CUDA and CPU paths draw the replacement noise z' with torch.randn_like: one draw the shape
    of x (`full_noise`, RePaint), or one [B, R, R, R] draw per replaced channel (the conditional sampler's draw order)."""

    def __init__(self, known, mask, channels, B, full_noise=True):
        self.known = known.to(torch.float32).contiguous()
        C = self.known.shape[1]
        self.mask = mask.to(torch.float32).reshape(mask.shape[0], *self.known.shape[2:]).contiguous()
        for t in (self.known, self.mask):
            if t.shape[0] not in (1, B):
                raise ValueError("the kept region (known / mask) must have batch 1 or the sampling batch")
        self.channels = sorted({int(c) for c in channels})
        if not self.channels or self.channels[0] < 0 or self.channels[-1] >= C:
            raise ValueError(f"kept region: channels must be a non-empty subset of 0 .. {C - 1}, got {channels!r}")
        self.kb = self.known[0].numel() if self.known.shape[0] == B and B > 1 else 0
        self.mb = self.mask[0].numel() if self.mask.shape[0] == B and B > 1 else 0
        self.full_noise = full_noise

    def noise(self, x):
        """z' shaped like x (zero outside the replaced channels when not `full_noise`)."""
        if self.full_noise:
            return torch.randn_like(x)
        z = torch.zeros_like(x)
        for c in self.channels:
            z[:, c] = torch.randn_like(x[:, c])
        return z

    def struct(self, noise=None):
        s = _native.SolverKnownC()
        s.known, s.known_bstride = self.known.data_ptr(), self.kb
        s.mask, s.mask_bstride = self.mask.data_ptr(), self.mb
        s.channels = sum(1 << c for c in self.channels)
        s.noise = noise.data_ptr() if noise is not None else None
        return s


def _replace_channel(xc, known, kmask, mask, coef, std, z):
    """x_c <- (x_c (1 - m) + (coef known + std z) m) g, fp32, in solver_update_kernel's operation order."""
    sampled = known * coef + z * std
    return (xc * (1.0 - kmask) + sampled * kmask) * mask


def _update_eager(eps, x, x0_hist, mask, row, noise=None, known=None, known_noise=None, eps_u=None, w=1.0):
    """One entry in torch fp32 ops, in place on x and x0_hist, with the operation order of solver_update_kernel (each
    product and sum rounded on its own), so it is the kernel's bit-exact oracle. `row`: a float32 REPAINT_COLUMNS row
    (_rows32); `mask` broadcasts over x; `known`: a _Known; known_noise: z' shaped like x. With `eps_u` (the null-class
    output) a denoise entry uses the guided eps_u + w (eps - eps_u) in place of eps."""
    kind, _, sg, inv_a, c_x, c_0, c_1, c_z, coef, std = (float(v) for v in row)
    if kind:
        xn = (x * c_x + noise * c_z) * mask
    else:
        if eps_u is not None:
            eps = eps_u + (eps - eps_u) * float(np.float32(w))
        x0 = (x - eps * sg) * inv_a
        xn = x * c_x + x0 * c_0
        if c_1 != 0.0:
            xn = xn + x0_hist * c_1
        if c_z != 0.0:
            xn = xn + noise * c_z
        xn = xn * mask
        x0_hist.copy_(x0)
    if known is not None:
        for c in known.channels:
            xn[:, c] = _replace_channel(xn[:, c], known.known[:, c], known.mask, mask, coef, std, known_noise[:, c])
    x.copy_(xn)
    return x


def _update(eps, x, x0_hist, mask_flat, entry_c, noise=None, known=None, known_noise=None, seed=0, offset=0, eps_u=None,
            w=1.0):
    """One entry through mdb_solver_update (mdb_solver_update_guided with `eps_u`), in place on x and x0_hist;
    noise=None draws it in-kernel."""
    L = _native.lib()
    B, C = x.shape[0], x.shape[1]
    ks = known.struct(noise=known_noise) if known is not None else None
    if eps_u is not None:
        _native.check(L.mdb_solver_update_guided(_native.ptr(eps), _native.ptr(eps_u), float(w), _native.ptr(x),
                                                 _native.ptr(x0_hist), _native.ptr(mask_flat), ctypes.byref(entry_c),
                                                 x[0, 0].numel(), C, B, _native.ptr(noise), int(seed), int(offset),
                                                 ctypes.byref(ks) if ks is not None else None, _native.current_stream()))
        return x
    _native.check(L.mdb_solver_update(_native.ptr(eps), _native.ptr(x), _native.ptr(x0_hist), _native.ptr(mask_flat),
                                      ctypes.byref(entry_c), x[0, 0].numel(), C, B, _native.ptr(noise), int(seed),
                                      int(offset), ctypes.byref(ks) if ks is not None else None,
                                      _native.current_stream()))
    return x


def _native_run(net, x, x0_hist, mask_flat, entries_c, seed, step0=0, n=None, known=None, replace_until=None,
                class_ids=None, w=1.0):
    """Entries step0 .. step0+n-1 of a table inside the library (mdb_solver_run), in place on x and x0_hist. `entries_c`
    is the whole table (_entries_c), indexed by the GLOBAL entry; `known` is replaced after the global entries below
    `replace_until` (default: all of them). With `class_ids` (device int32 [B]) the table runs through
    mdb_solver_run_guided at guidance scale w."""
    L = _native.lib()
    B = x.shape[0]
    n = len(entries_c) - step0 if n is None else n
    replace_until = len(entries_c) if replace_until is None else replace_until
    net._ensure_engine(B, x.device)
    net.sync_parameters()
    eps_buf = torch.empty_like(x)
    labels_buf = torch.empty(B, device=x.device, dtype=torch.float32)
    part = (_native.SolverEntryC * n).from_buffer(entries_c, step0 * ctypes.sizeof(_native.SolverEntryC))
    ks = known.struct() if known is not None else None
    if class_ids is not None:
        eps_u_buf = torch.empty_like(x) if w != 1.0 else None
        _native.check(L.mdb_solver_run_guided(net._handle, _native.ptr(x), _native.ptr(x0_hist), _native.ptr(mask_flat), part,
                                              n, B, int(seed), _native.ptr(class_ids), float(w), _native.ptr(eps_buf),
                                              _native.ptr(eps_u_buf), _native.ptr(labels_buf), int(step0),
                                              ctypes.byref(ks) if ks is not None else None, int(replace_until),
                                              _native.current_stream()))
        return x
    net._set_classes(net._handle, None, B)
    _native.check(L.mdb_solver_run(net._handle, _native.ptr(x), _native.ptr(x0_hist), _native.ptr(mask_flat), part, n, B,
                                   int(seed), _native.ptr(eps_buf), _native.ptr(labels_buf), int(step0),
                                   ctypes.byref(ks) if ks is not None else None, int(replace_until),
                                   _native.current_stream()))
    return x


def _run_table(sde, table, model, x, grid_mask, name, known=None, replace_until=None, native=False, seed=0,
               class_labels=None, w=1.0):
    """Runs a solver table on x (fp32 [B, C, R, R, R]) and returns the result: the driver behind the four table samplers.

    x is multiplied by the grid mask first. With `known` (a _Known) its kept region is replaced at label N - 1 (alpha,
    sigma of N - 1, fresh noise), then after every entry below `replace_until` (default: all). Paths: with `native`, a
    native ScoreNet and x on CUDA the whole table runs in the library (mdb_solver_run, Philox noise keyed by `seed` and
    the entry); other CUDA states run model + mdb_solver_update per entry with torch.randn_like noise; CPU tensors run the
    eager fp32 update (_update_eager), which is the kernel's oracle.

    `class_labels` (ids of a class-conditional model, one per sample or one for the batch) conditions every network
    call; with w != 1 each denoise entry also calls the model without them (the null class) and uses the classifier-free
    guided eps_u + w (eps_c - eps_u)."""
    B = x.shape[0]
    w = float(w)
    if w != 1.0 and class_labels is None:
        raise ValueError(f"{name}: guidance_scale {w} needs class_labels")
    if grid_mask.numel() != x[0, 0].numel():
        raise ValueError(f"{name}: grid_mask must hold one value per voxel")
    mask_v = grid_mask.to(device=x.device, dtype=torch.float32).reshape(x.shape[2:]).contiguous()
    x = (x * mask_v).contiguous()
    rows, entries_c = _rows32(table), _entries_c(table)
    replace_until = len(rows) if replace_until is None else replace_until
    if known is not None:
        abar_T = float(sde.alphas_cumprod[sde.N - 1])
        a_T, s_T = (float(np.float32(v)) for v in (np.sqrt(abar_T), np.sqrt(1.0 - abar_T)))
        z = known.noise(x)
        for c in known.channels:
            x[:, c] = _replace_channel(x[:, c], known.known[:, c], known.mask, mask_v, a_T, s_T, z[:, c])
    x0_hist = torch.empty_like(x)
    net = _native_net(model)
    if native and x.is_cuda and net is not None:
        net._ensure_engine(B, x.device)
        ids = net._class_ids(class_labels, B, x.device)
        with net.frozen():  # nobody edits the weights inside the loop: skip per-step change detection
            return _native_run(net, x, x0_hist, mask_v.reshape(-1), entries_c, seed, known=known,
                               replace_until=replace_until, class_ids=ids, w=w)
    for e, row in enumerate(rows):
        renoise = row[0] != 0
        eps = eps_u = None
        if not renoise:
            lab = torch.full((B,), float(row[1]), device=x.device)
            eps = (model(x, lab) if class_labels is None else model(x, lab, class_labels=class_labels)).float()
            if w != 1.0:
                eps_u = model(x, lab).float().contiguous()
        noise = torch.randn_like(x) if (renoise or row[7] != 0) else None
        ke = known if e < replace_until else None
        z2 = ke.noise(x) if ke is not None else None
        if x.is_cuda:
            _update(None if renoise else eps.contiguous(), x, x0_hist, mask_v.reshape(-1), entries_c[e], noise, ke, z2,
                    eps_u=eps_u, w=w)
        else:
            _update_eager(eps, x, x0_hist, mask_v, row, noise, ke, z2, eps_u=eps_u, w=w)
    return x


def get_dpm_solver_sampler(sde, shape, inverse_scaler, n_steps=25, stochastic=False, denoise=True, device="cuda",
                           grid_mask=None, native_rng=False, seed=42, guidance_scale=1.0):
    """Returns `dpm_solver_sampler(model, partial=None, partial_mask=None, partial_channel=0, freeze_iters=None, x0=None)`
    -> (samples, number of network evaluations), the signature of pc_sampler, on dpm_solver_schedule's labels and table.

    The prior is pc_sampler's (sde.prior_sampling(shape) * grid_mask), or x0 * grid_mask when `x0` (shape `shape`) is
    given: no prior is drawn then. With `partial`, channel c is replaced before step 0
    (alpha, sigma of label N-1) and after every step k but the last whose label n_k has N-1-n_k < freeze_iters (alpha,
    sigma of n_{k+1}), with fresh per-sample noise; the x0 history keeps the network's prediction. Paths (_run_table): on
    CUDA with `native_rng` and a native ScoreNet the whole loop runs in the library (mdb_solver_run, Philox noise keyed by
    seed + rank and step); other CUDA states run model + mdb_solver_update per step with torch.randn_like noise; CPU
    tensors run the eager fp32 update (_update_eager), which is the kernel's oracle.

    The sampler also takes `class_labels` (a class-conditional model's ids) and `guidance_scale` (w, default the one
    given here): w != 1 is classifier-free guidance, two network evaluations per step (_run_table)."""
    labels, table = dpm_solver_schedule(sde, n_steps, stochastic, denoise)
    return _solver_sampler(sde, shape, inverse_scaler, labels, table, device, grid_mask, native_rng, seed, "dpm_solver",
                           guidance_scale)


def get_distilled_sampler(sde, shape, inverse_scaler, n_steps=8, device="cuda", grid_mask=None, native_rng=False, seed=42,
                          guidance_scale=1.0):
    """The sampler of a progressively distilled student (`sampling.method='distilled'`, `sampling.distill_steps`): the
    DDIM ODE on `ddim_grid(sde, n_steps)`, through get_dpm_solver_sampler's paths and conditioning with the first-order
    rows of `ddim_table`. Same signature and return as get_dpm_solver_sampler."""
    labels = ddim_grid(sde, n_steps)
    return _solver_sampler(sde, shape, inverse_scaler, labels, ddim_table(sde, labels), device, grid_mask, native_rng,
                           seed, "distilled", guidance_scale)


def _solver_sampler(sde, shape, inverse_scaler, labels, table, device, grid_mask, native_rng, seed, name, guidance_scale=1.0):
    """get_dpm_solver_sampler's sampler on any 9-column solver table along `labels`."""
    K_eff = len(labels) - 1

    def dpm_solver_sampler(model, partial=None, partial_mask=None, partial_channel=0, freeze_iters=None, x0=None,
                           class_labels=None, guidance_scale=guidance_scale):
        w = float(guidance_scale)
        with torch.no_grad():
            if freeze_iters is None:
                freeze_iters = sde.N + 10
            c = partial_channel
            if x0 is not None and tuple(x0.shape) != tuple(shape):
                raise ValueError(f"{name}: x0 has shape {tuple(x0.shape)}, the sampler {tuple(shape)}")
            x = sde.prior_sampling(shape).to(device) if x0 is None else x0.to(device=device, dtype=torch.float32)
            assert x.dim() == 5
            known, until = None, 0
            if partial is not None:
                assert partial.dim() == 5
                # only channel c of partial (cond_gen's has that one channel) and of partial_mask counts
                kept = torch.zeros(partial.shape[0], *x.shape[1:], device=x.device)
                kept[:, c] = partial[:, c]
                known = _Known(kept, partial_mask[:, c].to(x.device), [c], shape[0], full_noise=False)
                until = sum(1 for k in range(K_eff - 1) if sde.N - 1 - labels[k] < freeze_iters)
            x = _run_table(sde, table, model, x, grid_mask, name, known, until, native_rng, seed + _rank(), class_labels, w)
            return inverse_scaler(x), K_eff * (2 if w != 1.0 else 1)

    return dpm_solver_sampler


def get_dpm_solver_inverter(sde, shape, n_steps=25, grid_mask=None, device="cuda"):
    """Returns `invert(model, x) -> (z, number of network evaluations)`: the latent at label N - 1 of grids x (shape
    `shape`), taken as the state at label 0 after the grid mask is applied, by the ODE form of DPM-Solver++(2M) run
    backwards (dpm_solver_inversion_schedule). The dpm_solver sampler with the same `n_steps`, started from z
    (x0=z), maps it back to x up to discretisation error. No noise is drawn. Paths (_run_table): a native ScoreNet on
    CUDA runs the whole loop in the library (mdb_solver_run); other CUDA models run model + mdb_solver_update per step;
    CPU tensors run the eager fp32 update."""
    labels, table = dpm_solver_inversion_schedule(sde, n_steps)

    def invert(model, x):
        with torch.no_grad():
            if tuple(x.shape) != tuple(shape):
                raise ValueError(f"dpm_solver inversion: x has shape {tuple(x.shape)}, expected {tuple(shape)}")
            x = x.to(device=device, dtype=torch.float32)
            return _run_table(sde, table, model, x, grid_mask, "dpm_solver inversion", native=True), len(labels) - 1

    return invert


def get_repaint_sampler(sde, shape, inverse_scaler, n_steps=25, jump=5, resample=5, stochastic=False, denoise=True,
                        device="cuda", grid_mask=None, native_rng=False, seed=42):
    """Returns `repaint_sampler(model, known, known_mask, channels, x0=None)` -> (samples, number of network
    evaluations): samples of shape `shape` whose kept region (known_mask = 1, batch 1 or shape[0]) holds `known` (batch 1
    or shape[0]) exactly on `channels`, the rest regenerated by repaint_schedule's entries.

    The prior is sde.prior_sampling(shape) * grid_mask, or x0 * grid_mask; its kept region is replaced at label N - 1
    (alpha, sigma of N - 1, fresh noise), as the conditional dpm_solver sampler does. Paths (_run_table): on CUDA with
    `native_rng` and a native ScoreNet the whole schedule runs in the library (mdb_solver_run, Philox noise keyed by
    seed + rank and entry); other CUDA states run model + mdb_solver_update per entry with torch.randn_like noise; CPU
    tensors run the eager fp32 update (_update_eager), which is the kernel's oracle."""
    table, nfe = repaint_schedule(sde, n_steps, jump, resample, stochastic, denoise)

    def repaint_sampler(model, known, known_mask, channels, x0=None):
        with torch.no_grad():
            if x0 is not None and tuple(x0.shape) != tuple(shape):
                raise ValueError(f"repaint: x0 has shape {tuple(x0.shape)}, the sampler {tuple(shape)}")
            x = sde.prior_sampling(shape).to(device) if x0 is None else x0.to(device=device, dtype=torch.float32)
            if tuple(known.shape[1:]) != tuple(shape[1:]):
                raise ValueError(f"repaint: known has shape {tuple(known.shape)}, the sampler {tuple(shape)}")
            kn = _Known(known.to(x.device), known_mask.to(x.device), channels, shape[0])
            x = _run_table(sde, table, model, x, grid_mask, "repaint", kn, None, native_rng, seed + _rank())
            return inverse_scaler(x), nfe

    return repaint_sampler
