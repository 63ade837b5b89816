"""Log-likelihood of data under the probability-flow ODE (reference: lib/diffusion/likelihood.py:26-113).

`get_likelihood_fn(...)(model, data)` integrates dx/dt = drift(x, t) together with d(log p)/dt = div drift from t = eps to
t = 1 with `scipy.integrate.solve_ivp` over a flat fp64 host state, as the reference does, and returns (bpd, z, nfe). The
score is the continuous VP form -e / std(t) (`get_score_fn(..., continuous=True)`), and the divergence is the
Hutchinson-Skilling estimate h^T (d drift / d x) h.

Two ways to evaluate the right-hand side:
  * generic (any torch model): the reference's arithmetic, with the divergence from `torch.autograd.grad`;
  * native (the model is a `ScoreNet`): one forward of the training-plan engine, one input-only backward
    (`mdb_unet_backward_input`, no parameter gradients) and one fused `mdb_pflow_drift_div` pass.

Conventions. With `grid_mask=None` the ODE runs over every entry of `data` and bpd carries the reference's
dequantisation offset 7 - inverse_scaler(-1) (an 8-bit image convention). With a grid mask the ODE runs over the
D = C |mask| live entries only (the state is gathered to them), the Hutchinson noise is zero outside the mask, the prior
is taken over those D dimensions and bpd = -(log p_T(z) + delta log p) / (D ln 2), with no offset: DMTet grids are not
quantised images.
"""
import numpy as np
import torch
from scipy import integrate

from .. import _native
from .models import utils as mutils

MASKED_CONVENTION = "masked: D = C*|mask| live dimensions, bpd = -(log p_T(z) + delta log p) / (D ln 2), no offset"
REFERENCE_CONVENTION = "reference: all dimensions, bpd offset 7 - inverse_scaler(-1)"


def get_div_fn(fn):
    """Divergence of `fn` by the Hutchinson-Skilling trace estimator: sum(noise * d(fn . noise)/dx)."""

    def div_fn(x, t, eps):
        with torch.enable_grad():
            x.requires_grad_(True)
            fn_eps = torch.sum(fn(x, t) * eps)
            grad_fn_eps = torch.autograd.grad(fn_eps, x)[0]
        x.requires_grad_(False)
        return torch.sum(grad_fn_eps * eps, dim=tuple(range(1, len(x.shape))))

    return div_fn


def hutchinson_noise(like, hutchinson_type, generator=None):
    if hutchinson_type == "Gaussian":
        return torch.randn(like.shape, generator=generator, device=like.device, dtype=like.dtype)
    if hutchinson_type == "Rademacher":
        return torch.randint(0, 2, like.shape, generator=generator, device=like.device).to(like.dtype) * 2 - 1.0
    raise NotImplementedError(f"Hutchinson type {hutchinson_type} unknown.")


def _native_net(model):
    from .models.ddpm import ScoreNet
    net = getattr(model, "module", model)
    return net if isinstance(net, ScoreNet) else None


def get_likelihood_fn(sde, inverse_scaler, hutchinson_type="Rademacher", rtol=1e-5, atol=1e-5, method="RK45", eps=1e-5,
                      grid_mask=None):
    """Returns likelihood_fn(model, data, noise=None) -> (bpd [B], z (data's shape), nfe). `noise` is the Hutchinson noise
    (data's shape); when omitted it is drawn like the reference draws it (`torch.randint_like` / `torch.randn_like`).
    `grid_mask`: [R,R,R] (or broadcastable [1,1,R,R,R]) 0/1 mask selecting the live grid entries, or None."""
    if hutchinson_type not in ("Rademacher", "Gaussian"):
        raise NotImplementedError(f"Hutchinson type {hutchinson_type} unknown.")

    def drift_fn(model, x, t):
        """VPSDE.sde + reverse(probability_flow=True) with the continuous score, in the reference's operation order."""
        score_fn = mutils.get_score_fn(sde, model, train=False, continuous=True)
        drift, diffusion = sde.sde(x, t)
        return drift - diffusion[:, None, None, None, None] ** 2 * score_fn(x, t) * 0.5

    def div_fn(model, x, t, noise):
        return get_div_fn(lambda xx, tt: drift_fn(model, xx, tt))(x, t, noise)

    def likelihood_fn(model, data, noise=None):
        with torch.no_grad():
            shape = data.shape
            B = shape[0]
            if noise is None:
                if hutchinson_type == "Gaussian":
                    noise = torch.randn_like(data)
                else:
                    noise = torch.randint_like(data, low=0, high=2).float() * 2 - 1.0
            if grid_mask is None:
                return _reference_convention(model, data, noise, shape, B)
            return _masked_convention(model, data, noise, shape, B)

    def _reference_convention(model, data, noise, shape, B):
        def ode_func(t, x):
            sample = mutils.from_flattened_numpy(x[:-B], shape).to(data.device).type(torch.float32)
            vec_t = torch.ones(sample.shape[0], device=sample.device) * t
            drift = mutils.to_flattened_numpy(drift_fn(model, sample, vec_t))
            logp_grad = mutils.to_flattened_numpy(div_fn(model, sample, vec_t, noise))
            return np.concatenate([drift, logp_grad], axis=0)

        init = np.concatenate([mutils.to_flattened_numpy(data), np.zeros((B,))], axis=0)
        solution = integrate.solve_ivp(ode_func, (eps, sde.T), init, rtol=rtol, atol=atol, method=method)
        nfe = solution.nfev
        zp = solution.y[:, -1]
        z = mutils.from_flattened_numpy(zp[:-B], shape).to(data.device).type(torch.float32)
        delta_logp = mutils.from_flattened_numpy(zp[-B:], (B,)).to(data.device).type(torch.float32)
        prior_logp = sde.prior_logp(z)
        bpd = -(prior_logp + delta_logp) / np.log(2)
        N = np.prod(shape[1:])
        bpd = bpd / N
        offset = 7.0 - inverse_scaler(-1.0)
        bpd = bpd + offset
        return bpd, z, nfe

    def _masked_convention(model, data, noise, shape, B):
        C = shape[1]
        m = grid_mask.reshape(-1).to(data.device).float()
        live = torch.nonzero(m, as_tuple=False).reshape(-1)
        M = live.numel()
        D = C * M
        if D == 0:
            raise ValueError("the grid mask selects no entries")
        V = m.numel()
        h = noise.reshape(B, C, V).float() * m  # zero outside the mask
        net = _native_net(model)

        def scatter(state):
            full = torch.zeros(B, C, V, device=data.device, dtype=torch.float32)
            full[:, :, live] = torch.from_numpy(state.reshape(B, C, M)).to(data.device, torch.float32)
            return full

        if net is not None:
            if net.scale_by_sigma:
                raise ValueError("the native likelihood path needs a network with scale_by_sigma=False")
            drift = torch.empty(B, C, V, device=data.device, dtype=torch.float32)
            div = torch.empty(B, device=data.device, dtype=torch.float64)
            h = h.contiguous()
            m_c = m.contiguous()
            L = _native.lib()

            def rhs(t, x):
                vec_t = torch.ones(B, device=data.device) * t
                std = float(sde.marginal_prob(torch.zeros(1, 1, 1, 1, 1, device=data.device), vec_t[:1])[1][0])
                beta = float(sde.beta_0 + t * (sde.beta_1 - sde.beta_0))
                e, g = net.score_vjp(x.reshape(shape), vec_t * (sde.N - 1), h.reshape(shape))
                _native.check(L.mdb_pflow_drift_div(_native.ptr(x), _native.ptr(e), _native.ptr(h), _native.ptr(g), _native.ptr(m_c),
                                                     beta, std, _native.ptr(drift), _native.ptr(div), B, C, V,
                                                     _native.current_stream()))
                return drift, div
        else:
            def rhs(t, x):
                sample = x.reshape(shape)
                vec_t = torch.ones(B, device=data.device) * t
                mk = m.reshape((1, 1) + tuple(shape[2:]))
                d = drift_fn(model, sample, vec_t) * mk
                dv = get_div_fn(lambda xx, tt: drift_fn(model, xx, tt) * mk)(sample, vec_t, h.reshape(shape))
                return d.reshape(B, C, V), dv.double()

        def ode_func(t, state):
            drift, div = rhs(t, scatter(state[:-B]))
            return np.concatenate([drift[:, :, live].double().cpu().numpy().reshape(-1), div.cpu().numpy()], axis=0)

        x0 = data.reshape(B, C, V)[:, :, live].double().cpu().numpy().reshape(-1)
        init = np.concatenate([x0, np.zeros((B,))], axis=0)
        solution = integrate.solve_ivp(ode_func, (eps, sde.T), init, rtol=rtol, atol=atol, method=method)
        zp = solution.y[:, -1]
        zl = zp[:-B].reshape(B, D)
        delta_logp = zp[-B:]
        prior_logp = -D / 2.0 * np.log(2 * np.pi) - np.sum(zl ** 2, axis=1) / 2.0
        bpd = -(prior_logp + delta_logp) / (D * np.log(2))
        z = scatter(zp[:-B]).reshape(shape)
        return torch.from_numpy(bpd), z, solution.nfev

    return likelihood_fn
