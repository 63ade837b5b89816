"""Model registry, model creation and score-function wrappers.

Same names / call conventions as the reference's lib/diffusion/models/utils.py (register_model/get_model :27-47,
get_sigmas :50-61, create_model :88-96, get_model_fn :99-125, get_score_fn :167-203).
"""
import numpy as np
import torch

_MODELS = {}


def register_model(cls=None, *, name=None):
    """`@register_model(name=...)` decorator or `register_model(cls, name=...)` call."""

    def _add(c):
        key = name if name is not None else c.__name__
        if key in _MODELS:
            raise ValueError(f"Already registered model with name: {key}")
        _MODELS[key] = c
        return c

    return _add if cls is None else _add(cls)


def get_model(name):
    return _MODELS[name]


def get_sigmas(config):
    """Geometric noise-level ladder kept in every checkpoint as the float64 `sigmas` buffer."""
    m = config.model
    return np.exp(np.linspace(np.log(m.sigma_max), np.log(m.sigma_min), m.num_scales))


class ReplicaShell(torch.nn.Module):
    """Takes the place of `torch.nn.DataParallel` in the reference's create_model (models/utils.py:95).

    The reference replicates the weights to every visible GPU on each forward; here every process owns one GPU
    (batch sharding for sampling, NCCL gradient all-reduce for training), so the shell only preserves the two
    things callers and checkpoints depend on: the `.module` attribute and the `module.` state-dict prefix.
    """

    def __init__(self, module):
        super().__init__()
        self.module = module

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)


def create_model(config, use_parallel=True):
    from . import ddpm  # noqa: F401  (registers the score networks)
    net = get_model(config.model.name)(config)
    if use_parallel:
        net = ReplicaShell(net).to(config.device)
    return net


def get_model_fn(model, train=False):
    def model_fn(x, labels, class_labels=None):
        model.train() if train else model.eval()
        if class_labels is None:
            return model(x, labels)
        return model(x, labels, class_labels=class_labels)

    return model_fn


def get_score_fn(sde, model, train=False, continuous=False, std_scale=True):
    """VP-SDE score from the noise-prediction network: labels = t (N-1); score = -eps / std.

    continuous=False: std = sqrt(1 - alpha_bar)[labels.long()], the discrete table the sampler and the loss use.
    continuous=True: std = sde.marginal_prob(0, t)[1], smooth in t -- the form the probability-flow likelihood asks for
    (the reference's likelihood.py:61, score_sde's VP likelihood): the table lookup is piecewise constant, so the ODE's
    right-hand side would jump N - 1 times on [eps, 1] and an adaptive solver would reject a step at every jump."""
    from .. import sde_lib
    if not isinstance(sde, sde_lib.VPSDE):
        raise NotImplementedError(f"SDE class {sde.__class__.__name__} not yet supported.")
    model_fn = get_model_fn(model, train=train)

    def score_fn(x, t, class_labels=None):
        labels = t * (sde.N - 1)
        eps = model_fn(x, labels, class_labels)
        if not std_scale:
            return eps
        if continuous:
            std = sde.marginal_prob(torch.zeros_like(x), t)[1]
        else:
            std = sde.sqrt_1m_alphas_cumprod.to(labels.device)[labels.long()]
        return -eps / std[:, None, None, None, None]

    return score_fn


def to_flattened_numpy(x):
    return x.detach().cpu().numpy().reshape((-1,))


def from_flattened_numpy(x, shape):
    return torch.from_numpy(x.reshape(shape))
