"""Training-step host logic behind the reference's callables (lib/diffusion/losses.py:26-141): `get_optimizer`,
`optimization_manager`, `get_ddpm_loss_fn`, `get_step_fn`. Semantics kept:

* Adam(lr, (beta1, 0.999), eps, weight_decay); linear learning-rate warm-up on the MICRO-step counter, then
  `clip_grad_norm_`, then `optimizer.step()`.
* loss = mean_b[ mean_{c,v}((eps_theta - eps)^2 * mask) ] * numel(mask) / sum(mask) (l2; l1 uses |.|), with
  integer labels ~ U{0..N-1} and x_t = (sqrt(abar_t) x_0 + sqrt(1-abar_t) eps) * mask.
* `step_fn(state, batch, clear_grad, update_param)`: gradients of successive micro-batches add up (no division),
  `state['step']` and the EMA advance on EVERY micro-step, evaluation runs under the EMA weights.

The network forward and backward run inside the sm_90a engine; `loss.backward()` reaches it through one autograd node
(models/ddpm.py::_ScoreNetFn). The arithmetic around it runs in the library's optimiser-side kernels (train_ops.py):
the forward perturbation and the masked l2 loss + its gradient (mdb_ddpm_perturb / mdb_ddpm_loss, one autograd node),
clip_grad_norm_ as a coefficient (mdb_grad_clip_coef) and Adam + the EMA update in ONE pass over the parameters
(mdb_adam_ema_step). The optimiser is still a torch.optim.Adam as far as `state_dict()` / `param_groups` go.
"""
import numpy as np
import torch

from .. import train_ops
from .models import utils as mutils
from .sde_lib import VPSDE

_PENALTIES = {"l2": torch.square, "l1": torch.abs}


def get_optimizer(config, params):
    o = config.optim
    if o.optimizer != "Adam":
        raise NotImplementedError(f"Optimizer {o.optimizer} not supported yet!")
    return train_ops.FusedAdam(params, lr=o.lr, betas=(o.beta1, 0.999), eps=o.eps, weight_decay=o.weight_decay)


def optimization_manager(config):
    base_lr, base_warmup, base_clip = config.optim.lr, config.optim.warmup, config.optim.grad_clip

    def optimize_fn(optimizer, params, step, lr=base_lr, warmup=base_warmup, grad_clip=base_clip, ema=None):
        """Warm-up, clipping and the Adam step of the reference's optimize_fn (losses.py:38-52). With the library's
        FusedAdam the clip is a device-side coefficient and `ema` (optional) is updated in the same pass; returns True
        when that happened, so that step_fn does not update the EMA a second time."""
        if warmup > 0:
            scaled = lr * np.minimum(step / warmup, 1.0)
            for group in optimizer.param_groups:
                group["lr"] = scaled
        if isinstance(optimizer, train_ops.FusedAdam):
            if grad_clip >= 0:
                optimizer.grad_norm_coef(grad_clip)
            return optimizer.step(ema=ema)
        if grad_clip >= 0:  # a user-supplied stock optimiser: the reference's own sequence
            torch.nn.utils.clip_grad_norm_(list(params), max_norm=grad_clip)
        optimizer.step()
        return False

    return optimize_fn


def get_ddpm_loss_fn(vpsde, train, mask=None, loss_type="l2"):
    if not isinstance(vpsde, VPSDE):
        raise TypeError("DDPM training only works for VPSDEs.")
    if loss_type not in _PENALTIES:
        raise NotImplementedError(loss_type)
    penalty = _PENALTIES[loss_type]

    mask_sum = [None]

    def loss_fn(model, batch, class_labels=None):
        dev = batch.device
        model_fn = mutils.get_model_fn(model, train=train)
        net = lambda x, t: model_fn(x, t, class_labels)  # noqa: E731
        t = torch.randint(0, vpsde.N, (batch.shape[0],), device=dev)
        eps = torch.randn_like(batch)
        if batch.is_cuda and mask is not None and loss_type == "l2" and batch.dtype == torch.float32:
            # native tail: one pass builds x_t, one pass gives the loss and d loss / d prediction (same arithmetic as below)
            x_t = train_ops.ddpm_perturb(batch, eps, mask, vpsde.sqrt_alphas_cumprod.to(dev)[t], vpsde.sqrt_1m_alphas_cumprod.to(dev)[t])
            if mask_sum[0] is None:
                mask_sum[0] = float(mask.sum().item())  # the mask is fixed for the life of the step function
            return train_ops.DDPMLossFn.apply(net(x_t, t), eps, mask, mask_sum[0])
        signal = vpsde.sqrt_alphas_cumprod.to(dev)[t, None, None, None, None]
        sigma = vpsde.sqrt_1m_alphas_cumprod.to(dev)[t, None, None, None, None]
        x_t = (signal * batch + sigma * eps) * mask
        err = penalty(net(x_t, t) - eps)
        if mask is None:
            return err.reshape(err.shape[0], -1).mean(dim=-1).mean()
        per_sample = (err * mask).reshape(err.shape[0], -1).mean(dim=-1)
        return per_sample.mean() / mask.sum() * np.prod(mask.size())

    return loss_fn


def get_update_fn(optimize_fn=None):
    """`update(state, loss, update_param)`: the optimiser and EMA sequencing of a training micro-step, shared by
    `--mode=train` and `--mode=distill`: backward, then (last micro-batch only) optimize_fn, then the micro-step counter
    and the EMA, which advance on every micro-step (losses.py:104-139 of the reference)."""
    takes_ema = False
    if optimize_fn is not None:
        import inspect
        ps = inspect.signature(optimize_fn).parameters
        takes_ema = "ema" in ps or any(p.kind is inspect.Parameter.VAR_KEYWORD for p in ps.values())

    def update(state, loss, update_param):
        model, optimizer = state["model"], state["optimizer"]
        loss.backward()
        ema_done = False
        if update_param:
            kw = {"ema": state["ema"]} if takes_ema else {}  # an optimize_fn with the reference's exact signature has no `ema`
            ema_done = optimize_fn(optimizer, model.parameters(), step=state["step"], **kw) is True
        state["step"] += 1
        if not ema_done:
            state["ema"].update(model.parameters())

    return update


def get_step_fn(sde, train, optimize_fn=None, mask=None, loss_type="l2"):
    loss_fn = get_ddpm_loss_fn(sde, train, mask=mask, loss_type=loss_type)
    update = get_update_fn(optimize_fn)

    def train_step(state, batch, clear_grad, update_param, class_labels=None):
        model, optimizer = state["model"], state["optimizer"]
        if clear_grad:
            optimizer.zero_grad()
        loss = loss_fn(model, batch, class_labels)
        update(state, loss, update_param)
        return loss

    def eval_step(state, batch, class_labels=None):
        model, ema = state["model"], state["ema"]
        with torch.no_grad():
            ema.store(model.parameters())
            ema.copy_to(model.parameters())
            try:
                return loss_fn(model, batch, class_labels)
            finally:
                ema.restore(model.parameters())

    def step_fn(state, batch, clear_grad=True, update_param=True, class_labels=None):
        """class_labels: the ids of a class-conditional network's batch (None: unconditional / the null class)."""
        loss = (train_step(state, batch, clear_grad, update_param, class_labels) if train
                else eval_step(state, batch, class_labels))
        return {"loss": loss}

    return step_fn
