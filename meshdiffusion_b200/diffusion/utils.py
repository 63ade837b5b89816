"""Checkpoint IO. The on-disk layout is the reference's (lib/diffusion/utils.py:6-30) so files interchange:
one `torch.save` of a dict with the four entries of `CKPT_FIELDS`; `model` carries the `module.` key prefix of the
DataParallel-shaped shell, `ema` the positional shadow list, `step` the micro-step counter."""
import logging
import os

import torch

# entry -> how it is captured from / poured back into the training state
CKPT_FIELDS = ("optimizer", "model", "ema", "step")


def _capture(state):
    out = {}
    for key in CKPT_FIELDS:
        obj = state[key]
        out[key] = obj if key == "step" else obj.state_dict()
    return out


def save_checkpoint(ckpt_dir, state):
    """Writes `state` (optimizer / model / ema / step) to the file `ckpt_dir` (the reference's name for the path)."""
    parent = os.path.dirname(ckpt_dir)
    if parent:
        os.makedirs(parent, exist_ok=True)
    torch.save(_capture(state), ckpt_dir)


def restore_checkpoint(ckpt_dir, state, device, strict=False):
    """Loads a checkpoint into `state` in place and returns it. A missing file is not an error (fresh run): like the
    reference it only warns and prepares the directory -- unless `strict`, which raises."""
    if not os.path.exists(ckpt_dir):
        if strict:
            raise FileNotFoundError(ckpt_dir)
        parent = os.path.dirname(ckpt_dir)
        if parent:
            os.makedirs(parent, exist_ok=True)
        logging.warning("No checkpoint found at %s. Returned the same state as input", ckpt_dir)
        return state
    blob = torch.load(ckpt_dir, map_location=device, weights_only=False)
    net = getattr(state["model"], "module", None)
    if hasattr(net, "num_classes"):  # before the optimiser's positional state is matched against the parameters
        from .models.ddpm import check_class_count
        check_class_count(blob["model"], net.num_classes, "module.label_embed.weight")
    for key in CKPT_FIELDS:
        if key == "step":
            state[key] = blob[key]
        elif key == "model":
            state[key].load_state_dict(blob[key], strict=False)  # tolerate extra / missing buffers as the reference does
        else:
            state[key].load_state_dict(blob[key])
    return state
