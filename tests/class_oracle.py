"""fp32 forward of a class-conditional score network, on top of oracle/unet_oracle.py.

The conditional network adds row y of `label_embed.weight` to the output of `all_modules.1` before the SiLU. That
Linear's bias is added right there too, so the conditional forward is the unconditional oracle with a per-sample bias
b1 + E[y]. With a zero embedding the bias is b1 on every row and the result equals the unconditional oracle exactly.
"""
import torch

from oracle import unet_oracle


def unet_forward(sd, arch, x, labels, class_labels=None):
    """score_model(x, labels, class_labels) in eval mode; class_labels None or K = the null class."""
    if "label_embed.weight" not in sd:
        if class_labels is not None:
            raise ValueError("class_labels given to an unconditional state dict")
        return unet_oracle.unet_forward(sd, arch, x, labels)
    E = sd["label_embed.weight"]
    K = E.shape[0] - 1
    B = x.shape[0]
    y = torch.full((B,), K, dtype=torch.long) if class_labels is None else torch.as_tensor(class_labels).long().reshape(-1)
    y = y.to(E.device).expand(B) if y.numel() == 1 else y.to(E.device)
    sd = dict(sd)
    sd["all_modules.1.bias"] = sd["all_modules.1.bias"][None, :] + E[y]
    return unet_oracle.unet_forward(sd, arch, x, labels)
