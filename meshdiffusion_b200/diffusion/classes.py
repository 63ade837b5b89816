"""Class conditioning for training and sampling: config validation and class-name resolution, the per-class dataset,
class-dependent synthetic grids and label dropout (the null class of classifier-free guidance).

Config keys (all absent = one unconditional network, today's behaviour):
  model.num_classes          K, the number of classes (0)
  data.class_meta_paths      one meta JSON per class; class k is the list position
  data.class_filter_meta_paths   optional, one filter list per class
  data.class_names           optional, one name per class
  training.class_dropout     probability of replacing a label with the null class K (0.1)
  sampling.guidance_scale    w of classifier-free guidance (1.0)
  eval.class_label           an id or a name from data.class_names (none: the null class)
"""
import torch
from torch.utils.data import ConcatDataset, Dataset

def num_classes(config):
    return int(config.model.get("num_classes", 0) or 0)


def _unset(v):
    return v in (None, "", "PLACEHOLDER")


def validate(config):
    """Checks the class keys against model.num_classes; returns K."""
    K = num_classes(config)
    if K < 0:
        raise ValueError(f"model.num_classes must be >= 0, got {K}")
    for key in ("class_meta_paths", "class_filter_meta_paths", "class_names"):
        v = config.data.get(key, None)
        if _unset(v):
            continue
        if K == 0:
            raise ValueError(f"data.{key} is set but model.num_classes is 0")
        if len(v) != K:
            raise ValueError(f"data.{key} lists {len(v)} entries for model.num_classes = {K}")
    names = config.data.get("class_names", None)
    if not _unset(names) and len(set(names)) != len(names):
        raise ValueError(f"data.class_names has duplicates: {list(names)}")
    p = float(config.training.get("class_dropout", 0.1))
    if not 0.0 <= p <= 1.0:
        raise ValueError(f"training.class_dropout must be in [0, 1], got {p}")
    w = float(config.sampling.get("guidance_scale", 1.0))
    if w != 1.0 and K == 0:
        raise ValueError(f"sampling.guidance_scale {w} needs a class-conditional network (model.num_classes > 0)")
    return K


def resolve_class_label(config):
    """eval.class_label as an id in 0..K-1 (a name is looked up in data.class_names), or None when unset."""
    K = validate(config)
    label = config.eval.get("class_label", None)
    if _unset(label):
        if float(config.sampling.get("guidance_scale", 1.0)) != 1.0:
            raise ValueError("sampling.guidance_scale != 1 needs eval.class_label")
        return None
    if K == 0:
        raise ValueError("eval.class_label is set but model.num_classes is 0")
    if isinstance(label, str) and not label.lstrip("-").isdigit():
        names = config.data.get("class_names", None)
        if _unset(names) or label not in list(names):
            raise ValueError(f"eval.class_label {label!r} is not in data.class_names {list(names or [])}")
        return list(names).index(label)
    k = int(label)
    if not 0 <= k < K:
        raise ValueError(f"eval.class_label {k} is outside 0..{K - 1}")
    return k


def sampling_kwargs(config):
    """The class_labels keyword of a sampler call for `uncond_gen` / `cond_gen`: {} for the unconditional behaviour."""
    k = resolve_class_label(config)
    return {} if k is None else {"class_labels": k}


def refuse_conditional(config, mode):
    """The modes whose conditional versions are not built refuse a class-conditional network (and so its checkpoint)."""
    if num_classes(config) > 0:
        raise ValueError(f"--mode={mode} does not support class-conditional networks (model.num_classes = "
                         f"{num_classes(config)}) yet")


class _Labeled(Dataset):
    """Items (grid, k) of one class's dataset."""

    def __init__(self, dataset, k):
        self.dataset, self.k = dataset, int(k)

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, idx):
        return self.dataset[idx], self.k


def class_dataset(datasets):
    """One dataset per class, joined: items (grid, class) with class = the position of the dataset."""
    return ConcatDataset([_Labeled(d, k) for k, d in enumerate(datasets)])


def synthetic_class_grids(labels, resolution, device, generator=None):
    """trainer.synthetic_grids with the sphere's radius set by the class: 0.2 + 0.05 k for labels [B] in 0..K-1."""
    from ..geometry.dmtet import grid_coords_of_tet_vertices, load_tet_grid
    verts, _ = load_tet_grid(resolution)
    v = torch.tensor(verts, device=device)
    c = grid_coords_of_tet_vertices(v.cpu()).to(device)
    r = v.norm(dim=1)
    radius = 0.2 + 0.05 * labels.to(device).float()
    B = labels.shape[0]
    sdf = torch.sign(radius[:, None] - r[None, :])
    near = ((r[None, :] - radius[:, None]).abs() < (1.0 / resolution)).float()
    x = torch.zeros(B, 4, resolution, resolution, resolution, device=device)
    x[:, 0, c[:, 0], c[:, 1], c[:, 2]] = sdf
    d = (torch.rand(B, 3, v.shape[0], device=device, generator=generator) - 0.5) * near[:, None, :]
    x[:, 1:, c[:, 0], c[:, 1], c[:, 2]] = d
    return x


def drop_labels(labels, K, p, generator=None):
    """Classifier-free guidance training: each label is replaced by the null class K with probability p, drawn on the
    labels' device from `generator`."""
    if p <= 0.0:
        return labels
    drop = torch.rand(labels.shape, device=labels.device, generator=generator) < p
    return torch.where(drop, torch.full_like(labels, K), labels)
