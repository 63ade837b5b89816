"""Class conditioning's host layers on the CPU: config validation and class-name resolution, the per-class dataset,
class-dependent synthetic grids, label dropout and the modes that refuse a class-conditional network."""
import math

import pytest
import torch

from helpers import tiny_config


def _cfg(K=3, **data):
    cfg = tiny_config("res64")
    cfg.device = torch.device("cpu")
    cfg.model.num_classes = K
    for k, v in data.items():
        cfg.data[k] = v
    return cfg


def test_validation_and_name_resolution():
    from meshdiffusion_b200.diffusion import classes
    cfg = _cfg(3, class_names=("chair", "car", "table"))
    assert classes.validate(cfg) == 3
    assert classes.resolve_class_label(cfg) is None and classes.sampling_kwargs(cfg) == {}
    for label, k in (("car", 1), (2, 2), ("0", 0)):
        cfg.eval.class_label = label
        assert classes.resolve_class_label(cfg) == k
        assert classes.sampling_kwargs(cfg) == {"class_labels": k}
    for label, msg in (("sofa", "not in data.class_names"), (3, "outside 0..2"), (-1, "outside 0..2")):
        cfg.eval.class_label = label
        with pytest.raises(ValueError, match=msg):
            classes.resolve_class_label(cfg)
    with pytest.raises(ValueError, match="lists 2 entries for model.num_classes = 3"):
        classes.validate(_cfg(3, class_meta_paths=("a.json", "b.json")))
    with pytest.raises(ValueError, match="duplicates"):
        classes.validate(_cfg(2, class_names=("a", "a")))
    with pytest.raises(ValueError, match="model.num_classes is 0"):
        classes.validate(_cfg(0, class_names=("a",)))
    cfg = _cfg(0)
    cfg.sampling.guidance_scale = 3.0
    with pytest.raises(ValueError, match="needs a class-conditional network"):
        classes.validate(cfg)
    cfg = _cfg(2)
    cfg.sampling.guidance_scale = 3.0
    with pytest.raises(ValueError, match="needs eval.class_label"):
        classes.resolve_class_label(cfg)
    cfg.training.class_dropout = 1.5
    with pytest.raises(ValueError, match="class_dropout"):
        classes.validate(cfg)


def test_concatenated_dataset_yields_class_per_item():
    from meshdiffusion_b200.diffusion import classes
    ds = classes.class_dataset([[torch.full((1,), float(i)) for i in range(n)] for n in (3, 1, 2)])
    items = [ds[i] for i in range(len(ds))]
    assert [k for _, k in items] == [0, 0, 0, 1, 2, 2]
    assert [float(g) for g, _ in items] == [0, 1, 2, 0, 0, 1]
    loader = torch.utils.data.DataLoader(ds, batch_size=6, shuffle=False)
    grids, ks = next(iter(loader))
    assert ks.tolist() == [0, 0, 0, 1, 2, 2] and grids.shape == (6, 1)


def test_label_dropout_rate_within_binomial_bounds():
    from meshdiffusion_b200.diffusion import classes
    K, p, n = 5, 0.1, 200000
    y = torch.randint(0, K, (n,), generator=torch.Generator().manual_seed(0))
    d = classes.drop_labels(y, K, p, torch.Generator().manual_seed(1))
    dropped = (d == K).sum().item()
    assert abs(dropped - n * p) < 5 * math.sqrt(n * p * (1 - p))
    assert torch.equal(d[d != K], y[d != K])
    assert torch.equal(classes.drop_labels(y, K, 0.0), y)
    assert (classes.drop_labels(y, K, 1.0, torch.Generator().manual_seed(2)) == K).all()


def test_synthetic_grids_depend_on_the_class():
    from meshdiffusion_b200.diffusion import classes
    g = torch.Generator().manual_seed(0)
    x = classes.synthetic_class_grids(torch.tensor([0, 1, 0]), 64, "cpu", g)
    inside = (x[:, 0] > 0).sum(dim=(1, 2, 3))
    assert inside[1] > inside[0] and inside[0] == inside[2]  # the class sets the sphere's radius


@pytest.mark.parametrize("mode", ["eval_completion", "edit", "uncond_gen_interp", "distill", "eval_likelihood"])
def test_unconditional_modes_refuse_a_conditional_network(mode, tmp_path):
    import importlib
    mod, fn = {"eval_completion": ("completion", "eval_completion"), "edit": ("edit", "edit"),
               "uncond_gen_interp": ("interp", "uncond_gen_interp"), "distill": ("distill", "distill"),
               "eval_likelihood": ("eval_likelihood", "eval_likelihood")}[mode]
    cfg = _cfg(2)
    cfg.eval.eval_dir = str(tmp_path)
    with pytest.raises(ValueError, match=f"--mode={mode} does not support class-conditional"):
        getattr(importlib.import_module(f"meshdiffusion_b200.diffusion.{mod}"), fn)(cfg)


def test_pc_and_ddim_configs_refuse_guidance():
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    sde = sde_lib.VPSDE(0.1, 20.0, 1000, device="cpu")
    for method in ("pc", "ddim"):
        cfg = _cfg(2)
        cfg.sampling.method = method
        cfg.sampling.guidance_scale = 3.0
        fn = sampling.get_sampling_fn(cfg, sde, (1, 4, 4, 4, 4), lambda v: v, 1e-3, grid_mask=torch.ones(1, 1, 4, 4, 4))
        with pytest.raises(ValueError, match="guidance_scale = 1"):
            fn(lambda x, t, class_labels=None: x, class_labels=torch.tensor([0]))
