"""CPU: checkpoints interchange with the REFERENCE's own code in both directions (the drop-in contract of SURVEY 8b:
`torch.save({'optimizer','model','ema','step'})` with `module.`-prefixed model keys, positional EMA shadow list, the stock
Adam state).

What the reference did is stored under tests/golden/: `checkpoint_reference.pth.xz` is a checkpoint written by its own
`save_checkpoint` (one Adam step on seeded gradients + two EMA updates) for a one-level network whose weights and gradients
are drawn from small sets of values (multiples of 1/8 and of 1e-2), so that the file compresses into a fixture; and `checkpoint_reference_restored.json` records what
its `restore_checkpoint` (into its `DDPMRes64` inside `nn.DataParallel`, `ExponentialMovingAverage`, `losses.get_optimizer`)
read back from the seeded checkpoint this test writes -- keys, dtypes, shapes and a sha256 of every tensor. Both were produced
by REF_SIDE below, run on the unmodified reference modules in a subprocess (nothing of this package is imported there);
`python tests/test_checkpoint_interchange.py` regenerates them where the reference is staged under baseline/_ref."""
import hashlib
import json
import lzma
import os
import shutil
import subprocess
import sys
import tempfile

import torch

from helpers import ROOT, tiny_config

GOLD_CKPT = os.path.join(ROOT, "tests", "golden", "checkpoint_reference.pth.xz")
GOLD_RESTORED = os.path.join(ROOT, "tests", "golden", "checkpoint_reference_restored.json")

REF_SIDE = r"""
import hashlib, json, os, sys, torch
root, ours_ckpt, ref_ckpt, restored_json = sys.argv[1:5]
sys.path.insert(0, root)
from baseline import reference_arm
ref, config = reference_arm.load("cpu")
import lib.diffusion.utils as rutils, lib.diffusion.losses as rlosses
from lib.diffusion.models.ema import ExponentialMovingAverage
config.data.image_size, config.model.nf, config.model.ch_mult = 16, 32, (1, 2)
config.model.num_res_blocks, config.model.attn_resolutions = 1, (8,)

def digest(t):
    t = t.detach().cpu().contiguous()
    return [str(t.dtype), list(t.shape), hashlib.sha256(t.numpy().tobytes()).hexdigest()]

def fresh(seed):
    torch.manual_seed(seed)
    model = ref["mutils"].create_model(config)            # models/utils.py:88-96 -> nn.DataParallel shell, `module.` keys
    ema = ExponentialMovingAverage(model.parameters(), decay=config.model.ema_rate)
    opt = rlosses.get_optimizer(config, model.parameters())
    return dict(optimizer=opt, model=model, ema=ema, step=0)

# (1) the checkpoint written by meshdiffusion_b200 restores through the reference's restore_checkpoint
state = rutils.restore_checkpoint(ours_ckpt, fresh(1), "cpu")
ost = state["optimizer"].state_dict()
rec = {"step": int(state["step"]), "model": {k: digest(v) for k, v in state["model"].state_dict().items()},
       "ema_num_updates": int(state["ema"].num_updates), "ema_decay": float(state["ema"].decay),
       "ema_shadow": [digest(t) for t in state["ema"].shadow_params],
       "opt_state": {str(i): {"step": float(s["step"]), "exp_avg": digest(s["exp_avg"]), "exp_avg_sq": digest(s["exp_avg_sq"])}
                     for i, s in ost["state"].items()}}
# the restored reference optimiser keeps stepping (its state is the stock Adam layout)
for p in state["model"].parameters():
    p.grad = torch.zeros_like(p)
state["optimizer"].step()
json.dump(rec, open(restored_json, "w"), indent=0, sort_keys=True)

# (2) a checkpoint written by the reference: one Adam step on seeded gradients + two EMA updates, its own save_checkpoint.
# A one-level network with weights and gradients from small value sets keeps the compressed file small.
config.data.image_size, config.model.ch_mult, config.model.num_res_blocks, config.model.attn_resolutions = 8, (1,), 0, ()
st = fresh(2)
g = torch.Generator().manual_seed(3)
with torch.no_grad():
    for p in st["model"].parameters():
        p.copy_(torch.randint(-8, 9, p.shape, generator=g) / 8.0)
st["ema"] = ExponentialMovingAverage(st["model"].parameters(), decay=config.model.ema_rate)
for p in st["model"].parameters():
    p.grad = torch.randint(-2, 3, p.shape, generator=g) * 1e-2
st["optimizer"].step()
st["ema"].update(st["model"].parameters())
st["ema"].update(st["model"].parameters())
st["step"] = 11
rutils.save_checkpoint(ref_ckpt, st)
print("REF_DONE")
"""


def _config(small=False):
    cfg = tiny_config()
    if small:  # the reference checkpoint's network
        cfg.data.image_size, cfg.model.ch_mult, cfg.model.num_res_blocks, cfg.model.attn_resolutions = 8, (1,), 0, ()
    cfg.device = torch.device("cpu")
    return cfg


def _fresh(cfg, seed):
    from meshdiffusion_b200.diffusion import losses
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from meshdiffusion_b200.diffusion.models.ema import ExponentialMovingAverage
    torch.manual_seed(seed)
    model = mutils.create_model(cfg)
    return dict(optimizer=losses.get_optimizer(cfg, model.parameters()), model=model,
                ema=ExponentialMovingAverage(model.parameters(), decay=cfg.model.ema_rate), step=0)


def _write_ours(path):
    """A seeded checkpoint through this package's save_checkpoint; returns the state it holds. The fused optimiser step
    needs the GPU, so its (stock Adam) state is filled in by hand."""
    from meshdiffusion_b200.diffusion.utils import save_checkpoint
    st = _fresh(_config(), 5)
    g = torch.Generator().manual_seed(6)
    with torch.no_grad():
        for p in st["model"].parameters():
            p.add_(torch.randn(p.shape, generator=g) * 1e-2)
    opt = st["optimizer"]
    for p in st["model"].parameters():
        if p.requires_grad:
            opt.state[p] = {"step": torch.tensor(3.0), "exp_avg": torch.randn(p.shape, generator=g),
                            "exp_avg_sq": torch.rand(p.shape, generator=g)}
    st["ema"].update(st["model"].parameters())
    st["step"] = 7
    save_checkpoint(path, st)
    return st


def _digest(t):
    t = t.detach().cpu().contiguous()
    return [str(t.dtype), list(t.shape), hashlib.sha256(t.numpy().tobytes()).hexdigest()]


def regenerate():
    with tempfile.TemporaryDirectory() as d:
        ours = os.path.join(d, "ours.pth")
        _write_ours(ours)
        r = subprocess.run([sys.executable, "-c", REF_SIDE, ROOT, ours, os.path.join(d, "ref.pth"), os.path.join(d, "restored.json")],
                           capture_output=True, text=True, env=dict(os.environ, OMP_NUM_THREADS="4"), timeout=600)
        assert r.returncode == 0 and "REF_DONE" in r.stdout, r.stdout + r.stderr
        with open(os.path.join(d, "ref.pth"), "rb") as f, lzma.open(GOLD_CKPT, "wb", preset=9 | lzma.PRESET_EXTREME) as g:
            shutil.copyfileobj(f, g)
        shutil.copyfile(os.path.join(d, "restored.json"), GOLD_RESTORED)


def test_checkpoints_interchange_with_the_reference_code(tmp_path):
    _check_ours_restored_by_the_reference(tmp_path)
    _check_reference_checkpoint_restores_here(tmp_path)


def _check_ours_restored_by_the_reference(tmp_path):
    """What the reference's restore_checkpoint read from this package's checkpoint is, tensor for tensor, what was saved."""
    st = _write_ours(str(tmp_path / "ours.pth"))
    with open(GOLD_RESTORED) as f:
        rec = json.load(f)
    assert rec["step"] == 7
    sd = st["model"].state_dict()
    assert set(rec["model"]) == set(sd), set(rec["model"]) ^ set(sd)
    for k, v in sd.items():
        assert rec["model"][k] == _digest(v), k
    assert rec["ema_num_updates"] == st["ema"].num_updates and rec["ema_decay"] == st["ema"].decay
    assert rec["ema_shadow"] == [_digest(t) for t in st["ema"].shadow_params]
    ost = st["optimizer"].state_dict()["state"]
    assert set(rec["opt_state"]) == {str(i) for i in ost}
    for i, s in ost.items():
        r = rec["opt_state"][str(i)]
        assert r["exp_avg"] == _digest(s["exp_avg"]) and r["exp_avg_sq"] == _digest(s["exp_avg_sq"]), i
        assert r["step"] == float(s["step"])


def _check_reference_checkpoint_restores_here(tmp_path):
    """A checkpoint written by the reference's save_checkpoint restores through this package's restore_checkpoint into
    the model, EMA and Adam state it holds, tensor for tensor."""
    from meshdiffusion_b200.diffusion.utils import restore_checkpoint
    path = str(tmp_path / "reference.pth")
    with lzma.open(GOLD_CKPT, "rb") as f, open(path, "wb") as g:
        shutil.copyfileobj(f, g)
    raw = torch.load(path, map_location="cpu", weights_only=False)
    st2 = restore_checkpoint(path, _fresh(_config(small=True), 8), "cpu")
    assert st2["step"] == 11
    sd = st2["model"].state_dict()
    assert set(sd) == set(raw["model"])
    for k, v in raw["model"].items():
        assert sd[k].dtype == v.dtype and torch.equal(sd[k], v), k
    assert st2["ema"].num_updates == raw["ema"]["num_updates"] == 2
    for a, b in zip(st2["ema"].shadow_params, raw["ema"]["shadow_params"], strict=True):
        assert torch.equal(a, b)
    ost = st2["optimizer"].state_dict()
    assert set(ost["state"]) == set(raw["optimizer"]["state"])
    for i, s in raw["optimizer"]["state"].items():
        for f in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(ost["state"][i][f], s[f]), (i, f)
        assert float(ost["state"][i]["step"]) == float(s["step"]) == 1.0
    for ga, gb in zip(ost["param_groups"], raw["optimizer"]["param_groups"], strict=True):
        for key in ("lr", "betas", "eps", "weight_decay"):
            assert ga[key] == gb[key], key
        assert ga["params"] == gb["params"]


if __name__ == "__main__":
    regenerate()
