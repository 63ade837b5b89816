"""Score-network parity: the sm_90a engine vs (a) the committed golden vectors produced by the REFERENCE modules on
CPU fp32 (oracle/make_golden.py), (b) the oracle evaluated on the GPU in true fp32 at the full res64 size.

Tolerances are on max|diff|/max|ref| and relative L2. Split bf16 operands ("bf16x3", the parity-grade mode): 1e-3, the
tolerance BASELINE.json's north_star states. tf32 operands: 3e-3 (the reference's own stock GPU path runs
its convolutions in TF32 as well, torch.backends.cudnn.allow_tf32 defaults to True; its error against fp32 is measured
and printed next to ours in test_res64_full_vs_oracle). bf16 operands: 4e-2.
"""
import pytest
import torch

from helpers import build_model, engine_report, full_config, load_golden, rel_l2, rel_max, tiny_config
from oracle import synth, unet_oracle

pytestmark = pytest.mark.gpu

TOL_MAX = {"bf16x3": 1e-3, "tf32": 3e-3, "bf16": 4e-2}
TOL_L2 = {"bf16x3": 1e-3, "tf32": 2.5e-3, "bf16": 3e-2}


@pytest.mark.parametrize("precision", ["bf16x3", "tf32", "bf16"])
@pytest.mark.parametrize("name", ["res64", "res128"])
def test_tiny_matches_reference_golden(name, precision):
    gold = load_golden(f"unet_tiny_{name}.npz")
    cfg = tiny_config(name, precision)
    model, sd = build_model(cfg, "cuda:0", int(gold["state_seed"]))
    assert abs(synth.state_checksum(sd) - gold["checksum"]).max() < 1e-6, "synthetic weights drifted from the golden run"
    x, labels = synth.synthetic_inputs(cfg.data.image_size, 2, int(gold["input_seed"]), sd["mask"])
    out = model(x.cuda(), labels.cuda()).cpu()
    ref = torch.from_numpy(gold["out"])
    em, el = rel_max(out, ref), rel_l2(out, ref)
    print(f"tiny {name} {precision}: max {em:.3e}  l2 {el:.3e}")
    assert em < TOL_MAX[precision] and el < TOL_L2[precision]


@pytest.mark.parametrize("batch", [1, 3])
def test_batch_invariance(batch):
    """Every sample of a batch gets the result it would get alone (tiles spanning samples, stats per sample)."""
    cfg = tiny_config("res64", "tf32")
    model, sd = build_model(cfg, "cuda:0", 11)
    x, labels = synth.synthetic_inputs(16, 3, 99, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    full = model(x, labels)
    part = model(x[:batch].contiguous(), labels[:batch].contiguous())
    assert torch.equal(full[:batch], part)


@pytest.mark.parametrize("precision", ["bf16x3", "tf32", "bf16"])
def test_res64_full_vs_oracle(precision):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = full_config("res64", precision)
    model, sd = build_model(cfg, "cuda:0", 5)
    x, labels = synth.synthetic_inputs(64, 1, 6, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    out = model(x, labels)
    sdg = {k: v.cuda() for k, v in sd.items()}
    arch = unet_oracle.arch_from_config(cfg)
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sdg, arch, x, labels)
        torch.backends.cudnn.allow_tf32 = True   # the reference's stock GPU setting, for calibration only
        torch.backends.cuda.matmul.allow_tf32 = True
        stock = unet_oracle.unet_forward(sdg, arch, x, labels)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    em, el = rel_max(out, ref), rel_l2(out, ref)
    print(f"res64 full {precision}: ours max {em:.3e} l2 {el:.3e} | stock torch TF32 path max {rel_max(stock, ref):.3e} l2 {rel_l2(stock, ref):.3e}")
    assert em < TOL_MAX[precision] and el < TOL_L2[precision]


@pytest.mark.parametrize("precision", ["bf16x3", "tf32", "bf16"])
def test_res128_full_vs_oracle(precision):
    """ddpm_res128 at its real size (ddpm_res128.py:137-215: 6 levels, 5^3 stem / head, 388 M parameters, 34.5 TFLOP per
    evaluation) against the oracle in true fp32 on the GPU, B=1."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = full_config("res128", precision)
    model, sd = build_model(cfg, "cuda:0", 5)
    x, labels = synth.synthetic_inputs(128, 1, 6, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    out = model(x, labels)
    model.module.release_engine()
    sdg = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        ref = unet_oracle.unet_forward(sdg, unet_oracle.arch_from_config(cfg), x, labels)
    em, el = rel_max(out, ref), rel_l2(out, ref)
    print(f"res128 full {precision}: max {em:.3e} l2 {el:.3e}")
    assert torch.isfinite(out).all()
    assert em < TOL_MAX[precision] and el < TOL_L2[precision]


def test_state_dict_roundtrip_and_mask_update():
    """`score_model.module.mask.data[:] = mask` (trainer.py:61-63) must reach the engine."""
    cfg = tiny_config("res64", "tf32")
    model, sd = build_model(cfg, "cuda:0", 11)
    x, labels = synth.synthetic_inputs(16, 1, 3, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    a = model(x, labels)
    model.module.mask.data[:] = 1.0 - model.module.mask.data
    b = model(x, labels)
    assert not torch.equal(a, b)
    model.module.mask.data[:] = sd["mask"].cuda()
    assert torch.equal(model(x, labels), a)


def test_full_size_determinism_and_batch_invariance():
    """BASELINE-size network (res64, batch 8 of the engine): two evaluations are bitwise identical (integer-atomic
    GroupNorm statistics, fixed-order reductions), and a sample's result does not depend on its batch-mates."""
    cfg = full_config("res64", "bf16")
    cfg.model.engine_max_batch = 8
    model, sd = build_model(cfg, "cuda:0", 5)
    x, labels = synth.synthetic_inputs(64, 8, 7, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    a = model(x, labels)
    b = model(x, labels)
    assert torch.equal(a, b), "forward pass is not bitwise reproducible"
    c = model(x[:3].contiguous(), labels[:3].contiguous())
    assert torch.equal(a[:3], c), "a sample's output depends on the rest of the batch"
    assert torch.isfinite(a).all()


@pytest.mark.parametrize("precision,training", [("bf16", False), ("tf32", False), ("bf16x3", False), ("bf16", True),
                                                ("bf16x3", True)])
def test_dry_plan_matches_engine(precision, training):
    """The dry plan and the engine are built by the same code: they report the same launches, GEMM accounting, FLOPs,
    arena, backward plan and gradient readiness."""
    cfg = tiny_config("res64", precision)
    dry = engine_report(cfg, 2, precision, training, dry=True)
    assert dry["n_gemm"] > 0
    assert engine_report(cfg, 2, precision, training, dry=False) == dry
