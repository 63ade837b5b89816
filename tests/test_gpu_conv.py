"""Parity of the wgmma implicit-GEMM convolution against torch's fp32 conv3d (TF32 disabled) on the same inputs.

Tolerances (max |diff| / max |ref|): tf32 operands 2e-3, bf16 operands 2e-2 -- operand rounding only, the
accumulation is fp32 in registers in both modes; split bf16 ("bf16x3": hi*hi + hi*lo + lo*hi, the dropped lo*lo term is
2^-16 of a product; the 5^3 head case sums 16 000 products per output) 1e-4.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {"tf32": 2e-3, "bf16": 2e-2, "bf16x3": 1e-4}


def _ref_setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


CASES = [
    # (B, Cin, Cout, R, k, stride)
    (2, 128, 128, 16, 3, 1),   # (8,16,1,1) tile, y-halo reuse
    (1, 256, 128, 16, 3, 1),
    (2, 128, 256, 8, 3, 1),    # (8,8,2,1) tile
    (3, 512, 512, 4, 3, 1),    # (4,4,4,2) tile spanning samples, odd batch
    (2, 128, 128, 16, 3, 2),   # Downsample
    (2, 256, 256, 8, 3, 2),
    (2, 384, 128, 16, 1, 1),   # NIN-shaped
    (1, 128, 4, 16, 3, 1),     # head (N=4 -> BLOCK_N 32, scalar stores)
    (1, 128, 4, 32, 5, 1),     # res128 head, 5-tap reuse
    (1, 128, 128, 32, 3, 1),
    (3, 128, 128, 32, 3, 1),   # 768 M-tiles: CTA pairs with two M-tiles per CTA sharing the weight tiles (bf16 / tf32), odd batch
    (2, 256, 128, 32, 3, 1),
]


@pytest.mark.parametrize("precision", ["tf32", "bf16", "bf16x3"])
@pytest.mark.parametrize("case", CASES)
def test_conv3d_matches_torch(case, precision):
    from meshdiffusion_b200 import ops
    _ref_setup()
    B, Cin, Cout, R, k, stride = case
    g = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.randn(B, Cin, R, R, R, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, k, device="cuda", generator=g) / (Cin * k ** 3) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    if stride == 1:
        ref = F.conv3d(x, w, b, padding=k // 2)
    else:
        ref = F.conv3d(F.pad(x, (0, 1, 0, 1, 0, 1)), w, b, stride=2, padding=0)
    xin = ops.to_ndhwc(x, precision)
    y, stats = ops.conv3d(xin, w, b, stride=stride, want_stats=True, precision=precision)
    out = ops.from_ndhwc(y, precision)
    assert out.shape == ref.shape
    err = _rel(out, ref)
    print(f"conv {case} {precision}: rel err {err:.3e}")
    assert err < TOL[precision]
    # fused GroupNorm statistics: per-(sample, channel) sum and sum of squares of the fp32 result
    s_ref = ref.double().sum(dim=(2, 3, 4))
    q_ref = (ref.double() ** 2).sum(dim=(2, 3, 4))
    assert _rel(stats[..., 0], s_ref) < TOL[precision]
    assert _rel(stats[..., 1], q_ref) < TOL[precision]


@pytest.mark.parametrize("precision", ["tf32", "bf16", "bf16x3"])
def test_conv3d_epilogue_terms(precision):
    """bias + per-sample (time-embedding) bias + residual, as in ResnetBlockDDPM (layers.py:677-689)."""
    from meshdiffusion_b200 import ops
    _ref_setup()
    B, C, R = 2, 128, 16
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(B, C, R, R, R, device="cuda", generator=g)
    w = torch.randn(C, C, 3, 3, 3, device="cuda", generator=g) / (C * 27) ** 0.5
    b = torch.randn(C, device="cuda", generator=g)
    rb = torch.randn(B, C, device="cuda", generator=g)
    res = torch.randn(B, C, R, R, R, device="cuda", generator=g)
    ref = F.conv3d(x, w, b, padding=1) + rb[:, :, None, None, None] + res
    y = ops.conv3d(ops.to_ndhwc(x, precision), w, b, rowbias=rb, residual=ops.to_ndhwc(res, precision), precision=precision)
    err = _rel(ops.from_ndhwc(y, precision), ref)
    print(f"epilogue {precision}: rel err {err:.3e}")
    assert err < TOL[precision]


@pytest.mark.parametrize("precision", ["tf32", "bf16", "bf16x3"])
def test_groupnorm_silu(precision):
    from meshdiffusion_b200 import ops
    B, C, R = 2, 256, 8
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, C, R, R, R, device="cuda", generator=g) * 2 + 0.5
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.1
    xin = ops.to_ndhwc(x, precision)
    xr = ops.from_ndhwc(xin, precision)  # what the kernel actually sees
    stats = torch.stack([xr.double().sum(dim=(2, 3, 4)), (xr.double() ** 2).sum(dim=(2, 3, 4))], dim=-1).contiguous()
    ref = F.silu(F.group_norm(xr, 32, gamma, beta, eps=1e-6))
    y = ops.from_ndhwc(ops.groupnorm_act(xin, stats, gamma, beta, silu=True, precision=precision), precision)
    err = _rel(y, ref)
    print(f"gn+silu {precision}: rel err {err:.3e}")
    assert err < {"tf32": 2e-3, "bf16": 1e-2, "bf16x3": 2e-5}[precision]


def test_groupnorm_statistics_survive_large_activations():
    """Pre-normalisation activations of a few thousand (reached after a handful of optimiser steps in the full-size
    training test, and possible in any trained checkpoint) push sum(x^2) over a 32^3 grid past 5.5e11, where a single
    2^-24 fixed-point int64 wraps: the split (lo, hi) record must keep the statistics exact and GroupNorm correct."""
    from meshdiffusion_b200 import ops
    _ref_setup()
    B, C, R = 2, 64, 32
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.randn(B, C, R, R, R, device="cuda", generator=g) * 6000.0 + 2500.0)
    w = torch.randn(C, C, 3, 3, 3, device="cuda", generator=g) / (C * 27) ** 0.5
    xin = ops.to_ndhwc(x, "bf16")
    xr, wr = ops.from_ndhwc(xin), w.bfloat16().float()
    ref = F.conv3d(xr, wr, None, padding=1)
    y, stats = ops.conv3d(xin, w, None, want_stats=True, precision="bf16")
    ref_stats = torch.stack([ref.double().sum(dim=(2, 3, 4)), (ref.double() ** 2).sum(dim=(2, 3, 4))], dim=-1)
    assert ref_stats[..., 1].max().item() > 5.5e11, "the case must exceed the single-word range"
    es = ((stats - ref_stats).abs() / ref_stats.abs().clamp_min(1.0)).max().item()
    print(f"large-activation statistics: max sumsq {ref_stats[..., 1].max().item():.3e}, rel err {es:.3e}")
    assert es < 1e-3
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g) * 0.1
    out = ops.from_ndhwc(ops.groupnorm_act(y, stats, gamma, beta, silu=True, precision="bf16"))
    want = F.silu(F.group_norm(ops.from_ndhwc(y), 32, gamma, beta, eps=1e-6))
    assert _rel(out, want) < 2e-2
