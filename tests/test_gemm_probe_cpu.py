"""CPU: the GEMM probe cases of test_gpu_gemm_variants.py are the engine's own launches, and their gates can fail.

1. Every GPU case that mirrors a score-network launch is described to mdb_gemm_probe (or to the engine's composites,
   mdb_upsample_conv and mdb_attention_core) with dry = 1; its tile report (work items, split-K factor, k-steps, most
   k-steps per entry, BLOCK_N), FLOPs and fill bytes must equal those of the launch with that name in a GPU-less plan of
   the full res64 or the tiny network at the case's batch and precision. Without this the GPU tests could pass on a
   variant the engine never builds.
2. For every family, a plausible wrong answer misses its gate by at least 5x, so no gate is too loose to catch the bug it
   is there for.
"""
import pytest
import torch
import torch.nn.functional as F

import gemm_variants as gv
from helpers import full_config, tiny_config

_ENGINE = {}


def _engine(which, batch, precision):
    key = (which, batch, precision)
    if key not in _ENGINE:
        cfg = (full_config if which == "full" else tiny_config)("res64", precision)
        _ENGINE[key] = gv.engine_tiles(cfg, batch, precision)
    return _ENGINE[key]


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", [c for c in gv.SPLIT_CASES if "mirror" in c], ids=lambda c: c["id"])
def test_split_cases_are_engine_launches(case, precision):
    which, name = case["mirror"]
    eng = _engine(which, case["B"], precision)[name]
    assert gv.probe(gv.split_desc(case, precision, -1)) == eng, name


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", [c for c in gv.NIN_CASES if "mirror" in c], ids=lambda c: c["id"])
def test_nin_shortcut_cases_are_engine_launches(case, precision):
    which, name = case["mirror"]
    eng = _engine(which, case["B"], precision)[name]
    assert gv.probe(gv.nin_desc(case, precision)) == eng, name


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", [c for c in gv.ATTN_CASES if "mirror" in c], ids=lambda c: c["id"])
def test_attention_cases_are_engine_launches(case, precision):
    which, pre = case["mirror"]
    eng = _engine(which, case["B"], precision)
    V, C, B = case["V"], case["C"], case["B"]
    R = round(V ** (1 / 3))
    assert R ** 3 == V
    qk, pv = gv.attention_reports(V, C, B, precision)
    assert qk == eng[pre + ".qk"] and pv == eng[pre + ".pv"]
    for i in range(3):
        assert gv.probe(gv.nin_slot_desc(R, C, B, i, precision)) == eng[f"{pre}.nin{i}"], i


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.UP_MIRRORS, ids=lambda c: c["mirror"][1])
def test_upsample_cases_are_engine_launches(case, precision):
    which, pre = case["mirror"]
    eng = _engine(which, case["B"], precision)
    r, C, B = case["r"], case["C"], case["B"]
    reps = gv.upsample_reports(r, C, B, precision)
    for par in range(8):
        assert reps[par] == eng[f"{pre}.conv.p{par}"], par
        # the probe's own add_conv_up2 operand describes the same launch
        assert gv.probe(gv.upsample_probe_desc(r, C, B, par, precision)) == reps[par], par


def test_upsample_cases_cover_the_reuse_tiles():
    """The GPU upsample cases reach the multi-sample tile (r = 4), the plain tile (r = 8) and the y-halo-reuse tile (r = 16):
    the reuse entries take two k-steps each."""
    for r, nk in ((4, 1), (8, 1), (16, 2)):
        assert gv.upsample_reports(r, 128, 1, "bf16")[0][3] == nk, r


def test_split_cases_split():
    """Every split-K case splits under the engine's plan in every precision (else it would not test the reduction)."""
    for case in gv.SPLIT_CASES:
        for precision in gv.PRECISIONS:
            if case["id"].startswith("tiny"):
                continue
            assert gv.probe(gv.split_desc(case, precision, -1))[1] > 1, (case["id"], precision)


def test_forced_splits_clamp_to_the_groups():
    case = gv.SPLIT_CASES[0]
    groups = gv.probe(gv.split_desc(case, "bf16", 10 ** 6))[1]
    assert groups == 27 * 4  # one k-step per tap and 64-channel block: 108 groups
    assert gv.probe(gv.split_desc(case, "bf16", 7))[1] == 7


# ------------------------------------------------------------------------------ the gates can fail
def _conv_ref(x, w, pad=1):
    return F.conv3d(x.double(), w.double(), padding=pad)


def _gen(seed=0):
    return torch.Generator().manual_seed(seed)


def test_gate_split_catches_a_dropped_split_range():
    """Dropping one of 7 split ranges of a 108-group 3^3 convolution (64-channel blocks x taps)."""
    g = _gen(1)
    x = torch.randn(1, 128, 6, 6, 6, generator=g, dtype=torch.float64)
    w = torch.randn(64, 128, 3, 3, 3, generator=g, dtype=torch.float64)
    ref = _conv_ref(x, w)
    # groups in table order: channel block outer, taps inner; range 3 of 7 over the 54 groups
    groups = [(c, t) for c in range(2) for t in range(27)]
    lo, hi = 3 * len(groups) // 7, 4 * len(groups) // 7
    wd = w.clone().reshape(64, 2, 64, 27)
    for c, t in groups[lo:hi]:
        wd[:, c, :, t] = 0
    bad = _conv_ref(x, wd.reshape(64, 128, 3, 3, 3))
    for precision in gv.PRECISIONS:
        assert gv.rel_err(bad, ref) > 5 * gv.GATES["split"][precision]


def test_gate_upsample_catches_swapped_parity_classes():
    g = _gen(2)
    x = torch.randn(1, 16, 4, 4, 4, generator=g, dtype=torch.float64)
    w = torch.randn(16, 16, 3, 3, 3, generator=g, dtype=torch.float64)
    ref = _conv_ref(F.interpolate(x, scale_factor=2, mode="nearest"), w)
    bad = ref.clone()
    bad[..., 0::2] = ref[..., 1::2]  # parity px = 0 and 1 exchanged
    bad[..., 1::2] = ref[..., 0::2]
    for precision in gv.PRECISIONS:
        assert gv.rel_err(bad, ref) > 5 * gv.GATES["upsample"][precision]
    # the fp64 fold is the sub-pixel identity the engine relies on
    f = gv.fold_upconv(w)
    R = 8
    sub = torch.zeros_like(ref)
    for par in range(8):
        px, py, pz = par & 1, (par >> 1) & 1, par >> 2
        # output 2h + p reads input h - 1 + p + e for e in {0, 1}
        xp = F.pad(x, (1, 1, 1, 1, 1, 1))[..., pz:pz + 5, py:py + 5, px:px + 5]
        sub[..., pz::2, py::2, px::2] = F.conv3d(xp, f[par])[..., :R // 2, :R // 2, :R // 2]
    assert gv.rel_err(sub, ref) < 1e-12


def test_gate_attention_catches_missing_alpha_and_swapped_slots():
    g = _gen(3)
    V, C = 64, 64
    q, k, v = (torch.randn(V, C, generator=g, dtype=torch.float64) for _ in range(3))
    ref = q @ k.T / C ** 0.5
    for precision in gv.PRECISIONS:
        assert gv.rel_err(q @ k.T, ref) > 5 * gv.GATES["attn"][precision]      # alpha omitted
        assert gv.rel_err(k @ q.T / C ** 0.5, ref) > 5 * gv.GATES["attn"][precision]  # q and k slots swapped
    o = torch.softmax(ref, -1) @ v
    bad = torch.softmax(k @ q.T / C ** 0.5, -1) @ v
    for precision in gv.PRECISIONS:
        assert gv.rel_err(bad, o) > 5 * gv.GATES["attn"][precision]


def test_gate_split_bf16_catches_a_dropped_lo_hi_term():
    """Split bf16 without the lo(A) hi(W) product."""
    g = _gen(4)
    a = torch.randn(256, 512, generator=g)
    w = torch.randn(512, 128, generator=g)
    ah, wh = a.to(torch.bfloat16).double(), w.to(torch.bfloat16).double()
    al, wl = (a - ah.float()).to(torch.bfloat16).double(), (w - wh.float()).to(torch.bfloat16).double()
    ref = (ah + al) @ (wh + wl)
    bad = ah @ wh + ah @ wl
    for fam in gv.GATES:
        assert gv.rel_err(bad, ref) > 5 * gv.GATES[fam]["bf16x3"]


def test_gate_nin_catches_a_dropped_second_source():
    g = _gen(5)
    C0, C1, N = 64, 32, 32
    a2 = torch.randn(1, N, 6, 6, 6, generator=g, dtype=torch.float64)
    h = torch.randn(1, C0, 6, 6, 6, generator=g, dtype=torch.float64)
    skip = torch.randn(1, C1, 6, 6, 6, generator=g, dtype=torch.float64)
    w1 = torch.randn(N, N, 3, 3, 3, generator=g, dtype=torch.float64) / (27 * N) ** 0.5
    wn = torch.randn(C0 + C1, N, generator=g, dtype=torch.float64) / (C0 + C1) ** 0.5
    ref = _conv_ref(a2, w1) + torch.einsum("bcxyz,cn->bnxyz", torch.cat([h, skip], 1), wn)
    bad = _conv_ref(a2, w1) + torch.einsum("bcxyz,cn->bnxyz", h, wn[:C0])
    for precision in gv.PRECISIONS:
        assert gv.rel_err(bad, ref) > 5 * gv.GATES["nin"][precision]


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", [c for c in gv.ATTN_CASES if "mirror" in c], ids=lambda c: c["id"])
def test_probe_logits_are_the_engine_launch(case, precision):
    """The probe's activation-B description of the logits (test_logits_through_the_probe) is attn*.qk."""
    which, pre = case["mirror"]
    eng = _engine(which, case["B"], precision)
    assert gv.probe(gv.logits_desc(case["V"], case["C"], case["B"], precision)) == eng[pre + ".qk"]


def test_groupnorm_backward_probe_refuses_what_the_epilogue_is_not_built_for():
    """tf32 operands and split-K: the engine never fuses these (the dgrad then runs unfused), and the probe says so."""
    from meshdiffusion_b200 import _native
    case = gv.GNB_CASES[1]
    gv.probe(gv.gnb_desc(case, "bf16", 1, 2))
    with pytest.raises(_native.NativeError, match="bf16"):
        gv.probe(gv.gnb_desc(case, "tf32", 1, 2))
    d = gv.gnb_desc(case, "bf16", 1, 2)
    d.splits = 2
    with pytest.raises(_native.NativeError, match="split-K"):
        gv.probe(d)


def _gn_backward(x, gamma, beta, da, mask, silu=True):
    """fp64 dL/dx, dgamma, dbeta of dropout(act(GroupNorm(32)(x))) with the dropout mask (already scaled) `mask`."""
    x = x.clone().requires_grad_(True)
    gamma, beta = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    a = F.group_norm(x, 32, gamma, beta, eps=1e-6)
    if silu:
        a = F.silu(a)
    (a * mask).backward(da)
    return x.grad, gamma.grad, beta.grad


def test_gate_groupnorm_backward_catches_a_shifted_dropout_mask():
    """The dropout mask applied one voxel row off (x shifted by one)."""
    g = _gen(6)
    B, C, R = 1, 96, 6
    x = torch.randn(B, C, R, R, R, generator=g, dtype=torch.float64)
    gamma, beta = 1 + 0.5 * torch.randn(C, generator=g, dtype=torch.float64), torch.randn(C, generator=g, dtype=torch.float64)
    da = torch.randn(B, C, R, R, R, generator=g, dtype=torch.float64)
    keep = (torch.rand(B, C, R, R, R, generator=g) >= 0.3).double() / 0.7
    good = _gn_backward(x, gamma, beta, da, keep)
    bad = _gn_backward(x, gamma, beta, da, torch.roll(keep, 1, dims=-1))
    for precision in ("bf16", "bf16x3"):
        for gd, bd in zip(good, bad):
            assert gv.rel_err(bd, gd) > 5 * gv.GATES["gnb"][precision]
