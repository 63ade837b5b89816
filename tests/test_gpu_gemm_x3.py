"""Split-bf16 ("bf16x3") implicit-GEMM convolutions against an fp64 CPU reference, and the per-launch accounting of the
GEMM plan.

In bf16x3 an entry of the load table brings the hi and lo parts of its A box and every k-step the W_hi and W_lo tiles;
per k16 step A_hi . [W_hi; W_lo] is one m64n(2 BLOCK_N) wgmma and A_lo . W_hi one m64nBLOCK_N wgmma. These cases cover
the tile shapes of the load tables: the y-halo box (3^3 and the 5-tap head), tiles without halo that span samples
(bb > 1), the stride-2 parity maps, pointwise (NIN-shaped) and N <= 32. Split-K, the sub-pixel upsample and the
attention pair with an activation B operand run inside the full network (test_gpu_unet.py, smoke()).
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-4  # the bf16x3 tolerance of test_gpu_conv.py (max |diff| / max |ref|)

CASES = [
    # (B, Cin, Cout, R, k, stride)
    (2, 128, 128, 16, 3, 1),   # (8,16,1,1) tile, 3-tap y-halo reuse
    (1, 128, 4, 32, 5, 1),     # 5-tap reuse, N = 4 (BLOCK_N 32)
    (2, 128, 256, 8, 3, 1),    # (8,8,2,1) tile, no halo
    (3, 512, 512, 4, 3, 1),    # (4,4,4,2) tile spanning samples, odd batch
    (2, 256, 256, 8, 3, 2),    # stride 2: parity sub-grid maps
    (2, 384, 128, 16, 1, 1),   # pointwise
    (2, 64, 32, 16, 3, 1),     # N = 32, one channel chunk
]


def _conv_ref64(x, w, b, k, stride):
    x, w, b = x.double().cpu(), w.double().cpu(), b.double().cpu()
    if stride == 1:
        return F.conv3d(x, w, b, padding=k // 2)
    return F.conv3d(F.pad(x, (0, 1, 0, 1, 0, 1)), w, b, stride=2, padding=0)


def _inputs(case, seed=1234):
    B, Cin, Cout, R, k, _ = case
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, Cin, R, R, R, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, k, device="cuda", generator=g) / (Cin * k ** 3) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    return x, w, b


def _conv(x, w, b, stride):
    from meshdiffusion_b200 import ops
    y = ops.conv3d(ops.to_ndhwc(x, "bf16x3"), w, b, stride=stride, precision="bf16x3")
    return ops.from_ndhwc(y, "bf16x3")


@pytest.mark.parametrize("case", CASES)
def test_x3_conv_matches_fp64(case):
    x, w, b = _inputs(case)
    out = _conv(x, w, b, case[5]).double().cpu()
    ref = _conv_ref64(x, w, b, case[4], case[5])
    assert out.shape == ref.shape
    err = (out - ref).abs().max().item() / ref.abs().max().item()
    print(f"bf16x3 conv {case}: rel err vs fp64 {err:.3e}")
    assert err < TOL


@pytest.mark.parametrize("case", [CASES[0], CASES[3], CASES[4]])
def test_x3_conv_batch_invariant_and_reproducible(case):
    x, w, b = _inputs(case)
    stride = case[5]
    full = _conv(x, w, b, stride)
    again = _conv(x, w, b, stride)
    assert torch.equal(full, again), "two identical launches differ"
    for i in range(x.shape[0]):
        one = _conv(x[i:i + 1].contiguous(), w, b, stride)
        assert torch.equal(one[0], full[i]), f"sample {i} depends on the rest of the batch"


def _tiny_engine(precision, B=2):
    from configs import res64
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth
    cfg = res64.get_config()
    synth.apply_tiny(cfg, "res64")
    cfg.model.compute_dtype = precision
    cfg.model.engine_max_batch = B
    cfg.device = torch.device("cuda:0")
    model = mutils.create_model(cfg)
    model.eval()
    net = model.module
    x = torch.randn(B, 4, 16, 16, 16, device="cuda")
    with torch.no_grad():
        model(x, torch.full((B,), 10.0, device="cuda"))
    return net


def test_gemm_ops_accounting():
    """bf16x3 moves each A box and weight tile part once: exactly twice the bf16 fill bytes, for the same FLOPs."""
    ops = {}
    for prec in ("bf16", "bf16x3"):
        net = _tiny_engine(prec)
        ops[prec] = net.gemm_ops()
        net.release_engine()
    assert [r[0] for r in ops["bf16"]] == [r[0] for r in ops["bf16x3"]]
    for (name, fl1, fb1), (_, fl3, fb3) in zip(ops["bf16"], ops["bf16x3"]):
        assert fl1 > 0 and fb1 > 0, name
        assert fl3 == fl1, name
        assert fb3 == 2 * fb1, name
