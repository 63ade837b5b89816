"""The operand ring depth of the implicit-GEMM kernel changes when its loads are issued, never what it computes: the same
launches at MDB_MAX_BSLOTS=2 (the ring depth of the kernel that staged all 128 accumulator columns at once) and at the
default give the same bits, for outputs, GroupNorm statistics, data / weight gradients and a training step with the fused
GroupNorm-backward epilogue."""
import hashlib

import pytest
import torch

pytestmark = pytest.mark.gpu


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def _at_caps(monkeypatch, fn):
    """fn() at MDB_MAX_BSLOTS=2 and at the default ring depth: two lists of digests."""
    out = []
    for cap in ("2", None):
        with monkeypatch.context() as m:
            m.delenv("MDB_MAX_STAGES", raising=False)
            if cap is None:
                m.delenv("MDB_MAX_BSLOTS", raising=False)
            else:
                m.setenv("MDB_MAX_BSLOTS", cap)
            out.append([_digest(t) for t in fn()])
            torch.cuda.synchronize()
    return out


CONV_CASES = [
    # (B, Cin, Cout, R, k): a res64 level-0 ResnetBlock conv0 (3^3 halo, three k-steps per entry) and a 5^3 conv
    (1, 256, 128, 64, 3),
    (1, 128, 128, 32, 5),
]


@pytest.mark.parametrize("precision", ["bf16", "tf32", "bf16x3"])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv3d_bits_independent_of_ring_depth(case, precision, monkeypatch):
    from meshdiffusion_b200 import ops
    B, Cin, Cout, R, k = case
    g = torch.Generator(device="cuda").manual_seed(21)
    x = ops.to_ndhwc(torch.randn(B, Cin, R, R, R, device="cuda", generator=g), precision)
    res = ops.to_ndhwc(torch.randn(B, Cout, R, R, R, device="cuda", generator=g), precision)
    w = torch.randn(Cout, Cin, k, k, k, device="cuda", generator=g) / (Cin * k ** 3) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    small, deep = _at_caps(monkeypatch, lambda: ops.conv3d(x, w, b, residual=res, want_stats=True, precision=precision))
    assert small == deep


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_conv3d_backward_bits_independent_of_ring_depth(precision, monkeypatch):
    from meshdiffusion_b200 import ops
    B, Cin, Cout, R, k = CONV_CASES[0]
    g = torch.Generator(device="cuda").manual_seed(22)
    x = ops.to_ndhwc(torch.randn(B, Cin, R, R, R, device="cuda", generator=g), precision)
    dy = ops.to_ndhwc(torch.randn(B, Cout, R, R, R, device="cuda", generator=g), precision)
    w = torch.randn(Cout, Cin, k, k, k, device="cuda", generator=g) / (Cin * k ** 3) ** 0.5
    small, deep = _at_caps(monkeypatch, lambda: ops.conv3d_backward(dy, x, w, precision=precision))
    assert small == deep


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_training_step_bits_independent_of_ring_depth(precision, monkeypatch):
    """One training step at the tiny config (batch 2, dropout 0.1): forward output and the flat gradient buffer."""
    from configs import res64
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth

    def step():
        torch.manual_seed(1234)  # the dropout seed derives from torch.initial_seed() and a per-model call counter
        cfg = res64.get_config()
        synth.apply_tiny(cfg, "res64")
        cfg.model.compute_dtype = precision
        cfg.training.compute_dtype = precision
        cfg.model.dropout = 0.1
        cfg.model.scale_by_sigma = False
        cfg.device = torch.device("cuda:0")
        model = mutils.create_model(cfg)
        net = model.module
        sd = synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=3)
        net.load_state_dict(sd)
        net.train()
        x, labels = synth.synthetic_inputs(cfg.data.image_size, 2, 8, sd["mask"])
        y = model(x.cuda(), labels.cuda())
        y.square().mean().backward()
        out = [y.detach().clone(), net._flat_grad.detach().clone()]
        net.release_engine()
        return out

    small, deep = _at_caps(monkeypatch, step)
    assert small == deep
