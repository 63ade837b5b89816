"""Operator-level wrappers over the C ABI (used by the parity tests; the engine itself stays inside the library).

Activations are NDHWC torch tensors on the GPU: bfloat16 for precision='bf16', float32 for precision='tf32', and for
precision='bf16x3' (split bf16) bfloat16 rows of 2C entries: the hi parts bf16(v) of the C channels followed by their
lo parts bf16(v - hi).
"""
import torch

from . import _native

PRECISIONS = {"bf16": 0, "tf32": 1, "bf16x3": 2}
STAT_WORDS = 4  # csrc/gn_stats.cuh: (sum lo, sum hi, sumsq lo, sumsq hi); value = lo * 2^-24 + hi * 2^16


def stats_to_words(stats):
    """float64 [B,C,2] (sum, sum of squares) -> the library's int64 [B,C,4] split fixed-point record."""
    v = stats.double()
    hi = torch.round(v / 65536.0)
    lo = torch.round((v - hi * 65536.0) * 16777216.0)
    return torch.stack([lo[..., 0], hi[..., 0], lo[..., 1], hi[..., 1]], dim=-1).to(torch.int64).contiguous()


def words_to_stats(words):
    w = words.double()
    return torch.stack([w[..., 0] / 16777216.0 + w[..., 1] * 65536.0, w[..., 2] / 16777216.0 + w[..., 3] * 65536.0], dim=-1)


def _act_dtype(precision):
    return torch.float32 if precision == "tf32" else torch.bfloat16


def to_ndhwc(x_ncdhw, precision):
    """[B,C,D,H,W] fp32 -> contiguous [B,D,H,W,C] in the operand dtype ([B,D,H,W,2C] = hi | lo for 'bf16x3')."""
    y = x_ncdhw.permute(0, 2, 3, 4, 1).contiguous()
    if precision == "bf16x3":
        hi = y.to(torch.bfloat16)
        lo = (y.float() - hi.float()).to(torch.bfloat16)
        return torch.cat([hi, lo], dim=-1).contiguous()
    return y.to(_act_dtype(precision))


def from_ndhwc(y, precision=None):
    if precision == "bf16x3":
        C = y.shape[-1] // 2
        y = y[..., :C].float() + y[..., C:].float()
    return y.float().permute(0, 4, 1, 2, 3).contiguous()


def conv3d(x, weight, bias=None, stride=1, rowbias=None, residual=None, want_stats=False, precision="bf16"):
    """nn.Conv3d (k in {1,3,5}; stride 1 'same' or the Downsample stride-2 pad-high variant) on NDHWC input.

    x: [B,Z,Y,X,Cin]; weight: fp32 [Cout,Cin,k,k,k]. Returns y [B,Zo,Yo,Xo,Cout] (and stats [B,Cout,2] float64).
    """
    L = _native.lib()
    assert x.is_cuda and x.is_contiguous() and x.dtype == _act_dtype(precision)
    B, Z, Y, X, Cin = x.shape
    parts = 2 if precision == "bf16x3" else 1
    Cin //= parts
    Cout, k = weight.shape[0], weight.shape[2]
    assert weight.shape[1] == Cin
    w = weight.detach().float().contiguous()
    y = torch.empty((B, Z // stride, Y // stride, X // stride, Cout * parts), device=x.device, dtype=x.dtype)
    stats = torch.zeros((B, Cout, STAT_WORDS), device=x.device, dtype=torch.int64) if want_stats else None
    b = bias.detach().float().contiguous() if bias is not None else None
    rb = rowbias.detach().float().contiguous() if rowbias is not None else None
    if residual is not None:
        assert residual.shape == y.shape and residual.dtype == y.dtype and residual.is_contiguous()
    _native.check(L.mdb_conv3d(_native.ptr(x), B, Cin, Z, Y, X, _native.ptr(w), _native.ptr(b), Cout, k, stride,
                               _native.ptr(y), _native.ptr(rb), _native.ptr(residual), _native.ptr(stats),
                               PRECISIONS[precision], _native.current_stream()))
    # statistics are split fixed-point integers inside the library; return them as float64 (sum, sum of squares)
    return (y, words_to_stats(stats)) if want_stats else y


def groupnorm_act(x, stats, gamma, beta, silu=True, precision="bf16"):
    """GroupNorm(32, eps=1e-6) (+SiLU) on NDHWC x using per-channel (sum, sumsq) statistics."""
    L = _native.lib()
    B, C = x.shape[0], x.shape[-1]
    V = x.numel() // (B * C)
    if precision == "bf16x3":
        C //= 2
    y = torch.empty_like(x)
    stats = stats_to_words(stats)
    g = gamma.detach().float().contiguous()
    bt = beta.detach().float().contiguous()
    _native.check(L.mdb_groupnorm_act(_native.ptr(x), _native.ptr(stats), _native.ptr(g), _native.ptr(bt), _native.ptr(y),
                                      B, V, C, 1 if silu else 0, PRECISIONS[precision], _native.current_stream()))
    return y


def sampler_update(eps, x, noise, mask, beta, std, seed=0, offset=0):
    """In-place ancestral update; returns (x, x_mean). eps/x/noise: fp32 [B,C,R,R,R]; mask fp32 [R,R,R]."""
    L = _native.lib()
    B, C = x.shape[0], x.shape[1]
    V = x[0, 0].numel()
    x_mean = torch.empty_like(x)
    _native.check(L.mdb_sampler_update(_native.ptr(eps), _native.ptr(x), _native.ptr(x_mean), _native.ptr(noise),
                                       _native.ptr(mask), float(beta), float(std), V, C, B, seed, offset, None,
                                       _native.current_stream()))
    return x, x_mean


def conv3d_backward(dy, x, weight, stride=1, want_dw=True, want_dx=True, precision="bf16"):
    """NDHWC conv3d backward: dy [B,Zo,Yo,Xo,Cout], x [B,Z,Y,X,Cin], weight fp32 OIDHW -> (dw fp32 OIDHW, dx).

    precision 'bf16' (bf16 tensors) or 'bf16x3' (split bf16: rows of 2C, see to_ndhwc); dx has the dtype / layout of x."""
    L = _native.lib()
    if precision not in ("bf16", "bf16x3"):
        raise ValueError("conv3d_backward: precision must be 'bf16' or 'bf16x3'")
    assert dy.dtype == torch.bfloat16 and x.dtype == torch.bfloat16 and dy.is_contiguous() and x.is_contiguous()
    B, Z, Y, X, Cin = x.shape
    parts = 2 if precision == "bf16x3" else 1
    Cin //= parts
    Cout, k = weight.shape[0], weight.shape[2]
    assert weight.shape[1] == Cin and dy.shape[-1] == Cout * parts
    w = weight.detach().float().contiguous()
    dw = torch.zeros_like(w) if want_dw else None
    dx = torch.empty_like(x) if want_dx else None
    _native.check(L.mdb_conv3d_backward_prec(_native.ptr(dy), _native.ptr(x), _native.ptr(w), B, Cin, Cout, Z, Y, X, k, stride,
                                             _native.ptr(dw), _native.ptr(dx), PRECISIONS[precision], _native.current_stream()))
    return dw, dx


def groupnorm_act_backward(x, stats, gamma, beta, da, add=None, silu=True, dropout_p=0.0, seed=0, precision="bf16"):
    """Backward of groupnorm_act: returns (dx [B,...,C], dgamma fp32 [C], dbeta fp32 [C]).

    precision 'bf16' (bf16 tensors) or 'bf16x3' (x, da, add and dx as split-bf16 rows of 2C, see to_ndhwc)."""
    L = _native.lib()
    if precision not in ("bf16", "bf16x3"):
        raise ValueError("groupnorm_act_backward: precision must be 'bf16' or 'bf16x3'")
    B, C = x.shape[0], x.shape[-1]
    V = x.numel() // (B * C)
    if precision == "bf16x3":
        C //= 2
    stats = stats_to_words(stats)
    g = gamma.detach().float().contiguous()
    bt = beta.detach().float().contiguous()
    dx = torch.empty_like(x)
    dg = torch.empty(C, device=x.device, dtype=torch.float32)
    db = torch.empty(C, device=x.device, dtype=torch.float32)
    da = da.clone()  # the kernel pair overwrites dL/dy with the pre-activation gradient
    _native.check(L.mdb_groupnorm_act_backward_prec(_native.ptr(x), _native.ptr(stats), _native.ptr(g), _native.ptr(bt),
                                                    _native.ptr(da), _native.ptr(add), _native.ptr(dx), _native.ptr(dg),
                                                    _native.ptr(db), B, V, C, 1 if silu else 0, float(dropout_p), int(seed),
                                                    PRECISIONS[precision], _native.current_stream()))
    return dx, dg, db
