"""The implicit-GEMM epilogue at the shapes where its output box is clipped: partial M-tiles (batch 3 at 4^3 and 8^3),
partial column blocks (N = 96, 104), residual launches, in bf16, bf16x3 and tf32.

bf16 and bf16x3 128-column tiles store each 64-column round as one TMA box from a shared-memory slot, and load the
residual the same way; TMA clips the box at the grid, the batch and N. tf32 keeps the per-thread stores. Every case
compares against an fp64 reference at the gates of test_gpu_conv.py, and checks that nothing outside the output tensor
was written: the output sits between two guard regions of a larger buffer, filled with a sentinel. Channel-offset
outputs (the attention's qkv rows) and the sub-pixel upsample's parity-strided outputs have their own cases in
test_gpu_gemm_variants.py.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = {"tf32": 2e-3, "bf16": 2e-2, "bf16x3": 1e-4}
GUARD = 4096  # elements of sentinel on each side of the output
CASES = [
    # (B, Cin, Cout, R, k, residual)
    (3, 128, 128, 4, 3, False),   # (4,4,4,2) tiles: the second batch tile has one sample of two
    (3, 128, 128, 4, 3, True),
    (3, 64, 256, 8, 3, True),     # (8,8,2,1) tiles, two column blocks
    (2, 64, 96, 16, 3, False),    # N = 96: round 1 half past N
    (2, 64, 104, 16, 3, True),    # N = 104: a chunk straddles N (dense rows need N % 8 == 0: 16-byte vectors)
    (2, 128, 64, 16, 1, True),    # N = 64: round 1 wholly past N, pointwise
    (3, 96, 128, 8, 3, True),     # K not a multiple of the k-step
]


def _case_id(c):
    return "B{}_ci{}_co{}_R{}_k{}{}".format(*c[:5], "_res" if c[5] else "")


def _to_ndhwc(x, precision):
    from meshdiffusion_b200 import ops
    return ops.to_ndhwc(x, precision)


def _run(x, w, b, res, precision):
    """mdb_conv3d into the middle of a sentinel-filled buffer: (output [B,R,R,R,Cout*parts], the two guard regions)."""
    from meshdiffusion_b200 import _native, ops
    L = _native.lib()
    B, Cin, R = x.shape[0], x.shape[1], x.shape[2]
    Cout, k = w.shape[0], w.shape[2]
    parts = 2 if precision == "bf16x3" else 1
    xa = _to_ndhwc(x, precision)
    dt = xa.dtype
    n = B * R * R * R * Cout * parts
    buf = torch.full((GUARD + n + GUARD,), 7.0, device="cuda", dtype=dt)
    y = buf[GUARD:GUARD + n].view(B, R, R, R, Cout * parts)
    ra = _to_ndhwc(res, precision) if res is not None else None
    _native.check(L.mdb_conv3d(_native.ptr(xa), B, Cin, R, R, R, _native.ptr(w.contiguous()), _native.ptr(b), Cout, k, 1,
                               _native.ptr(y), None, _native.ptr(ra), None, ops.PRECISIONS[precision],
                               _native.current_stream()))
    torch.cuda.synchronize()
    return ops.from_ndhwc(y, precision), buf[:GUARD], buf[GUARD + n:]


@pytest.mark.parametrize("precision", ["bf16", "bf16x3", "tf32"])
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_epilogue_clipped_boxes(case, precision):
    B, Cin, Cout, R, k, with_res = case
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(B, Cin, R, R, R, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, k, device="cuda", generator=g) / (Cin * k ** 3) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, Cout, R, R, R, device="cuda", generator=g) if with_res else None
    out, lo, hi = _run(x, w, b, res, precision)
    # the reference sees the operands as the kernel does: rounded to the operand format
    from meshdiffusion_b200 import ops
    xr = ops.from_ndhwc(_to_ndhwc(x, precision), precision)
    ref = F.conv3d(xr.double().cpu(), w.double().cpu(), b.double().cpu(), padding=k // 2)
    if with_res:
        ref = ref + ops.from_ndhwc(_to_ndhwc(res, precision), precision).double().cpu()
    err = (out.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
    print(f"{precision} {case}: rel err {err:.3e}")
    assert err < TOL[precision]
    assert bool((lo == 7.0).all()) and bool((hi == 7.0).all()), "the epilogue wrote outside the output tensor"
