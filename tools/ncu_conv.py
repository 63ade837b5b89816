"""One convolution through the C ABI, for profiler captures of the wgmma implicit-GEMM kernel, e.g.:

    ncu --set full --import-source on -k regex:gemm_tc -s 1 -c 1 -o conv_prof \
        python tools/ncu_conv.py <bf16|tf32|bf16x3> <B> <Cin> <Cout> <R> [reps]
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from meshdiffusion_b200 import ops  # noqa: E402

prec, B, Cin, Cout, R = sys.argv[1], int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5])
reps = int(sys.argv[6]) if len(sys.argv) > 6 else 3
g = torch.Generator(device="cuda").manual_seed(0)
x = ops.to_ndhwc(torch.randn(B, Cin, R, R, R, device="cuda", generator=g), prec)
w = torch.randn(Cout, Cin, 3, 3, 3, device="cuda", generator=g) / (Cin * 27) ** 0.5
b = torch.randn(Cout, device="cuda", generator=g)
for _ in range(reps):
    y, st = ops.conv3d(x, w, b, want_stats=True, precision=prec)
torch.cuda.synchronize()
print("ok", y.shape)
