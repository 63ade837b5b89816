"""Context number (not a bench arm): forward + backward of the reference's op sequence with stock PyTorch autograd on the
same GPU (bf16 autocast, and fp32 with TF32 convolutions = torch's default, what the reference's trainer runs), next to
which tools/bench_train.py's fwd+bwd time can be read. Uses the oracle restatement as the stock-torch model."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from configs import res64
from meshdiffusion_b200.diffusion.models import utils as mutils
from meshdiffusion_b200.diffusion.models.init_utils import random_init_nondegenerate
from oracle import unet_oracle

B = int(sys.argv[1]) if len(sys.argv) > 1 else 4
cfg = res64.get_config(); cfg.device = torch.device("cpu")
torch.manual_seed(0)
net = mutils.create_model(cfg, use_parallel=False)
random_init_nondegenerate(net)
sd = {k: (v.detach().cuda().requires_grad_(v.dtype == torch.float32 and k not in ("mask", "coords"))) for k, v in net.state_dict().items()}
arch = dict(net.arch)
x = torch.randn(B, 4, 64, 64, 64, device="cuda"); labels = torch.rand(B, device="cuda") * 999
noise = torch.randn_like(x)
res = {"batch": B}
for name, amp in (("bf16_autocast", True), ("fp32_tf32conv", False)):
    torch.backends.cudnn.allow_tf32 = True; torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    try:
        def step():
            for v in sd.values():
                v.grad = None
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                pred = unet_oracle.unet_forward(sd, arch, x, labels)
            (pred.float() - noise).square().mean().backward()
        for _ in range(2): step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        n = 3
        for _ in range(n): step()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        res[name] = {"ms_per_fwd_bwd": ms, "samples_per_s": B / (ms * 1e-3), "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30}
    except Exception as ex:
        res[name] = {"error": str(ex)[:200]}
    torch.cuda.empty_cache()
print(json.dumps(res))
