"""Context number (not a bench arm): the reference's op sequence (oracle restatement = the same torch ops the reference
modules issue: conv3d / group_norm / silu / einsum / softmax / interpolate / cat) on the same GPU with stock PyTorch:
fp32 with TF32 convs (torch's default, what the reference runs) and bf16 autocast. Stand-in for the "1xA100-equivalent
PyTorch-GPU" figure of the north star (the reference publishes no number)."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from configs import res64
from meshdiffusion_b200.diffusion.models import utils as mutils
from meshdiffusion_b200.diffusion.models.init_utils import random_init_nondegenerate
from oracle import unet_oracle

B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
cfg = res64.get_config(); cfg.device = torch.device("cpu")
torch.manual_seed(0)
net = mutils.create_model(cfg, use_parallel=False)
random_init_nondegenerate(net)
sd = {k: v.detach().cuda() for k, v in net.state_dict().items()}
arch = dict(net.arch)
x = torch.randn(B, 4, 64, 64, 64, device="cuda"); labels = torch.rand(B, device="cuda") * 999
res = {"batch": B}
for name, tf32, amp in (("fp32_tf32conv", True, False), ("bf16_autocast", True, True), ("fp32_strict", False, False)):
    torch.backends.cudnn.allow_tf32 = tf32; torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.benchmark = True
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            for _ in range(2): unet_oracle.unet_forward(sd, arch, x, labels)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            n = 3
            for _ in range(n): unet_oracle.unet_forward(sd, arch, x, labels)
            e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        res[name] = {"ms_per_forward": ms, "sample_steps_per_s": B / (ms * 1e-3), "tflops": 5.757 * B / (ms * 1e-3) / 1e3}
    except Exception as ex:
        res[name] = {"error": str(ex)[:200]}
print(json.dumps(res))
