"""Class-conditional score networks and classifier-free guidance on the GPU: the engine's forward and gradients against
the fp32 conditional oracle, the graph cache under changing class ids, the guided solver kernel against its eager
oracle, and the guided device loop against the per-entry public path."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import rel_l2, rel_max, tiny_config
from oracle import synth, unet_oracle

import class_oracle
from test_guidance_cpu import analytic_gate

pytestmark = pytest.mark.gpu

TOL_MAX = {"bf16x3": 1e-3, "bf16": 4e-2}
TOL_L2 = {"bf16x3": 1e-3, "bf16": 3e-2}
K = 3
GRAD_TOL = {"bf16": (3e-2, 1e-1), "bf16x3": (1e-3, 1e-2)}  # (global rel-L2, one tensor's rel-L2)


def _models(name, precision, embed_seed=1):
    """(conditional model, K = 0 model, conditional state dict): the same synthetic weights, a random label embedding."""
    from meshdiffusion_b200.diffusion.models import utils as mutils
    cfg = tiny_config(name, precision)
    cfg.device = torch.device("cuda:0")
    cfg.model.dropout = 0.0
    base = mutils.create_model(cfg)
    sd = synth.synthetic_state_dict({k: v.detach().cpu() for k, v in base.module.state_dict().items()}, seed=21)
    base.module.load_state_dict(sd)
    cfg.model.num_classes = K
    cond = mutils.create_model(cfg)
    sdc = dict(sd)
    sdc["label_embed.weight"] = torch.randn(K + 1, 4 * cfg.model.nf, generator=torch.Generator().manual_seed(embed_seed)) * 0.5
    cond.module.load_state_dict(sdc)
    base.eval(); cond.eval()
    return cond, base, sdc, cfg


@pytest.mark.parametrize("name", ["res64", "res128"])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_forward_matches_conditional_oracle(name, precision):
    cond, base, sd, cfg = _models(name, precision)
    x, labels = synth.synthetic_inputs(cfg.data.image_size, 4, 8, sd["mask"])
    y = torch.tensor([0, 2, 3, 1], dtype=torch.int32)
    with torch.no_grad():
        out = cond(x.cuda(), labels.cuda(), class_labels=y.cuda()).cpu()
        null = cond(x.cuda(), labels.cuda()).cpu()
    arch = unet_oracle.arch_from_config(cfg)
    ref = class_oracle.unet_forward(sd, arch, x, labels, y)
    ref_null = class_oracle.unet_forward(sd, arch, x, labels, None)
    print(f"{name}/{precision}: rel max {rel_max(out, ref):.2e}, rel l2 {rel_l2(out, ref):.2e}")
    assert rel_max(out, ref) < TOL_MAX[precision] and rel_l2(out, ref) < TOL_L2[precision]
    assert rel_max(null, ref_null) < TOL_MAX[precision]
    # the classes matter
    assert rel_max(out, ref_null) > 10 * TOL_MAX[precision]
    # a zero embedding: bitwise the K = 0 engine
    cond.module.label_embed.weight.data.zero_()
    with torch.no_grad():
        z = cond(x.cuda(), labels.cuda(), class_labels=y.cuda())
        b = base(x.cuda(), labels.cuda())
    assert torch.equal(z, b)


def test_out_of_range_ids_and_unconditional_refusal():
    from meshdiffusion_b200 import _native
    cond, base, sd, cfg = _models("res64", "bf16")
    x, labels = synth.synthetic_inputs(16, 2, 8, sd["mask"])
    with pytest.raises(_native.NativeError, match="outside 0..3"):
        cond(x.cuda(), labels.cuda(), class_labels=torch.tensor([0, 4], dtype=torch.int32).cuda())
    with pytest.raises(_native.NativeError, match="outside"):
        cond(x.cuda(), labels.cuda(), class_labels=torch.tensor([-1, 0], dtype=torch.int32).cuda())
    with pytest.raises(ValueError, match="unconditional"):
        base(x.cuda(), labels.cuda(), class_labels=torch.tensor([0, 1]).cuda())
    L = _native.lib()
    base(x.cuda(), labels.cuda())
    ids = torch.zeros(2, dtype=torch.int32, device="cuda")
    assert L.mdb_unet_set_classes(base.module._handle, _native.ptr(ids), 2, _native.current_stream()) != 0


def _oracle_grads(sd, arch, x, labels, y, noise, mask):
    # fp32 autograd: no TF32 in the oracle's convolutions and matmuls (as test_gpu_backward_x3.py)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sdg = {k: (v.cuda().clone().requires_grad_(True) if v.dtype == torch.float32 and k not in ("mask", "coords") else v.cuda())
           for k, v in sd.items()}
    pred = class_oracle.unet_forward(sdg, arch, x, labels, y)
    loss = (torch.square(pred - noise) * mask).reshape(x.shape[0], -1).mean(dim=-1).mean() / mask.sum() * mask.numel()
    loss.backward()
    return {k: v.grad for k, v in sdg.items() if v.dtype == torch.float32 and v.requires_grad and v.grad is not None}


@pytest.mark.parametrize("name,precision", [("res64", "bf16"), ("res128", "bf16"), ("res64", "bf16x3")])
def test_gradients_match_autograd_and_repeat(name, precision):
    cond, _, sd, cfg = _models(name, "bf16x3")
    cond.module.train_precision = precision
    net = cond.module
    R, B = cfg.data.image_size, 4
    x, labels = synth.synthetic_inputs(R, B, 31, sd["mask"])
    x, labels = x.cuda(), labels.cuda()
    y = torch.tensor([1, K, 1, 0], dtype=torch.int32, device="cuda")  # class 2 unused: its gradient row is zero
    noise = torch.randn(x.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    mask = sd["mask"].cuda().view(1, 1, R, R, R)
    ref = _oracle_grads(sd, unet_oracle.arch_from_config(cfg), x, labels, y, noise, mask)

    def run():
        for p in net.parameters():
            p.grad = None
        net.train()
        pred = cond(x, labels, class_labels=y)
        loss = (torch.square(pred - noise) * mask).reshape(B, -1).mean(dim=-1).mean() / mask.sum() * mask.numel()
        loss.backward()
        return {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}

    g1, g2 = run(), run()
    for n in g1:
        assert torch.equal(g1[n], g2[n]), f"{n}: repeat runs differ"
    num = sum((g1[n] - r).double().pow(2).sum().item() for n, r in ref.items() if n in g1)
    den = sum(r.double().pow(2).sum().item() for n, r in ref.items() if n in g1)
    e = (g1["label_embed.weight"] - ref["label_embed.weight"]).double().norm() / ref["label_embed.weight"].double().norm()
    print(f"{name}/{precision}: global rel-l2 {(num / den) ** 0.5:.3e}, label_embed {e.item():.3e}")
    glob_tol, tensor_tol = GRAD_TOL[precision]  # the gates of test_gpu_backward.py / test_gpu_backward_x3.py
    assert (num / den) ** 0.5 < glob_tol and e < tensor_tol
    assert torch.equal(g1["label_embed.weight"][2], torch.zeros_like(g1["label_embed.weight"][2]))
    # the all-reduce buckets see the new slot
    from meshdiffusion_b200 import _native
    off, rdy = ctypes.c_longlong(), ctypes.c_int()
    L = _native.lib()
    _native.check(L.mdb_unet_grad_offset(net._train_handle, b"label_embed.weight", ctypes.byref(off)))
    _native.check(L.mdb_unet_grad_ready(net._train_handle, b"label_embed.weight", ctypes.byref(rdy)))
    assert off.value + net.label_embed.weight.numel() == net._flat_grad.numel() and rdy.value > 0
    # ... in a bucket of its own: it is final only after the last launch, the head's gradients before it much earlier
    net.bucket_bytes, net._buckets = 4096, None
    buckets = net._grad_buckets()
    assert (rdy.value, off.value, net._flat_grad.numel()) in buckets
    before = [b for b in buckets if b[2] == off.value]
    assert len(before) == 1 and before[0][0] < rdy.value
    lo_ends = sorted((b[1], b[2]) for b in buckets)
    assert lo_ends[0][0] == 0 and all(a[1] == b[0] for a, b in zip(lo_ends, lo_ends[1:]))


def _table(n_steps=4, stochastic=False):
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    sde = sde_lib.VPSDE(0.1, 20.0, 1000, device="cuda:0")
    return sde, sampling.dpm_solver_schedule(sde, n_steps, stochastic)[1]


@pytest.mark.parametrize("second_order", [False, True])
@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("kept", [False, True])
def test_guided_entry_kernel_matches_eager(second_order, noise, kept):
    from meshdiffusion_b200.diffusion import sampling
    g = torch.Generator(device="cuda").manual_seed(3)
    B, C, R = 3, 4, 64  # res64: every block strides over its row
    shape = (B, C, R, R, R)
    eps_c, eps_u, x, h = (torch.randn(shape, device="cuda", generator=g) for _ in range(4))
    mask = (torch.rand(R, R, R, device="cuda", generator=g) < 0.7).float()
    z = torch.randn(shape, device="cuda", generator=g) if noise else None
    row = np.array([0, 500, 0.6, 1.3, 0.9, 0.4, -0.2 if second_order else 0.0, 0.3 if noise else 0.0, 0.8, 0.6], np.float32)
    entry = sampling._entries_c(row[None])[0]
    kn = zk = None
    if kept:
        kn = sampling._Known(torch.randn(shape, device="cuda", generator=g), (torch.rand(B, R, R, R, device="cuda", generator=g) < 0.5).float(),
                             [0, 2], B)
        zk = torch.randn(shape, device="cuda", generator=g)
    for w in (3.0, 1.0, 0.0):
        xa, ha, xb, hb = x.clone(), h.clone(), x.clone(), h.clone()
        sampling._update(eps_c, xa, ha, mask.reshape(-1), entry, z, kn, zk, eps_u=eps_u, w=w)
        sampling._update_eager(eps_c, xb, hb, mask, row, z, kn, zk, eps_u=eps_u, w=w)
        assert torch.equal(xa, xb) and torch.equal(ha, hb), w


@pytest.mark.parametrize("w", [3.0, 1.0])
def test_guided_device_loop_matches_per_entry_path(w):
    """mdb_solver_run_guided (CUDA graphs over alternating class ids and the null class on the same x) against model
    calls + mdb_solver_update_guided per entry, bitwise."""
    from meshdiffusion_b200.diffusion import sampling
    cond, _, sd, cfg = _models("res64", "bf16x3")
    R, B = cfg.data.image_size, 3
    sde, table = _table(6)
    y = torch.tensor([2, 0, 1], dtype=torch.int32, device="cuda")
    x0 = torch.randn(B, 4, R, R, R, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    gm = sd["mask"].cuda().reshape(R, R, R)
    a = sampling._run_table(sde, table, cond, x0.clone(), gm, "t", native=True, class_labels=y, w=w)
    b = sampling._run_table(sde, table, cond, x0.clone(), gm, "t", native=False, class_labels=y, w=w)
    assert torch.equal(a, b)
    if w == 1.0:
        # bitwise mdb_unet_set_classes + the plain device loop
        from meshdiffusion_b200 import _native
        net = cond.module
        L = _native.lib()
        xm = (x0 * gm).contiguous()
        hist = torch.empty_like(xm)
        entries = sampling._entries_c(table)
        eps_buf, lab = torch.empty_like(xm), torch.empty(B, device="cuda")
        with net.frozen():
            _native.check(L.mdb_unet_set_classes(net._handle, _native.ptr(y), B, _native.current_stream()))
            _native.check(L.mdb_solver_run(net._handle, _native.ptr(xm), _native.ptr(hist), _native.ptr(gm.reshape(-1)),
                                           entries, len(entries), B, 0, _native.ptr(eps_buf), _native.ptr(lab), 0, None,
                                           len(entries), _native.current_stream()))
        assert torch.equal(a, xm)
    else:
        # guidance changes the result
        c = sampling._run_table(sde, table, cond, x0.clone(), gm, "t", native=True, class_labels=y, w=1.0)
        assert not torch.equal(a, c)


def test_graph_cache_follows_class_ids():
    """Repeated forwards on the same x / labels / out buffers through the graph-replaying loop, with the class ids
    changing between calls (and the null class), equal fresh eager forwards."""
    from meshdiffusion_b200.diffusion import sampling
    cond, _, sd, cfg = _models("res64", "bf16x3")
    R, B = cfg.data.image_size, 2
    sde, table = _table(2)
    gm = torch.ones(R, R, R, device="cuda")
    x0 = torch.randn(B, 4, R, R, R, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    for ids in ([0, 1], [2, 2], [1, 0], [0, 1]):
        y = torch.tensor(ids, dtype=torch.int32, device="cuda")
        for _ in range(3):  # first call eager, second captures, third replays
            a = sampling._run_table(sde, table, cond, x0.clone(), gm, "t", native=True, class_labels=y, w=2.0)
        b = sampling._run_table(sde, table, cond, x0.clone(), gm, "t", native=False, class_labels=y, w=2.0)
        assert torch.equal(a, b), ids


def test_analytic_guided_gaussian_gpu():
    analytic_gate("cuda:0")


def test_pc_native_loop_with_a_single_python_int_class():
    """The pc sampler's device loop with class_labels given as one Python int (a temporary id tensor the engine must
    copy) equals the same loop with a persistent per-sample id tensor, and differs from another class."""
    from meshdiffusion_b200.diffusion import sampling, sde_lib
    cond, _, sd, cfg = _models("res64", "bf16")
    R, B = cfg.data.image_size, 2
    sde = sde_lib.VPSDE(0.1, 20.0, 1000, device="cuda:0")
    gm = sd["mask"].cuda().view(1, 1, R, R, R)
    fn = sampling.get_pc_sampler(sde, (B, 4, R, R, R), sampling.AncestralSamplingPredictor, sampling.NoneCorrector,
                                 lambda v: v, 0.16, device="cuda:0", grid_mask=gm, max_iters=4, native_rng=True, seed=3)
    ids = torch.ones(B, dtype=torch.int32, device="cuda")

    def run(cl):
        torch.manual_seed(0)
        return fn(cond, class_labels=cl)[0]

    a, b, c = run(1), run(ids), run(0)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)


def test_train_checkpoint_and_guided_uncond_gen_cli(tmp_path):
    """`--mode=train` on two synthetic classes, the checkpoint's layout and class count, then `uncond_gen` with a class
    label and guidance_scale 3 from that checkpoint, with files of the usual shape."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(args):
        r = subprocess.run([sys.executable, os.path.join(root, "main_diffusion.py"), f"--config={root}/configs/res64.py",
                            "--config.model.num_classes=2", "--config.model.nf=32", "--config.model.ch_mult=(1, 2, 2, 2)",
                            "--config.model.num_res_blocks=1", "--config.model.compute_dtype=bf16"] + args,
                           cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        return r

    wd = tmp_path / "run"
    r = run(["--mode=train", f"--config.training.train_dir={wd}", "--config.data.synthetic=True",
             "--config.training.batch_size=2", "--config.training.n_iters=3", "--config.training.log_freq=1",
             "--config.training.snapshot_freq_for_preemption=2", "--config.training.snapshot_freq=100000",
             "--config.training.class_dropout=0.5"])
    losses = [float(l.split("training_loss:")[1]) for l in (r.stderr + r.stdout).splitlines() if "training_loss:" in l]
    assert len(losses) >= 3 and all(np.isfinite(losses))
    ckpt = wd / "checkpoints" / "checkpoint_3.pth"
    ck = torch.load(ckpt, map_location="cpu", weights_only=False)
    assert tuple(ck["model"]["module.label_embed.weight"].shape) == (3, 128)
    assert ck["model"]["module.label_embed.weight"].abs().sum() > 0  # trained away from its zero init
    frozen = ("module.sigmas", "module.mask", "module.coords")  # the EMA list holds the trainable tensors, label_embed last
    assert len(ck["ema"]["shadow_params"]) == len([k for k in ck["model"] if k not in frozen])
    out = tmp_path / "samples"
    run(["--mode=uncond_gen", f"--config.eval.eval_dir={out}", f"--config.eval.ckpt_path={ckpt}",
         "--config.eval.batch_size=2", "--config.eval.class_label=1", "--config.sampling.guidance_scale=3.0",
         "--config.sampling.method=dpm_solver", "--config.sampling.dpm_steps=4", "--config.sampling.native_rng=True"])
    x = np.load(out / "0.npy")
    assert x.shape == (2, 4, 64, 64, 64) and x.dtype == np.float32 and np.isfinite(x).all()
    # the checkpoint round trip: a config with another class count is refused, naming both counts
    r = subprocess.run([sys.executable, os.path.join(root, "main_diffusion.py"), f"--config={root}/configs/res64.py",
                        "--config.model.num_classes=3", "--config.model.nf=32", "--config.model.ch_mult=(1, 2, 2, 2)",
                        "--config.model.num_res_blocks=1", "--mode=uncond_gen", f"--config.eval.eval_dir={out}",
                        f"--config.eval.ckpt_path={ckpt}", "--config.eval.batch_size=1"],
                       cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "has 2 classes" in r.stderr and "num_classes) 3" in r.stderr
