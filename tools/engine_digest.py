"""SHA-256 digests of what the native engine computes on seeded inputs, one line per output.

Two builds compute the same bits exactly when their digest lists are identical; this is the check for changes that must
not move a single bit (refactors, build changes). Covered, on synthetic weights and inputs:
  * the inference forward of every operand mode (bf16, tf32, bf16x3) at the tiny config;
  * one training step (forward output and the flat gradient buffer) with dropout 0.1 in bf16 and bf16x3, at the tiny
    config (batch 2) and at res64 (batch 1), with the fused GroupNorm-backward epilogue (MDB_GNB unset);
  * dx of the input-only backward (`mdb_unet_backward_input`, through ScoreNet.score_vjp) in bf16 and bf16x3;
  * ops.conv3d_backward (dw, dx) and ops.groupnorm_act_backward (dx, dgamma, dbeta; SiLU, dropout 0.1, an addend) in
    bf16 and bf16x3.

    python tools/engine_digest.py [--out digests.txt]
"""
import argparse
import hashlib
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def _model(name, precision, dropout=0.0, tiny=True):
    from configs import res64
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from oracle import synth
    cfg = res64.get_config()
    if tiny:
        synth.apply_tiny(cfg, name)
    cfg.model.compute_dtype = precision
    cfg.training.compute_dtype = precision if precision != "tf32" else "bf16"
    cfg.model.dropout = dropout
    cfg.model.scale_by_sigma = False
    cfg.device = torch.device("cuda:0")
    model = mutils.create_model(cfg)
    net = model.module
    sd = synth.synthetic_state_dict({k: v.detach().cpu() for k, v in net.state_dict().items()}, seed=3)
    net.load_state_dict(sd)
    return model, net, sd, cfg.data.image_size


def digests():
    from meshdiffusion_b200 import ops
    from oracle import synth
    out = []
    for precision in ("bf16", "tf32", "bf16x3"):
        model, net, sd, R = _model("res64", precision)
        model.eval()
        x, labels = synth.synthetic_inputs(R, 2, 8, sd["mask"])
        with torch.no_grad():
            out.append((f"forward.{precision}", _digest(model(x.cuda(), labels.cuda()))))
        net.release_engine()
    for tiny, batch in ((True, 2), (False, 1)):
        for precision in ("bf16", "bf16x3"):
            torch.manual_seed(1234)  # the dropout seed derives from torch.initial_seed() and a per-model call counter
            model, net, sd, R = _model("res64", precision, dropout=0.1, tiny=tiny)
            net.train()
            x, labels = synth.synthetic_inputs(R, batch, 8, sd["mask"])
            y = model(x.cuda(), labels.cuda())
            y.square().mean().backward()
            tag = f"train.{'tiny' if tiny else 'res64'}.B{batch}.{precision}"
            out += [(tag + ".out", _digest(y)), (tag + ".grads", _digest(net._flat_grad))]
            net.release_engine()
            del model, net
            torch.cuda.empty_cache()
    for precision in ("bf16", "bf16x3"):
        model, net, sd, R = _model("res64", precision)
        model.eval()
        x, labels = synth.synthetic_inputs(R, 2, 8, sd["mask"])
        v = torch.randn(x.shape, generator=torch.Generator().manual_seed(11))
        y, dx = net.score_vjp(x.cuda(), labels.cuda(), v.cuda())
        out += [(f"backward_input.{precision}.out", _digest(y)), (f"backward_input.{precision}.dx", _digest(dx))]
        net.release_engine()
    g = torch.Generator().manual_seed(5)
    B, R, Cin, Cout = 2, 16, 64, 64
    for precision in ("bf16", "bf16x3"):
        x = ops.to_ndhwc(torch.randn(B, Cin, R, R, R, generator=g).cuda(), precision)
        dy = ops.to_ndhwc(torch.randn(B, Cout, R, R, R, generator=g).cuda(), precision)
        w = (torch.randn(Cout, Cin, 3, 3, 3, generator=g) * 0.05).cuda()
        dw, dxc = ops.conv3d_backward(dy, x, w, precision=precision)
        out += [(f"conv3d_backward.{precision}.dw", _digest(dw)), (f"conv3d_backward.{precision}.dx", _digest(dxc))]
        w1 = (torch.randn(Cin, Cin, 1, 1, 1, generator=g) * 0.1).cuda()
        h, stats = ops.conv3d(x, w1, want_stats=True, precision=precision)
        gamma = (1 + 0.1 * torch.randn(Cin, generator=g)).cuda()
        beta = (0.1 * torch.randn(Cin, generator=g)).cuda()
        da = ops.to_ndhwc(torch.randn(B, Cin, R, R, R, generator=g).cuda(), precision)
        add = ops.to_ndhwc(torch.randn(B, Cin, R, R, R, generator=g).cuda(), precision)
        dxg, dg, db = ops.groupnorm_act_backward(h, stats, gamma, beta, da, add=add, silu=True, dropout_p=0.1, seed=77,
                                                 precision=precision)
        out += [(f"groupnorm_act_backward.{precision}.{k}", _digest(t)) for k, t in (("dx", dxg), ("dgamma", dg), ("dbeta", db))]
    torch.cuda.synchronize()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", default=None, help="also write the list to this file")
    args = ap.parse_args()
    lines = [f"{name} {h}" for name, h in digests()]
    print("\n".join(lines))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
