"""Pins the oracle against the UNMODIFIED reference and writes the golden vectors under tests/golden/.

Run in the authoring container only (needs /root/reference; the GPU box never sees it):

    python oracle/make_golden.py

What it does, per piece of the hot path:
  1. imports the reference's own modules from /root/reference (with an `ml_collections` stand-in and
     `Tensor.cuda` neutralised -- sde_lib.py:189,192 hard-code .cuda()),
  2. runs reference and oracle on the same seeded inputs on CPU fp32 and ASSERTS they agree,
  3. stores inputs (or the seeds that generate them) + reference outputs as small fixtures.
The reference ships no tests / golden vectors for this path (SURVEY.md section 4), so these files are the pin.
"""
import io
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from meshdiffusion_b200.compat.install import ensure_ml_collections  # noqa: E402

ensure_ml_collections()
from oracle import unet_oracle, sampler_oracle, mt_oracle, synth  # noqa: E402



def savez_lzma(path, **arrays):
    """np.savez_compressed with LZMA instead of deflate (np.load reads both): keeps the larger fixtures under 1 MB."""
    import io
    import zipfile
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_LZMA) as zf:
        for k, v in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(v), allow_pickle=False)
            zf.writestr(k + ".npy", buf.getvalue())

def import_reference():
    sys.path.insert(0, REF)
    torch.Tensor.cuda = lambda self, *a, **k: self  # reference hard-codes .cuda() in table construction
    from lib.diffusion.models import ddpm_res64, ddpm_res128, utils as rutils  # noqa: F401
    from lib.diffusion import sde_lib as rsde, sampling as rsampling
    from configs import res64 as rcfg64, res128 as rcfg128
    return dict(ddpm_res64=ddpm_res64, ddpm_res128=ddpm_res128, rutils=rutils, rsde=rsde, rsampling=rsampling,
                rcfg64=rcfg64, rcfg128=rcfg128)


def ref_config(ref, name, tiny):
    cfg = (ref["rcfg128"] if name == "res128" else ref["rcfg64"]).get_config()
    if name == "res128":
        cfg.model.name = "ddpm_res128"  # the stock config names an unregistered model (SURVEY appendix D)
    if tiny:
        synth.apply_tiny(cfg, name)
    cfg.device = torch.device("cpu")
    return cfg


def build_ref_model(ref, cfg):
    cls = ref["rutils"].get_model(cfg.model.name)
    torch.manual_seed(0)
    return cls(cfg).eval()


def golden_param_tables(ref):
    out = {}
    for name in ("res64", "res128"):
        cfg = ref_config(ref, name, tiny=False)
        model = torch.nn.DataParallel(build_ref_model(ref, cfg))
        sd = model.state_dict()
        out[name] = dict(
            state_dict=[(k, list(v.shape), str(v.dtype)) for k, v in sd.items()],
            trainable=[n for n, p in model.named_parameters() if p.requires_grad],
        )
        print(name, len(sd), "state-dict entries;", sum(p.numel() for p in model.parameters() if p.requires_grad), "trainable")
        del model
    with open(os.path.join(GOLD, "param_tables.json"), "w") as f:
        json.dump(out, f)


def golden_unet_forward(ref):
    for name in ("res64", "res128"):
        cfg = ref_config(ref, name, tiny=True)
        model = build_ref_model(ref, cfg)
        sd = synth.synthetic_state_dict(model.state_dict(), seed=11)
        model.load_state_dict(sd)
        x, labels = synth.synthetic_inputs(cfg.data.image_size, batch=2, seed=12, mask=sd["mask"])
        with torch.no_grad():
            y_ref = model(x, labels)
            y_orc = unet_oracle.unet_forward(sd, unet_oracle.arch_from_config(cfg), x, labels)
        err = (y_ref - y_orc).abs().max().item()
        print(f"unet {name} tiny: |ref| max {y_ref.abs().max():.4f}, oracle-vs-reference max abs diff {err:.3e}")
        assert err <= 2e-5 * max(1.0, y_ref.abs().max().item()), "oracle U-Net disagrees with the reference"
        np.savez_compressed(os.path.join(GOLD, f"unet_tiny_{name}.npz"), out=y_ref.numpy(),
                            checksum=synth.state_checksum(sd), state_seed=11, input_seed=12)


def ddpm_loss(pred, noise, mask):
    """lib/diffusion/losses.py:69-78 (l2, masked)."""
    losses = torch.square(pred - noise) * mask
    losses = losses.reshape(losses.shape[0], -1).mean(dim=-1)
    return torch.mean(losses) / mask.sum() * np.prod(mask.size())


def grad_signature(name, g, seed=1234):
    """(L2 norm, 4 seeded random projections) of one gradient tensor -- a compact pin of the whole tensor."""
    gen = torch.Generator().manual_seed(seed + sum(ord(c) for c in name))
    r = torch.randn(4, g.numel(), generator=gen, dtype=torch.float64)
    gd = g.detach().double().reshape(-1)
    return np.concatenate([[gd.norm().item()], (r @ gd).numpy()])


def golden_unet_backward(ref):
    """Gradients of the reference modules (torch autograd, fp32 CPU) for the DDPM loss on seeded inputs; the oracle's
    autograd gradients must agree, and the per-tensor signatures are committed for the CPU and GPU parity tests."""
    for name in ("res64", "res128"):
        cfg = ref_config(ref, name, tiny=True)
        model = build_ref_model(ref, cfg)   # eval(): dropout is the identity, as in the 'dropout disabled' parity runs
        sd = synth.synthetic_state_dict(model.state_dict(), seed=21)
        model.load_state_dict(sd)
        R = cfg.data.image_size
        x, labels = synth.synthetic_inputs(R, batch=2, seed=31, mask=sd["mask"])
        noise = torch.randn(x.shape, generator=torch.Generator().manual_seed(5))
        mask = sd["mask"].view(1, 1, R, R, R)
        loss = ddpm_loss(model(x, labels), noise, mask)
        loss.backward()
        ref_g = {n: p.grad for n, p in model.named_parameters() if p.requires_grad and p.grad is not None}
        osd = {k: (v.clone().requires_grad_(True) if v.dtype == torch.float32 and k not in ("mask", "coords") else v) for k, v in sd.items()}
        oloss = ddpm_loss(unet_oracle.unet_forward(osd, unet_oracle.arch_from_config(cfg), x, labels), noise, mask)
        oloss.backward()
        tot = sum(g.double().pow(2).sum().item() for g in ref_g.values()) ** 0.5
        worst = 0.0
        for n, g in ref_g.items():
            worst = max(worst, (osd[n].grad - g).double().norm().item() / tot)
        print(f"unet {name} tiny backward: loss {loss.item():.6f} (oracle {oloss.item():.6f}), {len(ref_g)} gradient tensors, "
              f"|g| {tot:.4e}, worst oracle-vs-reference diff / |g| {worst:.3e}")
        assert abs(loss.item() - oloss.item()) < 1e-5 * abs(loss.item()) and worst < 1e-5, "oracle backward disagrees with the reference"
        names = sorted(ref_g)
        np.savez_compressed(os.path.join(GOLD, f"unet_tiny_{name}_grads.npz"), loss=loss.item(), names=np.array(names),
                            sig=np.stack([grad_signature(n, ref_g[n]) for n in names]), total_norm=tot,
                            state_seed=21, input_seed=31, noise_seed=5)


def golden_sampler(ref):
    import tqdm
    cfg = ref_config(ref, "res64", tiny=True)
    model = build_ref_model(ref, cfg)
    sd = synth.synthetic_state_dict(model.state_dict(), seed=21)
    model.load_state_dict(sd)
    R, B, n_it = cfg.data.image_size, 2, 4
    rsde, rsamp = ref["rsde"], ref["rsampling"]
    sde = rsde.VPSDE(beta_min=cfg.model.beta_min, beta_max=cfg.model.beta_max, N=cfg.model.num_scales)
    osde = sampler_oracle.VPSDETables(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales)
    for a, b in ((sde.discrete_betas, osde.discrete_betas), (sde.sqrt_1m_alphas_cumprod, osde.sqrt_1m_alphas_cumprod)):
        assert torch.equal(a, b), "VP-SDE tables differ"
    grid_mask = sd["mask"].view(1, R, R, R)
    real_trange = tqdm.trange
    rsamp.tqdm.trange = lambda n: range(min(n, n_it))  # first iterations of the N=1000 schedule (SURVEY 8c-5)
    try:
        sampler = rsamp.get_pc_sampler(sde, (B, 4, R, R, R), rsamp.get_predictor("ancestral_sampling"),
                                       rsamp.get_corrector("none"), lambda x: x, snr=cfg.sampling.snr, n_steps=1,
                                       probability_flow=False, continuous=False, denoise=True, eps=1e-3, device="cpu",
                                       grid_mask=grid_mask)
        torch.manual_seed(31)
        s_ref, _ = sampler(model)
        torch.manual_seed(31)
        fn = lambda x, t: unet_oracle.unet_forward(sd, unet_oracle.arch_from_config(cfg), x, t)
        s_orc = sampler_oracle.pc_sample_uncond(osde, fn, torch.randn(B, 4, R, R, R), grid_mask, torch.randn_like, n_iters=n_it)
        err = (s_ref - s_orc).abs().max().item()
        print(f"sampler uncond ({n_it} iters): oracle-vs-reference max abs diff {err:.3e}")
        assert err <= 1e-4
        # partial (conditional) branch
        g = torch.Generator().manual_seed(41)
        partial = torch.sign(torch.randn(B, 4, R, R, R, generator=g))
        pmask4 = (torch.rand(1, 1, R, R, R, generator=g) < 0.5).float().expand(B, 4, R, R, R).contiguous()
        gm5 = sd["mask"].view(1, 1, R, R, R)
        sampler5 = rsamp.get_pc_sampler(sde, (B, 4, R, R, R), rsamp.get_predictor("ancestral_sampling"),
                                        rsamp.get_corrector("none"), lambda x: x, snr=cfg.sampling.snr, n_steps=1,
                                        probability_flow=False, continuous=False, denoise=True, eps=1e-3, device="cpu",
                                        grid_mask=gm5)
        torch.manual_seed(32)
        c_ref, _ = sampler5(model, partial=partial, partial_mask=pmask4, freeze_iters=3)
        torch.manual_seed(32)
        c_orc = sampler_oracle.pc_sample_partial(osde, fn, torch.randn(B, 4, R, R, R), gm5, partial, pmask4,
                                                 torch.randn_like, freeze_iters=3, n_iters=n_it)
        cerr = (c_ref - c_orc).abs().max().item()
        print(f"sampler partial ({n_it} iters): oracle-vs-reference max abs diff {cerr:.3e}")
        assert cerr <= 1e-4
        # DDIM update (the reference's predictor works; only its sampler's return statement is broken)
        rscore = ref["rutils"].get_score_fn(sde, model, train=False, continuous=False, std_scale=False)
        g = torch.Generator().manual_seed(51)
        xd = torch.randn(B, 4, R, R, R, generator=g) * grid_mask
        td, tp = torch.full((B,), 0.64), torch.full((B,), 0.6084)
        with torch.no_grad():
            d_ref = sde.reverse(rscore, False).discretize_ddim(xd, td, tprev=tp)
            d_orc = sampler_oracle.ddim_update(osde, fn, xd, td, tp)
        derr = max((d_ref[0] - d_orc[0]).abs().max().item(), (d_ref[1] - d_orc[1]).abs().max().item())
        print(f"ddim update: oracle-vs-reference max abs diff {derr:.3e}")
        assert derr <= 1e-4
    finally:
        rsamp.tqdm.trange = real_trange
    np.savez_compressed(os.path.join(GOLD, "sampler_tiny.npz"), uncond=s_ref.numpy(), partial=c_ref.numpy(),
                        ddim_x=d_ref[0].numpy(), ddim_x0=d_ref[1].numpy(),
                        checksum=synth.state_checksum(sd), state_seed=21, n_iters=n_it,
                        betas=sde.discrete_betas.numpy(), sqrt_1m_ac=sde.sqrt_1m_alphas_cumprod.numpy())


def golden_sampler_variants(ref):
    """The other registered predictors / correctors (sampling.py:185-209, 259-321) and the `return_traj` x0-prediction
    branch (:410-420, 480-484) of the REFERENCE get_pc_sampler on the tiny network -> tests/golden/sampler_variants_tiny.npz.
    No oracle restatement exists for these: the fixtures are the reference's own outputs, which the GPU tests replay."""
    cfg = ref_config(ref, "res64", tiny=True)
    model = build_ref_model(ref, cfg)
    sd = synth.synthetic_state_dict(model.state_dict(), seed=21)
    model.load_state_dict(sd)
    R, B = cfg.data.image_size, 2
    rsde, rsamp = ref["rsde"], ref["rsampling"]
    sde = rsde.VPSDE(beta_min=cfg.model.beta_min, beta_max=cfg.model.beta_max, N=cfg.model.num_scales)
    grid_mask = sd["mask"].view(1, R, R, R)
    real_trange = rsamp.tqdm.trange
    out = {"state_seed": 21, "checksum": synth.state_checksum(sd), "snr": 0.16, "n_iters": 3, "traj_iters": 711}
    variants = [("euler_maruyama", "none"), ("reverse_diffusion", "none"), ("ancestral_sampling", "langevin"), ("reverse_diffusion", "ald")]
    try:
        for k, (pred, corr) in enumerate(variants):
            rsamp.tqdm.trange = lambda n: range(min(n, 3))
            sampler = rsamp.get_pc_sampler(sde, (B, 4, R, R, R), rsamp.get_predictor(pred), rsamp.get_corrector(corr), lambda x: x,
                                           snr=0.16, n_steps=1, probability_flow=False, continuous=False, denoise=True, eps=1e-3,
                                           device="cpu", grid_mask=grid_mask)
            torch.manual_seed(60 + k)
            s, _ = sampler(model)
            assert torch.isfinite(s).all()
            out[f"{pred}__{corr}"] = s.numpy()
            print(f"sampler variant {pred} + {corr}: |x| max {s.abs().max():.4f}")
        rsamp.tqdm.trange = lambda n: range(min(n, 711))
        sampler = rsamp.get_pc_sampler(sde, (B, 4, R, R, R), rsamp.get_predictor("ancestral_sampling"), rsamp.get_corrector("none"),
                                       lambda x: x, snr=0.16, n_steps=1, probability_flow=False, continuous=False, denoise=True,
                                       eps=1e-3, device="cpu", grid_mask=grid_mask, return_traj=True)
        torch.manual_seed(70)
        traj, _ = sampler(model)
        assert len(traj) == 2
        out["traj"] = torch.stack(traj).numpy()
        print(f"return_traj: {len(traj)} x0 predictions (iterations 700, 710), |x0| max {out['traj'].max():.4f}")
    finally:
        rsamp.tqdm.trange = real_trange
    np.savez_compressed(os.path.join(GOLD, "sampler_variants_tiny.npz"), **out)


def load_reference_mesh_ops():
    """auto_normals / compute_tangents from nvdiffrec/lib/render/mesh.py, exec'd from source (the module imports the
    renderer stack, which is absent); `Mesh` is replaced by a plain attribute bag and the device pin by 'cpu'."""
    import types
    src = open(os.path.join(REF, "nvdiffrec/lib/render/mesh.py")).read().split("\n")
    def grab(fn):
        start = next(i for i, l in enumerate(src) if l.startswith("def " + fn + "("))
        end = next((i for i in range(start + 1, len(src)) if src[i].startswith("def ") or src[i].startswith("####")), len(src))
        return "\n".join(src[start:end])
    usrc = open(os.path.join(REF, "nvdiffrec/lib/render/util.py")).read().split("\n")
    def grab_util(fn):
        start = next(i for i, l in enumerate(usrc) if l.startswith("def " + fn + "("))
        end = next(i for i in range(start + 1, len(usrc)) if usrc[i].startswith("def "))
        return "\n".join(usrc[start:end])
    util = types.SimpleNamespace()
    uns = {"torch": torch}
    exec(grab_util("dot") + "\n" + grab_util("length") + "\n" + grab_util("safe_normalize"), uns)
    util.dot, util.safe_normalize = uns["dot"], uns["safe_normalize"]

    class Mesh:
        def __init__(self, v_pos=None, t_pos_idx=None, v_nrm=None, t_nrm_idx=None, v_tex=None, t_tex_idx=None, v_tng=None,
                     t_tng_idx=None, f_nrm=None, base=None, **kw):
            for k in ("v_pos", "t_pos_idx", "v_nrm", "t_nrm_idx", "v_tex", "t_tex_idx", "v_tng", "t_tng_idx", "f_nrm"):
                val = locals()[k]
                setattr(self, k, val if val is not None else (getattr(base, k, None) if base is not None else None))

    ns = {"torch": torch, "util": util, "Mesh": Mesh}
    exec((grab("auto_normals") + "\n" + grab("compute_tangents")).replace("device='cuda'", "device='cpu'"), ns)
    return Mesh, ns["auto_normals"], ns["compute_tangents"]


def golden_mesh_ops():
    """Reference normals / tangents / OBJ text on a marching-tet mesh of the synthetic sphere; oracle must agree."""
    from oracle import mesh_oracle
    Mesh, ref_normals, ref_tangents = load_reference_mesh_ops()
    t = np.load(os.path.join(REF, "nvdiffrec/data/tets/64_tets_cropped.npz"))
    verts, idx = t["vertices"].astype(np.float32), t["indices"].astype(np.int64)
    sdf, pos = synth.synthetic_dmtet(verts, seed=3, noisy=False)  # smooth surface: every vertex normal is well conditioned
    v, f, uvs, uv_idx, _, _ = mt_oracle.marching_tets(pos, sdf, idx)
    m = Mesh(v_pos=torch.tensor(v), t_pos_idx=torch.tensor(f), v_tex=torch.tensor(uvs), t_tex_idx=torch.tensor(uv_idx))
    m = ref_normals(m)
    m2 = ref_tangents(m)
    on, ofn = mesh_oracle.auto_normals(v, f)
    ot = mesh_oracle.compute_tangents(v, f, uvs, uv_idx, on, f)
    en = np.abs(on - m.v_nrm.numpy()).max(); efn = np.abs(ofn - m.f_nrm.numpy()).max()
    # tangents: the per-face tangents of the marching-tet UV atlas point in unrelated directions, so a few vertex
    # averages nearly cancel and their direction is decided by fp32 rounding order (in the reference too): robust statistic
    terr = np.abs(ot - m2.v_tng.numpy()).max(1)
    et, frac = np.percentile(terr, 99), (terr > 1e-3).mean()
    print(f"mesh ops: {v.shape[0]} verts, {f.shape[0]} faces; oracle-vs-reference normals {en:.2e}, face normals {efn:.2e}, "
          f"tangents p99 {et:.2e} ({100 * frac:.2f} % ill-conditioned vertices)")
    assert en < 1e-5 and efn < 1e-9 and et < 1e-5 and frac < 0.01
    # OBJ text: the reference writer needs the material stack; its loop is restated literally in mesh_oracle.obj_text
    # (obj.py:165-216) and checked here on the first lines only against hand-formatted output of the same expressions.
    head = mesh_oracle.obj_text(v[:2], f[:1])
    assert head.startswith("g default\nv {} {} {} \n".format(v[0][0], v[0][1], v[0][2]))
    np.savez_compressed(os.path.join(GOLD, "mesh_ops_64.npz"), seed=3, v_nrm=m.v_nrm.numpy(), v_tng=m2.v_tng.numpy(),
                        f_nrm_sum=m.f_nrm.numpy().astype(np.float64).sum(0), n_verts=v.shape[0], n_faces=f.shape[0])


def load_reference_dmtet():
    """The DMTet class body (dmtet.py:32-163) depends only on torch/numpy; its module imports kaolin etc., so the
    class source is exec'd on its own with 'cuda' -> 'cpu'. Nothing from it is written into this repository."""
    src = open(os.path.join(REF, "nvdiffrec/lib/geometry/dmtet.py")).read().split("\n")
    start = next(i for i, l in enumerate(src) if l.startswith("class DMTet:"))
    end = next(i for i, l in enumerate(src) if l.startswith("def compute_sdf") or (i > start and l.startswith("class ")) or l.startswith("# Regularizer") or l.startswith("def ") and i > start)
    body = "\n".join(src[start:end]).replace("'cuda'", "'cpu'").replace('"cuda"', '"cpu"')
    ns = {"torch": torch, "np": np}
    exec(compile(body, "reference_dmtet", "exec"), ns)
    return ns["DMTet"]


def golden_marching_tets():
    DMTet = load_reference_dmtet()
    mt = DMTet()
    tets = np.load(os.path.join(REF, "nvdiffrec/data/tets/64_tets_cropped.npz"))
    verts, idx = tets["vertices"], tets["indices"]
    cases = {}
    for case, seed in (("sphere", 0), ("noisy", 1)):
        sdf, pos = synth.synthetic_dmtet(verts, seed=seed, noisy=(case == "noisy"))
        with torch.no_grad():
            r = mt(torch.tensor(pos), torch.tensor(sdf), torch.tensor(idx).long())
        r = [t.numpy() for t in r]
        o = mt_oracle.marching_tets(pos, sdf, idx)
        names = ["verts", "faces", "uvs", "uv_idx", "face_to_valid_tet", "valid_vert_idx"]
        for n, a, b in zip(names, r, o):
            assert a.shape == b.shape, (case, n, a.shape, b.shape)
            if a.dtype.kind in "iu":
                assert np.array_equal(a, b), f"marching tets {case}: integer output {n} differs"
            else:
                assert np.allclose(a, b, rtol=1e-6, atol=1e-7), f"marching tets {case}: {n} differs"
        print(f"marching tets {case}: {r[0].shape[0]} verts, {r[1].shape[0]} faces -- oracle == reference")
        cases[case + "_verts"] = r[0]
        cases[case + "_faces"] = r[1].astype(np.int32)
        cases[case + "_uv_idx"] = r[3].astype(np.int32)
        cases[case + "_face_to_valid_tet"] = r[4].astype(np.int32)
        cases[case + "_valid_vert_idx"] = r[5].astype(np.int32)
        cases[case + "_uvs_shape"] = np.array(r[2].shape)
        cases[case + "_uvs_head"] = r[2][:64]
        cases[case + "_uvs_tail"] = r[2][-64:]
        cases[case + "_uvs_sum"] = np.array([r[2].astype(np.float64).sum()])
    savez_lzma(os.path.join(GOLD, "marching_tets_64.npz"), **cases)
    golden_marching_tets_grad(mt, verts, idx)
    golden_marching_tets_128(mt)
    # grid mask derivable from the tet grid (data/get_tet_mask.py): check against the shipped mask
    coords = mt_oracle.grid_coords_of_tet_vertices(verts)
    mask = np.zeros((64, 64, 64), np.float32)
    mask[coords[:, 0], coords[:, 1], coords[:, 2]] = 1
    ref_mask = torch.load(os.path.join(REF, "data/grid_mask_64.pt"), map_location="cpu").numpy()
    assert np.array_equal(mask, ref_mask), "grid mask derived from the tet grid differs from data/grid_mask_64.pt"
    print("grid_mask_64 == scatter of tet vertices:", int(mask.sum()), "voxels")


def golden_marching_tets_grad(mt, verts, idx):
    """tests/golden/marching_tets_64_grad.npz: gradients of the REFERENCE DMTet's `verts` with respect to pos_nx3 and sdf_n
    (torch autograd through dmtet.py:125-132, L = sum(verts * W)); the numpy restatement must agree. The sdf of both cases is
    continuous here (the sign() of the sampling path has no gradient): sphere, and sphere + noise with deformed vertices."""
    cases = {}
    for case, seed in (("sphere", 0), ("noisy", 1)):
        sdf, pos = synth.synthetic_dmtet_grad_case(verts, seed=seed, noisy=(case == "noisy"))
        p = torch.tensor(pos, requires_grad=True)
        s = torch.tensor(sdf, requires_grad=True)
        v = mt(p, s, torch.tensor(idx).long())[0]
        W = synth.mt_grad_weights(v.shape[0], seed)
        (v * torch.tensor(W)).sum().backward()
        gp, gs = p.grad.numpy(), s.grad.numpy()
        op, os_ = mt_oracle.marching_tets_vertex_grad(pos, sdf, idx, W)
        sp, ss = np.abs(gp).max(), np.abs(gs).max()
        assert np.abs(gp - op).max() <= 1e-5 * sp and np.abs(gs - os_).max() <= 1e-5 * ss, (case, np.abs(gp - op).max() / sp, np.abs(gs - os_).max() / ss)
        print(f"marching tets grad {case}: {v.shape[0]} verts, |dpos| max {sp:.3g}, |dsdf| max {ss:.3g} -- oracle == reference autograd")
        nzp, nzs = np.flatnonzero(np.abs(gp).sum(1)), np.flatnonzero(gs)
        cases[case + "_n_verts"] = np.array([v.shape[0]])
        cases[case + "_pos_rows"] = nzp.astype(np.int32)
        cases[case + "_grad_pos"] = gp[nzp]
        cases[case + "_sdf_rows"] = nzs.astype(np.int32)
        cases[case + "_grad_sdf"] = gs[nzs]
    np.savez_compressed(os.path.join(GOLD, "marching_tets_64_grad.npz"), **cases)


def golden_dataset_items():
    """tests/golden/dataset_items.npz: items of the REFERENCE ShapeNetDMTetDataset (lib/dataset/shapenet_dmtet_dataset.py:8-54)
    on four synthetic 7^3 shapes under an 8^3 grid mask with a 3-id filter list -- `aug=False` then `aug=True` (global RNG
    seeded with 100 + index before each item, which fixes the jitter draw). The inputs (`raw`, `mask`, `filter`) are part of
    the fixture: when the file exists they are re-used and the regenerated items must equal the committed ones bit for bit;
    otherwise they are drawn from seed 7."""
    import importlib.util
    import tempfile
    spec = importlib.util.spec_from_file_location("ref_dataset", os.path.join(REF, "lib/dataset/shapenet_dmtet_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    path = os.path.join(GOLD, "dataset_items.npz")
    old = np.load(path) if os.path.exists(path) else None
    if old is not None:
        raw, mask, filt = old["raw"], old["mask"], old["filter"]
    else:
        g = torch.Generator().manual_seed(7)
        raw = (torch.randn(4, 4, 7, 7, 7, generator=g) * (torch.rand(4, 4, 7, 7, 7, generator=g) < 0.6)).numpy().astype(np.float32)
        mask = (torch.rand(1, 1, 8, 8, 8, generator=g) < 0.7).float().numpy()
        filt = np.array([0, 2, 3], np.int64)
    items = []
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i, r in enumerate(raw):
            p = os.path.join(tmp, f"shape_{i}.pt")
            torch.save(torch.tensor(r), p)
            paths.append(p)
        meta, fpath = os.path.join(tmp, "meta.json"), os.path.join(tmp, "filter.json")
        json.dump(paths, open(meta, "w"))
        json.dump([int(v) for v in filt], open(fpath, "w"))
        for aug in (False, True):
            ds = mod.ShapeNetDMTetDataset(meta, torch.tensor(mask), deform_scale=3.0, aug=aug, filter_meta_path=fpath,
                                          normalize_sdf=True, extension="pt")
            assert len(ds) == len(filt)
            for i in range(len(ds)):
                torch.manual_seed(100 + i)
                items.append(ds[i].numpy())
    items = np.stack(items)
    if old is not None:
        assert np.array_equal(items, old["items"]), "reference dataset items differ from the committed golden"
        print(f"dataset items: {items.shape[0]} items of the reference class == committed golden (bit-identical)")
        return
    np.savez_compressed(path, raw=raw, mask=mask, items=items, filter=filt)
    print("dataset items written:", items.shape)


def int_digest(a):
    """sha256 of an integer array as little-endian int64 -- pins every entry without storing 10^5 of them."""
    import hashlib
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, dtype="<i8").tobytes()).digest(), dtype=np.uint8)


def golden_marching_tets_128(mt):
    """R=128 tet grid (nvdiffrec/data/tets/128_tets_cropped.npz: 253 024 vertices, 1 387 746 tets): the reference DMTet's
    integer outputs are pinned by length + sha256 digests (bit-exactness is a hash equality), the float outputs by sampled
    entries and sums; the oracle must agree with the reference entry by entry first."""
    tets = np.load(os.path.join(REF, "nvdiffrec/data/tets/128_tets_cropped.npz"))
    verts, idx = tets["vertices"], tets["indices"]
    cases = {}
    for case, seed in (("sphere", 0), ("noisy", 1)):
        sdf, pos = synth.synthetic_dmtet(verts, seed=seed, noisy=(case == "noisy"), res=128)
        with torch.no_grad():
            r = [t.numpy() for t in mt(torch.tensor(pos), torch.tensor(sdf), torch.tensor(idx).long())]
        o = mt_oracle.marching_tets(pos, sdf, idx)
        names = ["verts", "faces", "uvs", "uv_idx", "face_to_valid_tet", "valid_vert_idx"]
        for n, a, b in zip(names, r, o):
            assert a.shape == b.shape, (case, n, a.shape, b.shape)
            if a.dtype.kind in "iu":
                assert np.array_equal(a, b), f"marching tets 128 {case}: integer output {n} differs"
            else:
                assert np.allclose(a, b, rtol=1e-6, atol=1e-7), f"marching tets 128 {case}: {n} differs"
        print(f"marching tets 128 {case}: {r[0].shape[0]} verts, {r[1].shape[0]} faces -- oracle == reference")
        for n, a in zip(names, r):
            cases[f"{case}_{n}_shape"] = np.array(a.shape)
            if a.dtype.kind in "iu":
                cases[f"{case}_{n}_sha256"] = int_digest(a)
            else:
                sel = np.linspace(0, a.shape[0] - 1, 257).astype(np.int64)
                cases[f"{case}_{n}_rows"] = sel
                cases[f"{case}_{n}_sample"] = a[sel]
                cases[f"{case}_{n}_sum"] = np.array([a.astype(np.float64).sum()])
    np.savez_compressed(os.path.join(GOLD, "marching_tets_128.npz"), **cases)
    coords = mt_oracle.grid_coords_of_tet_vertices(verts)
    mask = np.zeros((128, 128, 128), np.float32)
    mask[coords[:, 0], coords[:, 1], coords[:, 2]] = 1
    ref_mask = torch.load(os.path.join(REF, "data/grid_mask_128.pt"), map_location="cpu").numpy()
    assert np.array_equal(mask, ref_mask), "grid mask derived from the 128 tet grid differs from data/grid_mask_128.pt"
    print("grid_mask_128 == scatter of tet vertices:", int(mask.sum()), "voxels")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    ref = import_reference()
    golden_dataset_items()
    golden_marching_tets()
    golden_mesh_ops()
    golden_unet_forward(ref)
    golden_unet_backward(ref)
    golden_sampler(ref)
    golden_sampler_variants(ref)
    golden_param_tables(ref)
    print("golden vectors written to", GOLD)
