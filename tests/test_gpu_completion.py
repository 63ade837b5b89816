"""Shape completion on the GPU: `mdb_chamfer_pairs` (bitwise the Chamfer matrix's entries, the oracle's one-sided means
and maxima at unaligned sizes, reproducible, independent of the other pairs, refusals), the partial point cloud, the
per-sample routing of a packed conditional batch, the batching invariance of a partial's metrics, and
`main_diffusion.py --mode=make_partial` then `--mode=eval_completion` end to end (rerun identity, a two-rank split, the
`pc` path and `--mode=export` on the completions)."""
import glob
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, full_config
from oracle import completion_oracle as co

pytestmark = pytest.mark.gpu


def _clouds(n, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(n, N, 3, device="cuda", generator=g) - 0.5


def _pairs(clouds, pairs):
    from meshdiffusion_b200.geometry.pointcloud import chamfer_pairs
    out = chamfer_pairs(clouds, pairs)
    torch.cuda.synchronize()
    return [t.cpu() for t in out]


# ---- mdb_chamfer_pairs -------------------------------------------------------------------------------------------
def test_pairs_cd_bitwise_equal_to_the_matrix():
    from meshdiffusion_b200.geometry.pointcloud import chamfer_matrix
    x = _clouds(6, 2048, 0)
    pairs = [(a, b) for a in range(6) for b in range(6) if a != b]
    cd, _, _ = _pairs(x, pairs)
    cross = chamfer_matrix(x, x).cpu()
    self_m = chamfer_matrix(x).cpu()
    for p, (a, b) in enumerate(pairs):
        assert cd[p].item() == cross[a, b].item() == self_m[a, b].item(), (a, b)


@pytest.mark.parametrize("N", [1, 777, 2048])
def test_pairs_against_the_oracle(N):
    x = _clouds(4, N, N)
    pairs = [(0, 1), (1, 0), (2, 3), (3, 0)]
    cd, mean_ab, max_ab = _pairs(x, pairs)
    xs = x.cpu().numpy()
    for p, (a, b) in enumerate(pairs):
        want = co.pair_distances(xs[a], xs[b])
        assert math.isclose(cd[p].item(), want[0], rel_tol=2e-5), (p, cd[p], want)
        assert math.isclose(mean_ab[p].item(), want[1], rel_tol=2e-5), (p, mean_ab[p], want)
        assert math.isclose(max_ab[p].item(), want[2], rel_tol=2e-5), (p, max_ab[p], want)
        assert mean_ab[p].item() <= max_ab[p].item() * (1 + 1e-6)


def test_pairs_reproducible_and_independent_of_the_launch():
    x = _clouds(12, 1500, 5)
    base = [(0, 1), (4, 2), (7, 11)]
    first = _pairs(x, base)
    again = _pairs(x, base)
    rng = np.random.default_rng(0)
    more = [(int(a), int(b)) for a, b in rng.integers(0, 12, (300, 2)) if a != b]
    assert len(more) > 200
    big = more[:100] + [base[2]] + more[100:200] + [base[0], base[1]] + more[200:]
    out = _pairs(x, big)
    for t in range(3):
        assert torch.equal(first[t], again[t])
        for i, w in enumerate((201, 202, 100)):
            assert big[w] == base[i] and first[t][i].item() == out[t][w].item()


def test_pairs_refusals():
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.geometry.pointcloud import chamfer_pairs
    x = _clouds(3, 64, 1)
    with pytest.raises(ValueError, match="itself"):
        chamfer_pairs(x, [(0, 1), (2, 2)])
    with pytest.raises(ValueError, match="outside"):
        chamfer_pairs(x, [(0, 3)])
    with pytest.raises(ValueError, match="outside"):
        chamfer_pairs(x, [(-1, 0)])
    assert all(t.numel() == 0 for t in chamfer_pairs(x, []))
    L = _native.lib()
    pairs = torch.tensor([[0, 1], [1, 1], [0, 5]], dtype=torch.int32, device="cuda")
    cd = torch.zeros(3, dtype=torch.float64, device="cuda")
    mean_ab = torch.zeros_like(cd)
    max_ab = torch.zeros(3, device="cuda")
    args = (_native.ptr(pairs), 3, _native.ptr(cd), _native.ptr(mean_ab), _native.ptr(max_ab), _native.current_stream())
    assert L.mdb_chamfer_pairs(_native.ptr(x), 1, 64, *args) != 0 and b"two distinct" in L.mdb_last_error()
    assert L.mdb_chamfer_pairs(_native.ptr(x), 3, 0, *args) != 0
    assert L.mdb_chamfer_pairs(_native.ptr(x), 3, 64, _native.ptr(pairs), -1, *args[2:]) != 0
    assert L.mdb_chamfer_pairs(_native.ptr(x), 3, 1 << 20, *args) != 0 and b"shared memory" in L.mdb_last_error()
    # a caller that skips the host check gets NaN for the bad pairs, and the good pair is unaffected
    _native.check(L.mdb_chamfer_pairs(_native.ptr(x), 3, 64, *args))
    torch.cuda.synchronize()
    good = _pairs(x, [(0, 1)])
    assert cd[0].item() == good[0][0].item() and max_ab[0].item() == good[2][0].item()
    assert all(math.isnan(t[i].item()) for t in (cd, mean_ab, max_ab) for i in (1, 2))


# ---- the partial cloud -------------------------------------------------------------------------------------------
def _sphere_grid(R, radius, center=(0.0, 0.0, 0.0)):
    """[1, 4, R, R, R]: channel 0 = +1 inside the sphere, -1 outside, at the tet vertices; no deformation."""
    from meshdiffusion_b200.geometry import dmtet
    verts, _ = dmtet.load_tet_grid(R)
    v = torch.tensor(verts)
    c = dmtet.grid_coords_of_tet_vertices(v)
    g = torch.zeros(1, 4, R, R, R)
    inside = (v - torch.tensor(center)).norm(dim=1) < radius
    g[0, 0, c[:, 0], c[:, 1], c[:, 2]] = torch.where(inside, 1.0, -1.0)
    return g.cuda()


def _camera_position(view):
    from meshdiffusion_b200.geometry import singleview as sv
    ang = (view / sv.VIEWS_PER_TURN) * np.pi * 2
    mv = sv._translate(0, 0, -sv.RADIUS) @ (sv._rotate_x(-0.4) @ sv._rotate_y(ang))
    return torch.linalg.inv(mv.double())[:3, 3]


def test_partial_cloud_lies_on_visible_faces_facing_the_camera():
    from meshdiffusion_b200.diffusion import completion
    from meshdiffusion_b200.geometry import singleview
    R, res, view = 64, 256, 7
    mvp = singleview.view_mvp(view, res)
    packed = completion.extract_meshes(_sphere_grid(R, 0.35, (0.05, 0.0, -0.03)), R, 1.1, 3.0)
    v, f = completion.mesh(packed, 0)
    seen = completion.visible_faces(v, f, mvp.tolist(), res)
    _, face_id = singleview.rasterize([(v, f)], mvp.reshape(1, 4, 4), res)
    assert seen.cpu().tolist() == co.visible_face_ids(face_id.cpu().numpy())
    assert 0 < seen.numel() < f.shape[0]
    # convex: every face the view sees faces the camera (its outward normal points to the eye)
    tri = v[f[seen]].double().cpu()
    centroid = tri.mean(1)
    n = torch.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0], dim=1)
    n = n * torch.sign((n * (centroid - centroid.new_tensor([0.05, 0.0, -0.03]) * 1.1)).sum(1, keepdim=True))
    to_eye = _camera_position(view)[None] - centroid
    cos = (n * to_eye).sum(1) / (n.norm(dim=1) * to_eye.norm(dim=1))
    assert float(cos.min()) > -0.05 and float((cos > 0).double().mean()) > 0.99, float(cos.min())
    # every point of the partial cloud lies on a visible face
    pts, empty = completion.sample_meshes([(v, f[seen])], 2048, 42, completion.ID_STRIDE)
    assert not bool(empty[0])
    p = pts[0].double().cpu()
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    e0, e1 = b - a, c - a
    d = p[:, None, :] - a[None]
    d00, d01, d11 = (e0 * e0).sum(1), (e0 * e1).sum(1), (e1 * e1).sum(1)
    d20, d21 = (d * e0[None]).sum(2), (d * e1[None]).sum(2)
    den = d00 * d11 - d01 * d01
    s, t = (d11 * d20 - d01 * d21) / den, (d00 * d21 - d01 * d20) / den
    off = (d - s[..., None] * e0[None] - t[..., None] * e1[None]).norm(dim=2)
    on = (s >= -1e-4) & (t >= -1e-4) & (s + t <= 1 + 1e-4) & (off < 1e-5)
    assert bool(on.any(1).all())


# ---- routing through a packed batch ------------------------------------------------------------------------------
def _synthetic_partials(R):
    from meshdiffusion_b200.geometry import dmtet
    v = torch.tensor(dmtet.load_tet_grid(R)[0])
    r = v.norm(dim=1)
    a = {"sdf": torch.where(r < 0.3, 1.0, -1.0), "vis": (v[:, 2] > 0).float()}
    b = {"sdf": torch.where(r < 0.3, -1.0, 1.0), "vis": (v[:, 0] > 0).float()}
    return a, b


def test_packed_batch_routes_each_partial_to_its_own_slots():
    from meshdiffusion_b200.diffusion import completion, sampling, sde_lib
    from meshdiffusion_b200.diffusion.evaler import load_grid_mask, tet_grid_coords
    from meshdiffusion_b200.diffusion.models import utils as mutils
    from meshdiffusion_b200.geometry import dmtet
    cfg = full_config("res64", "bf16")
    cfg.device = torch.device("cuda")
    # K = 25: the last conditioned labels have alpha / sigma >= 44, so the re-noised visible values keep their sign
    cfg.sampling.method, cfg.sampling.dpm_steps = "dpm_solver", 25
    R, k = 64, 2
    torch.manual_seed(0)
    model = mutils.create_model(cfg)
    model.eval()
    net = model.module
    head = max(int(n.split(".")[1]) for n, _ in net.named_parameters() if n.startswith("all_modules."))
    with torch.no_grad():
        for n, p in net.named_parameters():
            if n.startswith(f"all_modules.{head}."):
                p.zero_()
    x = torch.randn(4, 4, R, R, R, device="cuda")
    with torch.no_grad():
        eps = model(x, torch.full((4,), 500.0, device="cuda"))
    assert bool((eps == 0).all()), "zeroing the last convolution must make the engine's output exactly 0"
    sde = sde_lib.VPSDE(cfg.model.beta_min, cfg.model.beta_max, cfg.model.num_scales, device="cuda")
    mask = load_grid_mask(R, "cuda").view(1, 1, R, R, R)
    fn = sampling.get_sampling_fn(cfg, sde, (4, 4, R, R, R), lambda t: t, 1e-3, grid_mask=mask)
    coords = tet_grid_coords(dmtet.tet_grid_path(R), "cuda")
    a, b = _synthetic_partials(R)
    samples, _ = completion.complete(fn, model, [a, b], coords, R, k, "dpm_solver", sde.N + 10)
    own = [completion.sign_agreement(samples[i * k:(i + 1) * k], p["sdf"], p["vis"], coords) for i, p in enumerate((a, b))]
    other = [completion.sign_agreement(samples[i * k:(i + 1) * k], p["sdf"], p["vis"], coords) for i, p in enumerate((b, a))]
    assert own == [[1.0, 1.0], [1.0, 1.0]], own
    assert all(s < 1.0 for row in other for s in row), other
    # the oracle's loop agrees on one slot
    ch0 = samples[0, 0, coords[:, 0], coords[:, 1], coords[:, 2]].cpu().numpy()
    assert co.sign_agreement(ch0, b["sdf"].numpy(), b["vis"].numpy()) == pytest.approx(other[0][0], abs=1e-12)


# ---- metrics -----------------------------------------------------------------------------------------------------
def test_metrics_of_a_partial_do_not_depend_on_its_group():
    from meshdiffusion_b200.diffusion import completion
    k, N = 3, 700
    gt, part, comp = _clouds(3, N, 11), _clouds(3, N, 12) * 0.5, _clouds(9, N, 13)
    comp[4] = float("nan")  # partial 1's second completion is empty
    empty = [False] * 9
    empty[4] = True
    group = completion.group_metrics(gt, part, comp, empty, [True, True, True], k)
    alone = completion.group_metrics(gt[1:2], part[1:2], comp[3:6], empty[3:6], [True], k)
    assert json.dumps(group[1]) == json.dumps(alone[0])
    assert group[1]["empty"] == 1 and math.isnan(group[1]["uhd"][1])
    # against the oracle's loops
    r = group[0]
    c = comp[0:3].cpu().numpy()
    g, p = gt[0].cpu().numpy(), part[0].cpu().numpy()
    lo, mean = co.accuracy(list(c), g)
    assert r["cd_gt_min"] == pytest.approx(lo, rel=2e-5) and r["cd_gt_mean"] == pytest.approx(mean, rel=2e-5)
    assert r["tmd"] == pytest.approx(co.tmd(list(c)), rel=2e-5)
    for j in range(k):
        assert r["uhd"][j] == pytest.approx(co.uhd(p, c[j]), rel=2e-5)
        assert r["p2c"][j] == pytest.approx(co.pair_distances(p, c[j])[1], rel=2e-5)
    skipped = completion.group_metrics(gt, part, comp, empty, [True, False, True], k)
    assert skipped[1] is None and json.dumps(skipped[2]) == json.dumps(group[2])


# ---- end to end --------------------------------------------------------------------------------------------------
def _run(args, cwd, env=None):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main_diffusion.py")] + args, cwd=cwd, capture_output=True,
                       text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return r


def _without_timings(m):
    m = dict(m)
    m.pop("seconds")
    return m


def test_make_partial_then_eval_completion_cli(tmp_path):
    from meshdiffusion_b200.diffusion.trainer import synthetic_grids
    from meshdiffusion_b200.geometry import dmtet
    grids = synthetic_grids(3, 64, torch.device("cuda"), generator=torch.Generator(device="cuda").manual_seed(2)).cpu()
    paths = []
    for i in range(3):
        p = os.path.join(tmp_path, f"grid_{100 + i}.pt")
        torch.save(grids[i].clone(), p)
        paths.append(p)
    meta = os.path.join(tmp_path, "meta.json")
    with open(meta, "w") as fh:
        json.dump(paths, fh)
    ev = os.path.join(tmp_path, "eval")
    base = [f"--config={ROOT}/configs/res64.py", f"--config.data.meta_path={meta}"]
    _run(base + ["--mode=make_partial", f"--config.eval.eval_dir={ev}", "--config.eval.partial_views=(0, 17)",
                 "--config.eval.partial_res=256"], cwd=str(tmp_path))
    common = base + ["--mode=eval_completion", f"--config.eval.ckpt_path={tmp_path}/missing/checkpoint.pth",
                     f"--config.eval.tet_path={dmtet.tet_grid_path(64)}", "--config.eval.completion_k=2",
                     "--config.eval.metric_points=512", "--config.model.compute_dtype=bf16"]
    dpm = ["--config.sampling.method=dpm_solver", "--config.sampling.dpm_steps=3", "--config.eval.batch_size=4"]

    def completion_run(name, extra, env=None):
        out = os.path.join(tmp_path, name)
        _run(common + [f"--config.eval.eval_dir={out}", f"--config.eval.partial_dir={ev}/partial"] + extra,
             cwd=str(tmp_path), env=env)
        return os.path.join(out, "completion")

    d = completion_run("a", dpm)
    names = [f"{i:06d}_view{v:02d}" for i in range(3) for v in (0, 17)]
    assert sorted(os.listdir(d)) == sorted([n + ".npy" for n in names] + ["metrics.json"])
    with open(os.path.join(d, "metrics.json")) as fh:
        m = json.load(fh)
    s = m["settings"]
    assert s["k"] == 2 and s["sampler"] == "dpm_solver" and s["dpm_steps"] == 3 and s["metric_points"] == 512
    assert s["deform_scale"] == 3.0 and s["compute_dtype"] == "bf16" and s["world_size"] == 1
    assert set(m["seconds"]) == {"sampling", "meshing", "distances", "writing"}
    assert [r["file"] for r in m["partials"]] == [n + ".pt" for n in names]
    for r in m["partials"]:
        x = np.load(os.path.join(d, r["file"][:-3] + ".npy"))
        assert x.shape == (2, 4, 64, 64, 64) and x.dtype == np.float32 and np.isfinite(x).all()
        assert r["visible_faces"] > 0 and r["source"] == paths[r["shape"]]
        for key in ("cd_gt_min", "cd_gt_mean", "tmd", "uhd_mean", "p2c_mean", "sign_agreement_mean"):
            assert r[key] is not None and math.isfinite(r[key]), (r["file"], key)
        assert len(r["cd_gt"]) == len(r["uhd"]) == len(r["sign_agreement"]) == 2
    assert m["means"]["scored"] == 6 and all(math.isfinite(m["means"][k]) for k in ("cd_gt_min", "tmd", "uhd_mean"))

    # a rerun writes the same bytes and the same report apart from the timings
    d2 = completion_run("b", dpm)
    for n in names:
        with open(os.path.join(d, n + ".npy"), "rb") as f1, open(os.path.join(d2, n + ".npy"), "rb") as f2:
            assert f1.read() == f2.read(), n
    with open(os.path.join(d2, "metrics.json")) as fh:
        m2 = json.load(fh)
    assert _without_timings(m2) == _without_timings(m)

    # two ranks cover every partial exactly once
    covered = []
    for rank in (0, 1):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK="0")
        dr = completion_run("ranks", dpm, env)
        with open(os.path.join(dr, f"metrics_{rank}.json")) as fh:
            covered += [r["index"] for r in json.load(fh)["partials"]]
    assert sorted(covered) == list(range(6))
    assert sorted(f for f in os.listdir(dr) if f.endswith(".npy")) == sorted(n + ".npy" for n in names)

    # the pc sampler, one partial per call, on a truncated schedule
    dp = completion_run("pc", ["--config.sampling.method=pc", "--config.eval.batch_size=2", "--config.sampling.max_iters=3",
                               "--config.eval.freeze_iters=2"])
    with open(os.path.join(dp, "metrics.json")) as fh:
        mp = json.load(fh)
    assert mp["settings"]["sampler"] == "pc" and len(mp["partials"]) == 6
    assert all(np.load(os.path.join(dp, n + ".npy")).shape == (2, 4, 64, 64, 64) for n in names)

    # export meshes and renders the completions
    _run([f"--config={ROOT}/configs/res64.py", "--mode=export", f"--config.eval.eval_dir={d}", "--config.render.res=64",
          "--config.render.ssaa=1"], cwd=str(tmp_path))
    meshes = sorted(os.listdir(os.path.join(d, "export", "mesh")))
    assert meshes == sorted(f"{n}_{i:06d}.obj" for n in names for i in range(2))
    assert glob.glob(os.path.join(d, "export", "viz", "*.png"))
