"""CPU: shape editing (`--mode=edit`) -- the RePaint entry table, the eager update against a float64 restatement, the box ->
kept-region mapping on the shipped tet grids, the argument checks, and an analytic gate: a stationary correlated Gaussian
whose exact conditional distribution of the regenerated voxels given the kept ones is known."""
import math

import numpy as np
import pytest
import torch

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from meshdiffusion_b200.diffusion import edit, sampling, sde_lib


def _sde():
    return sde_lib.VPSDE(0.1, 20.0, 1000, device="cpu")


def _alpha_sigma(sde):
    abar = sde.alphas_cumprod.double().numpy()
    return np.sqrt(abar), np.sqrt(1.0 - abar)


# ---- the entry table ---------------------------------------------------------------------------------------------
CASES = [(25, 5, 3, False), (25, 5, 3, True), (20, 2, 4, False), (10, 3, 3, True), (7, 7, 5, False), (12, 1, 2, True)]


@pytest.mark.parametrize("K,J,U,sto", CASES)
def test_schedule_structure(K, J, U, sto):
    sde = _sde()
    labels, dpm = sampling.dpm_solver_schedule(sde, K, sto)
    table, nfe = sampling.repaint_schedule(sde, K, J, U, sto)
    Ke = len(labels) - 1
    kind = table[:, 0]
    den = table[kind == 0]
    # labels: the first entry runs at N - 1, the last lands at 0 with the exact replacement pair
    assert table[0, 1] == sde.N - 1 and kind[0] == 0 and kind[-1] == 0
    assert table[-1, 1] == labels[-2] and tuple(table[-1, 8:]) == (1.0, 0.0)
    last = Ke - ((Ke - 1) // J) * J  # steps in the last block, which runs once
    assert nfe == len(den) == Ke + (U - 1) * (Ke - last)
    assert (kind == 1).sum() == (U - 1) * ((Ke - 1) // J)
    # every block's runs repeat the solver's labels; the first denoise entry after a renoise is first order
    k_of = {labels[k]: k for k in range(Ke)}
    for e in np.nonzero(kind == 1)[0]:
        nxt = table[e + 1]
        assert nxt[0] == 0 and nxt[1] == table[e, 1] and nxt[6] == 0.0
        k = k_of[int(nxt[1])]
        assert nxt[4] == dpm[k, 3] and nxt[7] == dpm[k, 6] and tuple(nxt[8:]) == tuple(dpm[k, 7:])
        if k > 0:  # the first-order weight: c_0 = b with b the second-order row's c_0 + c_1
            assert nxt[5] == pytest.approx(dpm[k, 4] + dpm[k, 5], rel=1e-12)
    assert sorted({int(v) for v in den[:, 1]}, reverse=True) == labels[:-1]


@pytest.mark.parametrize("K,sto", [(25, False), (25, True), (13, True)])
def test_resample_one_is_the_solver_table(K, sto):
    sde = _sde()
    _, dpm = sampling.dpm_solver_schedule(sde, K, sto)
    table, nfe = sampling.repaint_schedule(sde, K, 4, 1, sto)
    assert nfe == dpm.shape[0] and np.all(table[:, 0] == 0)
    assert np.array_equal(table[:-1, 1:], dpm[:-1]), "resample = 1 must be the solver's rows bit for bit"
    assert np.array_equal(table[-1, 1:8], dpm[-1, :7])


def test_renoise_coefficients():
    sde = _sde()
    alpha, sigma = _alpha_sigma(sde)
    labels, _ = sampling.dpm_solver_schedule(sde, 25)
    table, _ = sampling.repaint_schedule(sde, 25, 5, 3)
    for e in np.nonzero(table[:, 0] == 1)[0]:
        hi = int(table[e, 1])
        k0 = labels.index(hi)
        lo = labels[k0 + 5]
        assert int(table[e - 1, 1]) == labels[k0 + 4]  # the block's last step lands at lo
        a = alpha[hi] / alpha[lo]
        assert table[e, 4] == a and table[e, 7] == np.sqrt(1.0 - a * a)
        assert tuple(table[e, [2, 3, 5, 6]]) == (0.0, 0.0, 0.0, 0.0)
        assert tuple(table[e, 8:]) == (alpha[hi], sigma[hi])


def test_schedule_refusals():
    sde = _sde()
    for J, U in ((0, 3), (5, 0), (2.5, 2), (True, 2)):
        with pytest.raises(ValueError):
            sampling.repaint_schedule(sde, 10, J, U)


# ---- the eager update --------------------------------------------------------------------------------------------
def _f32(v):
    return np.float32(v)


def _restated(x, eps, hist, g, row, z, known, m, chans, z2):
    """The entry in float64 numpy with every operation rounded to float32 on its own."""
    kind, _, sg, inv_a, c_x, c_0, c_1, c_z, coef, std = (np.float64(_f32(v)) for v in row)
    r = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    x, eps, hist, z, z2 = (t.double().numpy() for t in (x, eps, hist, z, z2))
    h = hist
    if kind:
        xn = r(r(r(x * c_x) + r(z * c_z)) * g)
    else:
        x0 = r(r(x - r(eps * sg)) * inv_a)
        xn = r(r(x * c_x) + r(x0 * c_0))
        if c_1 != 0:
            xn = r(xn + r(hist * c_1))
        if c_z != 0:
            xn = r(xn + r(z * c_z))
        xn = r(xn * g)
        h = x0
    for c in chans:
        s = r(r(known[:, c] * coef) + r(z2[:, c] * std))
        xn[:, c] = r(r(r(xn[:, c] * r(1.0 - m)) + r(s * m)) * g)
    return xn, h


@pytest.mark.parametrize("entry", ["first_order", "second_order_sde", "renoise", "last"])
def test_eager_entry_against_float64_restatement(entry):
    sde = _sde()
    table, _ = sampling.repaint_schedule(sde, 10, 3, 3, stochastic=True)
    e = {"first_order": 0, "second_order_sde": 1, "renoise": 3, "last": len(table) - 1}[entry]
    assert (table[e, 0] == 1) == (entry == "renoise")
    row = table[e].astype(np.float32)
    gen = torch.Generator().manual_seed(3 + e)
    B, C, R = 3, 4, 6
    x, eps, hist, z, z2 = (torch.randn(B, C, R, R, R, generator=gen) for _ in range(5))
    g = (torch.rand(R, R, R, generator=gen) < 0.7).float()
    known = torch.randn(B, C, R, R, R, generator=gen)
    m = (torch.rand(B, R, R, R, generator=gen) < 0.5).float() * g
    kn = sampling._Known(known, m, [0, 2, 3], B)
    xe, he = x.clone(), hist.clone()
    sampling._update_eager(eps, xe, he, g, row, z, kn, z2)
    xr, hr = _restated(x, eps, hist, g.numpy(), row, z, known.double().numpy(), m.double().numpy(), [0, 2, 3], z2)
    assert np.array_equal(xe.double().numpy(), xr)
    assert np.array_equal(he.double().numpy(), hr)
    keep = (m > 0)[:, None].expand_as(xe)[:, [0, 2, 3]]
    if entry == "last":  # the exact pair writes the kept region as it is
        assert torch.equal(xe[:, [0, 2, 3]][keep], known[:, [0, 2, 3]][keep])


# ---- the kept region ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [64, 128])
def test_box_region_on_the_tet_grid(R):
    from meshdiffusion_b200.geometry import dmtet
    verts, _ = dmtet.load_tet_grid(R)
    coords = dmtet.grid_coords_of_tet_vertices(torch.from_numpy(verts))
    scale = 1.1
    boxes = edit.parse_boxes([[-1.0, -1.0, -0.2, 1.0, 0.0, 0.3], [0.2, 0.2, 0.2, 0.4, 0.4, 0.4]])
    sel, vox = edit.region(boxes, verts, coords, R, scale)
    p = verts.astype(np.float64) * scale
    want = np.zeros(len(p), bool)
    for b in boxes:
        want |= np.all((p >= b[:3]) & (p <= b[3:]), axis=1)
    assert np.array_equal(sel, want) and 0 < sel.sum() < len(sel)
    # one voxel per tet vertex: the regenerated voxels are exactly the selected vertices' voxels, inside the grid mask
    gm = dmtet.grid_mask_from_tets(R)
    assert int(vox.sum()) == int(sel.sum()) and torch.all(vox <= gm)
    c = coords[torch.from_numpy(sel)]
    assert torch.all(vox[c[:, 0], c[:, 1], c[:, 2]] == 1)
    # a box around everything regenerates every vertex
    sel_all, vox_all = edit.region(edit.parse_boxes([-5, -5, -5, 5, 5, 5]), verts, coords, R, scale)
    assert sel_all.all() and torch.equal(vox_all, gm)


def test_argument_refusals(tmp_path):
    from meshdiffusion_b200.geometry import dmtet
    verts, _ = dmtet.load_tet_grid(64)
    coords = dmtet.grid_coords_of_tet_vertices(torch.from_numpy(verts))
    for bad in (None, [], [[]], [0, 0, 0, 1, 1], [[0, 0, 0, 1, 1, float("nan")]], [0.5, 0, 0, 0.4, 1, 1], "box"):
        with pytest.raises(ValueError):
            edit.parse_boxes(bad)
    with pytest.raises(ValueError, match="contains no tet vertex"):
        edit.region(edit.parse_boxes([2.0, 2.0, 2.0, 3.0, 3.0, 3.0]), verts, coords, 64, 1.1)
    for B, k in ((6, 4), (2, 4), (0, 1), (4.0, 2)):
        with pytest.raises(ValueError, match="multiple"):
            edit.sources_per_call(B, k)
    assert edit.sources_per_call(8, 4) == 2
    for key in ("edit_k", "edit_jump", "edit_resample"):
        with pytest.raises(ValueError, match=key):
            edit.edit_settings({key: 0})
    assert edit.edit_settings({}) == (4, 5, 3)
    np.save(tmp_path / "bad.npy", np.zeros((2, 4, 32, 32, 32), np.float32))
    np.save(tmp_path / "good.npy", np.zeros((2, 4, 64, 64, 64), np.float32))
    torch.save(torch.zeros(4, 64, 64, 64), tmp_path / "grid_0.pt")
    torch.save({"sdf": torch.zeros(3)}, tmp_path / "dict.pt")
    with pytest.raises(ValueError, match="shape"):
        edit.load_sources(str(tmp_path / "bad.npy"), 64, 4)
    with pytest.raises(ValueError, match="grid tensor"):
        edit.load_sources(str(tmp_path / "dict.pt"), 64, 4)
    with pytest.raises(FileNotFoundError):
        edit.load_sources(str(tmp_path / "missing.npy"), 64, 4)
    assert edit.load_sources(str(tmp_path / "good.npy"), 64, 4).shape == (2, 4, 64, 64, 64)
    assert edit.load_sources(str(tmp_path / "grid_0.pt"), 64, 4).shape == (1, 4, 64, 64, 64)
    with pytest.raises(ValueError, match="channels"):
        sampling._Known(torch.zeros(1, 4, 2, 2, 2), torch.zeros(1, 2, 2, 2), [4], 2)


# ---- analytic gate -----------------------------------------------------------------------------------------------
G, MU, ELL = 8, 0.3, 1.5


class CirculantGaussian:
    """x0 ~ N(MU, Sigma) on a periodic G^3 grid, Sigma circulant with a Gaussian spectrum (unit marginal variance). The
    exact noise prediction sigma (alpha^2 Sigma + sigma^2 I)^-1 (x - alpha MU) is evaluated with float64 FFTs, and the
    exact conditional of the regenerated voxels given the kept ones with dense linear algebra."""

    def __init__(self, sde):
        self.alpha, self.sigma = _alpha_sigma(sde)
        d = np.minimum(np.arange(G), G - np.arange(G)).astype(np.float64)
        d2 = d[:, None, None] ** 2 + d[None, :, None] ** 2 + d[None, None, :] ** 2
        lam = np.exp(-(2 * np.pi / G) ** 2 * d2 * ELL ** 2 / 2) + 0.02
        self.lam = lam / np.real(np.fft.ifftn(lam))[0, 0, 0]
        row = np.real(np.fft.ifftn(self.lam))
        idx = np.stack(np.meshgrid(*[np.arange(G)] * 3, indexing="ij"), -1).reshape(-1, 3)
        diff = (idx[:, None, :] - idx[None, :, :]) % G
        self.Sigma = row[diff[..., 0], diff[..., 1], diff[..., 2]]

    def __call__(self, x, labels):
        n = int(labels[0].item())
        a, s = self.alpha[n], self.sigma[n]
        f = torch.fft.fftn(x.double() - a * MU, dim=(-3, -2, -1)) / torch.from_numpy(a * a * self.lam + s * s).to(x.device)
        return (s * torch.real(torch.fft.ifftn(f, dim=(-3, -2, -1)))).float()

    def problem(self, seed=5):
        """(known grid [G^3], kept mask [G^3] bool, exact conditional mean and variance of the regenerated voxels)."""
        keep = np.zeros((G, G, G), bool)
        keep[:, :, :4] = True
        keep[:2] = True
        K = keep.reshape(-1)
        U = ~K
        known = MU + 1.5 * (np.linalg.cholesky(self.Sigma) @ np.random.default_rng(seed).standard_normal(G ** 3))
        S_uk = self.Sigma[np.ix_(U, K)]
        sol = np.linalg.solve(self.Sigma[np.ix_(K, K)], np.c_[known[K] - MU, S_uk.T])
        mean = MU + S_uk @ sol[:, 0]
        var = np.diag(self.Sigma[np.ix_(U, U)] - S_uk @ sol[:, 1:])
        return known, K, mean, var


def gate_run(model, sde, n, jump, resample, device, seed=1, K_steps=20):
    """n edits of the analytic model's known grid -> (NFE, max |kept - known|, RMS error of the regenerated region's mean
    against the exact conditional mean, mean ratio of its variance to the exact conditional variance)."""
    known, K, cmean, cvar = model.problem()
    torch.manual_seed(seed)
    fn = sampling.get_repaint_sampler(sde, (n, 1, G, G, G), lambda x: x, n_steps=K_steps, jump=jump, resample=resample,
                                      device=device, grid_mask=torch.ones(1, G, G, G, device=device))
    kn = torch.from_numpy(known).float().reshape(1, 1, G, G, G)
    keep = torch.from_numpy(K.reshape(1, G, G, G)).float()
    out, nfe = fn(model, kn.to(device), keep.to(device), [0])
    o = out.double().reshape(n, -1).cpu().numpy()
    kept_err = np.abs(o[:, K] - kn.reshape(-1).double().numpy()[K]).max()
    mean_err = math.sqrt(((o[:, ~K].mean(0) - cmean) ** 2).mean())
    return nfe, kept_err, mean_err, float((o[:, ~K].var(0) / cvar).mean())


# Recorded on the CPU path (3000 samples, K = 20 ODE steps, seeds 1..3): plain replacement 0.506 .. 0.512 RMS error of the
# conditional mean (variance ratio 1.18 .. 1.19); jump = 2, resample = 4 (74 evaluations) 0.282 .. 0.291 (variance ratio
# 0.993 .. 0.996). The exact conditional's RMS standard deviation is 0.87, so the Monte Carlo error of a mean is ~0.016.
GATE_RATIO = 0.7       # resampled error / plain error must be below this (recorded 0.55 .. 0.57)
GATE_MEAN_ERR = 0.33   # and the resampled error below this
GATE_VAR_TOL = 0.05    # |variance ratio - 1| of the resampled run (recorded < 0.007)


def check_gate(device):
    sde = _sde()
    model = CirculantGaussian(sde)
    nfe0, kept0, err0, var0 = gate_run(model, sde, 3000, 1, 1, device)
    nfe1, kept1, err1, var1 = gate_run(model, sde, 3000, 2, 4, device)
    print(f"analytic gate on {device}: plain err {err0:.4f} var {var0:.4f} nfe {nfe0}; resampled err {err1:.4f} "
          f"var {var1:.4f} nfe {nfe1}")
    assert nfe0 == 20 and nfe1 == 20 + 3 * 18
    assert kept0 == 0.0 and kept1 == 0.0, "the kept region must equal the known grid in every sample"
    assert err1 < GATE_RATIO * err0 and err1 < GATE_MEAN_ERR
    assert abs(var1 - 1.0) < GATE_VAR_TOL


def test_analytic_gate_cpu():
    check_gate("cpu")
