"""CPU: the single-view camera against the reference's own matrices, the float32 rasterizer / visibility oracle on
hand-worked cases and against a direct restatement of nvdiffrec/lib/render/render.py:346-407, and `--mode=make_partial`'s
command line."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import GOLD, ROOT
from oracle import raster_oracle as ro

I4 = np.eye(4, dtype=np.float32)


def _ndc(X, Y, res):
    """Clip x, y (w = 1) of screen position (X, Y) in pixels."""
    return X / res * 2 - 1, Y / res * 2 - 1


def _tri(screen, z, res):
    return np.array([[*_ndc(X, Y, res), zz] for (X, Y), zz in zip(screen, z)], np.float32)


def test_view_mvp_matches_reference_cameras():
    from meshdiffusion_b200.geometry.singleview import view_mvp
    with open(os.path.join(GOLD, "singleview_cameras.json")) as fh:
        gold = json.load(fh)
    assert gold["views"] == [0, 1, 17, 49]
    for v, m in zip(gold["views"], gold["mvp"]):
        got = view_mvp(v, 1000)
        assert got.dtype == torch.float32 and got.shape == (4, 4)
        assert torch.equal(got, torch.tensor(m, dtype=torch.float32)), v


def test_one_triangle_coverage_and_depth():
    """Screen corners (1, 1), (7, 1), (1, 7) at res 8: the pixel centres with X, Y >= 1 and X + Y <= 8 (the hypotenuse is
    inclusive), i.e. columns c >= 1, rows r >= 1, c + r <= 7: 21 pixels. Depth is linear in the screen position."""
    res = 8
    verts = _tri([(1, 1), (7, 1), (1, 7)], [0.0, 0.6, -0.6], res)
    depth, face, behind = ro.rasterize(verts, np.array([[0, 1, 2]]), I4, res)
    r, c = np.mgrid[0:res, 0:res]
    want = (c >= 1) & (r >= 1) & (c + r <= 7)
    assert want.sum() == 21 and behind == 0
    np.testing.assert_array_equal(face, np.where(want, 0, -1))
    X, Y = c + 0.5, r + 0.5
    np.testing.assert_allclose(depth[want], (0.6 * (X - 1) / 6 - 0.6 * (Y - 1) / 6)[want], atol=1e-6)
    assert (depth[~want] == 100).all() and depth.dtype == np.float32 and face.dtype == np.int32
    # the other winding covers the same pixels with the same depths
    d2, f2, _ = ro.rasterize(verts, np.array([[0, 2, 1]]), I4, res)
    np.testing.assert_array_equal(f2, face)
    np.testing.assert_array_equal(d2[want], depth[want])


def test_two_overlapping_triangles_nearest_wins():
    res = 16
    big = _tri([(0, 0), (16, 0), (0, 16)], [0.5] * 3, res)
    small = _tri([(2, 2), (8, 2), (2, 8)], [-0.2] * 3, res)
    verts = np.concatenate([big, small])
    for faces, near_id in ((np.array([[0, 1, 2], [3, 4, 5]]), 1), (np.array([[3, 5, 4], [0, 1, 2]]), 0)):
        depth, face, _ = ro.rasterize(verts, faces, I4, res)
        r, c = np.mgrid[0:res, 0:res]
        in_small = (c >= 2) & (r >= 2) & (c + r <= 9)  # centres with X, Y >= 2.5 and X + Y <= 10
        in_big = (c + r <= 15)
        np.testing.assert_array_equal(face, np.where(in_small, near_id, np.where(in_big, 1 - near_id, -1)))
        np.testing.assert_allclose(depth[in_small], -0.2, atol=1e-6)  # interpolation rounds in the last bit
        np.testing.assert_allclose(depth[in_big & ~in_small], 0.5, atol=1e-6)


def test_duplicate_triangle_lower_id_wins():
    res = 8
    verts = _tri([(1, 1), (7, 1), (1, 7)], [0.1, 0.3, -0.2], res)
    # the same corners in the same order give bitwise equal depths: a tie, which the lower face index wins
    depth, face, _ = ro.rasterize(np.concatenate([verts, verts]), np.array([[3, 4, 5], [0, 1, 2], [0, 1, 2]]), I4, res)
    assert (face[face >= 0] == 0).all() and (face >= 0).sum() == 21


def test_fragment_beyond_far_plane_is_dropped():
    res = 8
    verts = _tri([(0, 0), (8, 0), (0, 8)], [1.5, 1.5, 1.5], res)
    depth, face, _ = ro.rasterize(verts, np.array([[0, 1, 2]]), I4, res)
    assert (face == -1).all() and (depth == 100).all()
    # depth 0.5 at X = 0 up to 1.5 at X = 8: only the fragments with z / w <= 1 remain
    verts = _tri([(0, 0), (8, 0), (0, 8)], [0.5, 1.5, 0.5], res)
    depth, face, _ = ro.rasterize(verts, np.array([[0, 1, 2]]), I4, res)
    kept = face == 0
    assert 0 < kept.sum() < 36 and (depth[kept] <= 1).all()
    c = np.mgrid[0:res, 0:res][1]
    assert (c[kept] <= 3).all() and kept[0, 3]


def test_triangle_behind_camera_is_counted_not_drawn():
    from meshdiffusion_b200.geometry.singleview import view_mvp
    mvp = view_mvp(0, 64).numpy()
    verts = np.array([[0, 0, 0], [0.2, 0, 0], [0, 0, 5.0], [0.1, 0.1, 0], [0.2, 0.1, 0], [0.1, 0.2, 0]], np.float32)
    assert (ro.mvp_rows(mvp, verts[2])[3] <= 0) and (ro.mvp_rows(mvp, verts[:2])[:, 3] > 0).all()
    depth, face, behind = ro.rasterize(verts, np.array([[0, 1, 2], [3, 4, 5]]), mvp, 64)
    assert behind == 1
    assert set(np.unique(face)) == {-1, 1}


def test_brute_force_pixels_match_full_rasterizer():
    rng = np.random.default_rng(3)
    verts = rng.uniform(-1.2, 1.2, (60, 3)).astype(np.float32)
    verts[:, 2] *= 0.8
    faces = rng.integers(0, 60, (40, 3))
    faces[5] = faces[4]  # a duplicate
    depth, face, _ = ro.rasterize(verts, faces, I4, 33)
    r, c = np.mgrid[0:33, 0:33]
    d2, f2 = ro.rasterize_pixels(verts, faces, I4, 33, r.ravel(), c.ravel())
    np.testing.assert_array_equal(f2, face.ravel())
    np.testing.assert_array_equal(d2, depth.ravel())


def _reference_visibility(n, f2t, depth, face_id):
    """render.py:346-407 restated with torch on the oracle's transformed centres n [T, 3]: returns (visible_tet_id,
    rast_tet_id) as sorted id arrays."""
    res = depth.shape[0]
    transformed = torch.from_numpy(n)
    it = torch.round((transformed / 2.0 + 0.5) * (res - 1)).long()
    tmp = it.clone()
    it[:, 0] = tmp[:, 1]
    it[:, 1] = tmp[:, 0]
    valid = (torch.logical_and(it <= res - 1, it >= 0).float()).prod(dim=-1) == 1
    vi = it[valid]
    vdepth = transformed[valid][:, -1]
    ids = torch.arange(n.shape[0])[valid]
    fid = torch.from_numpy(face_id)[None]
    d = torch.from_numpy(depth)[None].clone()
    d[fid < 0] = 100
    d = -torch.nn.functional.max_pool2d(-d, kernel_size=15, stride=1, padding=7)
    depth_filter = d[0, vi[:, 0], vi[:, 1]] >= vdepth
    empty = (-torch.nn.functional.max_pool2d(-(fid < 0).float(), kernel_size=15, stride=1, padding=7)).bool()
    empty_filter = empty[0, vi[:, 0], vi[:, 1]]
    visible = ids[torch.logical_or(empty_filter, depth_filter)]
    rast_tri = fid.unique()
    rast_tri = rast_tri[rast_tri >= 0]
    rast = torch.from_numpy(np.asarray(f2t))[rast_tri].unique()
    return visible.numpy(), rast.numpy()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_visibility_matches_maxpool_restatement(seed):
    rng = np.random.default_rng(seed)
    res = 40
    pos = rng.uniform(-2.6, 2.6, (300, 3)).astype(np.float32)
    tets = rng.integers(0, 300, (500, 4)).astype(np.int32)
    depth = rng.uniform(-0.2, 1, (res, res)).astype(np.float32)
    face_id = rng.integers(0, 50, (res, res)).astype(np.int32)
    face_id[:, : res // 3] = -1  # an empty band, wider than the window
    face_id[rng.random((res, res)) < 0.1] = -1
    depth[face_id < 0] = 100
    f2t = rng.integers(0, 500, 50)
    mvp = I4.copy()
    mvp[3, 3] = 1.1
    vis, rast = ro.visible_tets(pos, tets, f2t, mvp, depth, face_id)
    n, q, in_view = ro.centre_pixels(pos, tets, mvp, res)
    want_vis, want_rast = _reference_visibility(n, f2t, depth, face_id)
    assert 0 < in_view.sum() < in_view.size and 0 < vis.sum() < in_view.sum()
    assert (vis & (q[:, 0] > res // 3 + 7)).any()  # some pass the depth test, away from the empty band
    np.testing.assert_array_equal(np.nonzero(vis)[0], want_vis)
    np.testing.assert_array_equal(np.nonzero(rast)[0], want_rast)


def test_make_partial_mode_parses_and_default_config_is_unchanged():
    import main_diffusion
    cfg_path, mode, overrides = main_diffusion.parse_args([f"--config={ROOT}/configs/res64.py", "--mode=make_partial",
                                                           "--config.eval.partial_views=(0, 17)", "--config.eval.partial_res=256"])
    assert mode == "make_partial" and dict(overrides) == {"eval.partial_views": (0, 17), "eval.partial_res": 256}
    for name in ("res64", "res128"):
        cfg = main_diffusion.load_config_file(os.path.join(ROOT, "configs", f"{name}.py"))
        for key in ("partial_views", "partial_res", "mesh_scale", "deform_scale"):
            assert key not in cfg.eval
