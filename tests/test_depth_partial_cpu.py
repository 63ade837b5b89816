"""CPU: the depth-map oracle (oracle/depth_oracle.py) against a brute-force search of the whole depth triangulation, the
discontinuity rule, camera parsing and back-projection, and the refusals of malformed observations."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import depth_oracle as do
from oracle import fit_oracle as fo

CELL = 1.1 / 64


def _camera(view=0):
    from meshdiffusion_b200.geometry.depth_partial import parse_camera
    return parse_camera({"view": view})


def _sphere_depth(res, cam, radius=0.3):
    """Camera depth of a sphere at the origin seen from `cam`, ray-traced in float64 through the pixel centres."""
    inv_mv = cam["inv_mv"].double().numpy()
    P = cam["proj"].double().numpy()
    n = (np.arange(res) + 0.5) / res * 2 - 1
    yn, xn = np.meshgrid(n, n, indexing="ij")
    dirs = np.stack([(xn + P[0, 2]) / P[0, 0], (yn + P[1, 2]) / P[1, 1], -np.ones_like(xn)], -1)  # camera, depth 1
    eye = inv_mv[:3, 3]
    dw = dirs @ inv_mv[:3, :3].T
    a, b, c = (dw * dw).sum(-1), 2 * (dw * eye).sum(-1), eye @ eye - radius ** 2
    disc = b * b - 4 * a * c
    t = np.where(disc >= 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0)
    return t.astype(np.float32)


def test_window_search_matches_brute_force_when_the_closest_point_is_in_the_window():
    cam, res = _camera(3), 48
    depth = _sphere_depth(res, cam)
    zbuf, valid, pts, edge = do.unproject(depth, cam["proj"], cam["inv_mv"], CELL)
    assert (valid == 0).sum() > 200 and not edge[valid == 0].all()
    rng = np.random.default_rng(0)
    surf = pts[(valid == 0) & (edge == 0)]
    q = (surf[rng.integers(0, surf.shape[0], 300)] + rng.normal(0, 0.05, (300, 3))).astype(np.float32)
    radius = 0.01  # a one-block window at this resolution: windows that miss the true closest point occur as well
    d2, cp, found = do.closest_points(q, cam["mvp"], cam["proj"], radius, pts, valid, edge)
    verts, faces = do.triangulation(pts, valid, edge)
    bd2, bface, bcp = fo.closest_points(q, verts, faces, dtype=np.float64)
    inside = 0
    for i in range(q.shape[0]):
        r, c = divmod(int(faces[bface[i], 0]), res)
        win = do.window(q[i], cam["mvp"], cam["proj"], res, radius)
        if win is not None and win[0] <= r <= win[1] and win[2] <= c <= win[3]:
            inside += 1
            assert found[i]
            assert d2[i] == pytest.approx(bd2[i], rel=1e-4, abs=1e-9)
            np.testing.assert_allclose(cp[i], bcp[i], atol=1e-5)
        elif found[i]:
            assert d2[i] >= bd2[i] * (1 - 1e-4)  # the window never finds a point nearer than the whole surface has
    assert 100 < inside < q.shape[0]


def test_depth_step_is_an_edge_and_no_triangle_crosses_it():
    cam, res = _camera(0), 32
    depth = np.full((res, res), 2.0, np.float32)
    depth[:, res // 2:] = 2.3  # a step of 0.3, far more than a cell edge
    depth[:2] = 0.0            # rows with no surface
    zbuf, valid, pts, edge = do.unproject(depth, cam["proj"], cam["inv_mv"], CELL)
    assert (valid[:2] == -1).all() and (zbuf[:2] == do.EMPTY_DEPTH).all() and (edge[:2] == 0).all()
    assert (edge[2:, res // 2 - 1] == 1).all() and (edge[2:, res // 2] == 1).all()
    assert edge[2:, : res // 2 - 1].sum() == 0 and edge[2:, res // 2 + 1:].sum() == 0
    verts, faces = do.triangulation(pts, valid, edge)
    assert faces.shape[0] > 0
    dv = depth.reshape(-1)[faces]
    assert (dv == dv[:, :1]).all()  # every triangle lies on one plane
    # a point between the planes, at the step: its closest point lies on one of the planes, never on a wall across the step
    near, far = pts[10, res // 2 - 3], pts[10, res // 2 + 2]
    q = ((near + far) * 0.5).astype(np.float32)[None]
    d2, cp, found = do.closest_points(q, cam["mvp"], cam["proj"], 0.5, pts, valid, edge)
    assert found[0]
    cam_z = (cam["mv"].numpy() @ np.append(cp[0], 1.0))[2]
    assert min(abs(-cam_z - 2.0), abs(-cam_z - 2.3)) < 1e-4


def test_view_and_matrices_give_the_same_camera():
    from meshdiffusion_b200.geometry.depth_partial import parse_camera, view_camera
    from meshdiffusion_b200.geometry.singleview import view_mvp
    for view in (0, 17):
        mv, proj = view_camera(view)
        a = parse_camera({"view": view})
        b = parse_camera(json.loads(json.dumps({"mv": mv.tolist(), "proj": proj.tolist()})))
        for key in ("mvp", "proj", "mv", "inv_mv"):
            assert torch.equal(a[key], b[key]), key
        assert torch.equal(a["mvp"], view_mvp(view, 1000))


def test_known_depth_unprojects_to_its_world_point():
    cam, res = _camera(17), 64
    P, inv_mv = cam["proj"].double().numpy(), cam["inv_mv"].double().numpy()
    depth = np.zeros((res, res), np.float32)
    rows, cols, ds = [5, 31, 60], [40, 2, 33], [1.75, 2.0, 2.25]
    for r, c, d in zip(rows, cols, ds):
        depth[r, c] = d
    zbuf, valid, pts, edge = do.unproject(depth, cam["proj"], cam["inv_mv"], CELL)
    assert int((valid == 0).sum()) == 3
    for r, c, d in zip(rows, cols, ds):
        xn, yn = (c + 0.5) / res * 2 - 1, (r + 0.5) / res * 2 - 1
        world = inv_mv @ np.array([d * (xn + P[0, 2]) / P[0, 0], d * (yn + P[1, 2]) / P[1, 1], -d, 1.0])
        np.testing.assert_allclose(pts[r, c], world[:3], atol=2e-6)
        # and back: the world point projects to the pixel's centre at the given depth
        h = cam["mvp"].double().numpy() @ np.append(pts[r, c].astype(np.float64), 1.0)
        assert h[3] == pytest.approx(d, abs=1e-5)
        assert (h[0] / h[3] * 0.5 + 0.5) * res == pytest.approx(c + 0.5, abs=1e-3)
        assert (h[1] / h[3] * 0.5 + 0.5) * res == pytest.approx(r + 0.5, abs=1e-3)
        assert zbuf[r, c] == pytest.approx(h[2] / h[3], abs=1e-5)


def test_rendered_z_converts_back_to_camera_depth():
    from meshdiffusion_b200.geometry.depth_partial import camera_depth
    cam = _camera(0)
    d = torch.tensor([[1.5, 2.0], [2.5, 0.0]])
    z = (cam["proj"][2, 3] - cam["proj"][2, 2] * d) / d
    back = camera_depth(z, torch.tensor([[0, 3], [7, -1]]), cam["proj"])
    np.testing.assert_allclose(back.numpy(), [[1.5, 2.0], [2.5, 0.0]], rtol=1e-5)


def test_malformed_observations_are_refused():
    from meshdiffusion_b200.geometry.depth_partial import check_depth, check_inside_grid, grid_box, parse_camera, view_camera
    with pytest.raises(ValueError, match="square"):
        check_depth(np.ones((8, 9), np.float32))
    with pytest.raises(ValueError, match="square"):
        check_depth(np.ones(8, np.float32))
    with pytest.raises(ValueError, match="4096"):
        check_depth(np.zeros((4097, 4097), np.float32))
    with pytest.raises(ValueError, match="negative"):
        check_depth(np.array([[1.0, -0.5], [0.0, 1.0]], np.float32))
    ok = check_depth(np.array([[np.nan, np.inf], [-np.inf, 0.0]]))  # non-finite and 0: no surface, not an error
    assert ok.dtype == np.float32
    mv, proj = view_camera(0)
    with pytest.raises(ValueError, match="no camera"):
        parse_camera({"depth": "a.npy"})
    with pytest.raises(ValueError, match="not both"):
        parse_camera({"view": 0, "mv": mv.tolist(), "proj": proj.tolist()})
    with pytest.raises(ValueError, match="both 'mv' and 'proj'"):
        parse_camera({"mv": mv.tolist()})
    with pytest.raises(ValueError, match="integer"):
        parse_camera({"view": 1.5})
    ortho = torch.eye(4)
    ortho[2, 2] = -0.1
    with pytest.raises(ValueError, match="not a perspective matrix"):
        parse_camera({"mv": mv.tolist(), "proj": ortho.tolist()})
    skew = proj.clone()
    skew[0, 1] = 0.2
    with pytest.raises(ValueError, match="not a perspective matrix"):
        parse_camera({"mv": mv.tolist(), "proj": skew.tolist()})
    with pytest.raises(ValueError, match="4 x 4"):
        parse_camera({"mv": mv[:3].tolist(), "proj": proj.tolist()})
    with pytest.raises(ValueError, match="invertible"):
        parse_camera({"mv": torch.zeros(4, 4).tolist(), "proj": proj.tolist()})
    # an observed point outside the grid: the sphere seen from view 0, then the same depths scaled far beyond it
    cam, res = parse_camera({"view": 0}), 24
    lo, hi = grid_box(64)
    depth = _sphere_depth(res, cam, radius=0.3)
    _, valid, pts, _ = do.unproject(depth, cam["proj"], cam["inv_mv"], CELL)
    check_inside_grid(torch.from_numpy(pts)[None], torch.from_numpy(valid)[None], lo, hi)
    _, valid, pts, _ = do.unproject(depth * 3, cam["proj"], cam["inv_mv"], CELL)
    with pytest.raises(ValueError, match="outside the grid"):
        check_inside_grid(torch.from_numpy(pts)[None], torch.from_numpy(valid)[None], lo, hi, [(7,)])


def test_depth_meta_refusals(tmp_path):
    from meshdiffusion_b200.diffusion.evaler import read_depth_meta
    np.save(os.path.join(tmp_path, "a.npy"), np.ones((16, 16), np.float32))
    np.save(os.path.join(tmp_path, "wide.npy"), np.ones((16, 8), np.float32))

    def meta(entries):
        p = os.path.join(tmp_path, "meta.json")
        with open(p, "w") as fh:
            json.dump(entries, fh)
        return p
    obs = read_depth_meta(meta([{"depth": "a.npy", "view": 2}]))
    assert obs[0][0] == "a.npy" and obs[0][1].shape == (16, 16)
    with pytest.raises(ValueError, match="non-empty JSON list"):
        read_depth_meta(meta([]))
    with pytest.raises(ValueError, match="no 'depth'"):
        read_depth_meta(meta([{"view": 0}]))
    with pytest.raises(ValueError, match="observation 0: an observation has no camera"):
        read_depth_meta(meta([{"depth": "a.npy"}]))
    with pytest.raises(ValueError, match="square"):
        read_depth_meta(meta([{"depth": "wide.npy", "view": 0}]))


def test_completion_refuses_an_index_without_ground_truth(tmp_path):
    from meshdiffusion_b200.diffusion.completion import check_sources, read_index
    d = os.path.join(tmp_path, "partial")
    os.makedirs(d)
    torch.save({}, os.path.join(d, "obs.pt"))
    with open(os.path.join(d, "index.json"), "w") as fh:
        json.dump({"resolution": 64, "res": 1000, "mesh_scale": 1.1, "deform_scale": 3.0,
                   "files": [{"file": "obs.pt", "depth": "obs.npy", "res": 1000}]}, fh)
    with pytest.raises(ValueError, match="no 'shape' field"):
        read_index(d)
    with pytest.raises(ValueError, match="no 'source' field"):
        check_sources([{"file": "x.pt", "shape": 0, "view": 0}], ["a"])
