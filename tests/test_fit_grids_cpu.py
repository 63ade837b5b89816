"""CPU: the OBJ reader and the normalisation of `--mode=fit_grids`, its camera set, the float32 oracles of the fitting
kernels on hand-worked cases, and the mode's command line."""
import json
import os

import numpy as np
import pytest

from helpers import ROOT
from oracle import fit_oracle as fo


def _write(tmp_path, name, text):
    p = os.path.join(tmp_path, name)
    with open(p, "w") as fh:
        fh.write(text)
    return p


def test_obj_reader_face_forms_negative_indices_polygons_and_groups(tmp_path):
    from meshdiffusion_b200.geometry.mesh_io import read_obj
    p = _write(tmp_path, "m.obj", """# every face form
mtllib m.mtl
o first
v 0 0 0
v 1 0 0
v 1 1 0
v 0 1 0
vt 0 0
vt 1 0
vt 1 1
vn 0 0 1
usemtl a
s 1
f 1 2 3
f 1/1 3/2 4/3
g second
v 0 0 1
v 1 0 1
v 1 1 1
v 0 1 1
v 0.5 1.5 1
f 5//1 6//1 7//1 8//1
f -5/1/1 -4/2/1 -3/3/1 -2/1/1 -1/2/1
l 1 2
f 9 8
""")
    v, f = read_obj(p)
    assert v.shape == (9, 3) and v.dtype == np.float64 and f.dtype == np.int64
    np.testing.assert_array_equal(v[8], [0.5, 1.5, 1])
    np.testing.assert_array_equal(f, [[0, 1, 2], [0, 2, 3],              # a, a/b
                                      [4, 5, 6], [4, 6, 7],              # a//c quad, fan-triangulated
                                      [4, 5, 6], [4, 6, 7], [4, 7, 8]])  # negative a/b/c pentagon


def test_obj_reader_refuses_undefined_vertices(tmp_path):
    from meshdiffusion_b200.geometry.mesh_io import read_obj
    with pytest.raises(ValueError, match="not defined"):
        read_obj(_write(tmp_path, "bad.obj", "v 0 0 0\nv 1 0 0\nf 1 2 3\nv 0 1 0\n"))
    with pytest.raises(ValueError, match="not defined"):
        read_obj(_write(tmp_path, "neg.obj", "v 0 0 0\nv 1 0 0\nv 0 1 0\nf -4 -2 -1\n"))


def test_normalize_ignores_unreferenced_vertices(tmp_path):
    from meshdiffusion_b200.geometry.mesh_io import load_mesh
    p = _write(tmp_path, "n.obj", "v 100 100 100\nv 1 2 3\nv 5 2 3\nv 1 4 3\nv 1 2 4\nv -50 0 0\n"
                                  "f 2 3 4\nf 2 3 5\n")
    v, f = load_mesh(p)
    assert v.dtype == np.float32
    used = v[np.unique(f)]
    lo, hi = used.min(0), used.max(0)
    np.testing.assert_array_equal(lo + hi, [0, 0, 0])          # centred on the box of the referenced vertices
    assert float((hi - lo).max()) == 1.0                         # largest side exactly 1
    np.testing.assert_array_equal(hi - lo, [1.0, 0.5, 0.25])
    np.testing.assert_array_equal(v[0], [24.25, 24.25, 24.125])  # unreferenced vertices move along, uncounted


def test_cameras_see_every_grid_corner_at_positive_w():
    from meshdiffusion_b200.geometry import dmtet
    from meshdiffusion_b200.geometry.fit import VIEWS, camera_mvps
    for R in (64, 128):
        verts, _ = dmtet.load_tet_grid(R)
        lo, hi = verts.min(0) * np.float32(1.1), verts.max(0) * np.float32(1.1)
        corners = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float32)
        for n in (VIEWS, 7):
            m = camera_mvps(n).numpy()
            assert m.shape == (n, 4, 4) and m.dtype == np.float32
            assert len({row.tobytes() for row in m}) == n  # the views are distinct
            for k in range(n):
                h = fo.mvp_rows(m[k], corners)
                assert (h[:, 3] > 0).all()
                ndc = h[:, :3] / h[:, 3:]
                assert (np.abs(ndc[:, :2]) < 1).all() and (np.abs(ndc[:, 2]) < 1).all()


def _dense_closest(p, a, b, c, n=800):
    """Closest point of p on the triangle by dense float64 barycentric sampling."""
    u, w = np.meshgrid(np.linspace(0, 1, n), np.linspace(0, 1, n), indexing="ij")
    keep = u + w <= 1
    pts = a + u[keep][:, None] * (b - a) + w[keep][:, None] * (c - a)
    d = ((pts - p) ** 2).sum(1)
    return pts[np.argmin(d)], d.min()


@pytest.mark.parametrize("region,p", [
    ("a", [-0.3, -0.2, 0.4]), ("b", [1.4, -0.2, -0.1]), ("c", [-0.1, 1.3, 0.2]),
    ("ab", [0.5, -0.4, 0.3]), ("bc", [0.7, 0.7, -0.2]), ("ca", [-0.4, 0.5, 0.1]), ("interior", [0.25, 0.3, 0.7]),
])
def test_closest_point_oracle_on_every_voronoi_region(region, p):
    a, b, c = np.array([0.0, 0, 0]), np.array([1.0, 0, 0]), np.array([0.0, 1, 0])
    p = np.array(p)
    want_p, want_d = _dense_closest(p, a, b, c)
    exact = {"a": a, "b": b, "c": c, "ab": [p[0], 0, 0], "bc": [(1 + p[0] - p[1]) / 2, (1 - p[0] + p[1]) / 2, 0],
             "ca": [0, p[1], 0], "interior": [p[0], p[1], 0]}[region]
    for dt, tol in ((np.float64, 1e-12), (np.float32, 1e-6)):
        d2, face, cp = fo.closest_points(p[None].astype(dt), np.stack([a, b, c]).astype(dt), [[0, 1, 2]], dtype=dt)
        assert face[0] == 0 and cp.dtype == dt
        np.testing.assert_allclose(cp[0], exact, atol=tol)
        np.testing.assert_allclose(cp[0], want_p, atol=2.0 / 800)  # the sampling's own spacing
        assert d2[0] <= want_d + tol


def test_closest_point_oracle_degenerate_faces_and_ties():
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 1, 0]], np.float32)
    # a collinear triangle, a point triangle, then two identical faces: the nearest, lower index wins
    f = np.array([[0, 1, 2], [3, 3, 3], [0, 1, 3], [0, 1, 3]])
    q = np.array([[1.5, 0.5, 0], [0, 1.2, 0], [0.2, 0.2, 1]], np.float32)
    d2, face, cp = fo.closest_points(q, v, f)
    np.testing.assert_array_equal(face, [0, 1, 2])
    np.testing.assert_allclose(cp, [[1.5, 0, 0], [0, 1, 0], [0.2, 0.2, 0]], atol=1e-7)
    np.testing.assert_allclose(d2, [0.25, 0.04, 1.0], rtol=1e-6)
    d, k = fo.nearest_vertex(np.array([[1, 0.5, 0], [0.5, 0, 0]], np.float32), v)
    np.testing.assert_array_equal(k, [1, 0])  # equidistant from 1 and 3; from 0 and 1: the lower index
    np.testing.assert_allclose(d, [0.25, 0.25])
    assert fo.nearest_vertex(q, np.zeros((0, 3), np.float32))[1].tolist() == [-1, -1, -1]


def test_carve_oracle_single_quad_one_view():
    """A unit quad at z = 0 seen along -z by an orthographic view (identity mvp): its pixels have depth 0. A point in front
    of it (z < 0) is seen, one behind it (z > 0) is not, one beside it is, and at the quad's rim the (2k+1)^2 window
    decides."""
    from oracle import raster_oracle as ro
    res, k = 16, 1
    v = np.array([[-0.5, -0.5, 0], [0.5, -0.5, 0], [0.5, 0.5, 0], [-0.5, 0.5, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    mvp = np.eye(4, dtype=np.float32)
    depth, face_id, _ = ro.rasterize(v, f, mvp, res)
    assert (face_id >= 0).sum() == 64 and (depth[face_id >= 0] == 0).all()
    pts = np.array([[0.1, 0.1, -0.5],   # in front of the quad: every pixel of its window is deeper
                    [0.1, 0.1, 0.5],    # behind it
                    [0.9, 0.9, 0.5],    # beside it, behind its plane: the window is empty
                    [0.55, 0.0, 0.5],   # behind, half a pixel beyond the rim: the window reaches the quad
                    [0.0, 0.0, 0.0],    # on it: depth 0 is not deeper than 0
                    [0.0, 0.0, 2.0]],   # outside the depth range of the view: still behind the quad
                   np.float32)
    np.testing.assert_array_equal(fo.carve(pts, mvp[None], depth[None], face_id[None], k), [1, 0, 1, 0, 0, 0])
    np.testing.assert_array_equal(fo.carve(pts, mvp[None], depth[None], face_id[None], 0), [1, 0, 1, 1, 0, 0])


def test_fit_grids_mode_parses_and_refuses_an_empty_mesh_list(tmp_path):
    import main_diffusion
    from meshdiffusion_b200.diffusion.fit_grids import fit_grids
    cfg_path, mode, overrides = main_diffusion.parse_args([f"--config={ROOT}/configs/res64.py", "--mode=fit_grids",
                                                           "--config.data.mesh_meta_path=/m.json", "--config.data.fit_iters=5"])
    assert mode == "fit_grids" and dict(overrides) == {"data.mesh_meta_path": "/m.json", "data.fit_iters": 5}
    cfg = main_diffusion.load_config_file(cfg_path)
    for key in ("mesh_meta_path", "grid_dir", "fit_views", "fit_res", "fit_window", "fit_iters", "fit_lr", "fit_points",
                "fit_reg", "fit_batch"):
        assert key not in cfg.data
    meta = _write(tmp_path, "meshes.json", json.dumps([]))
    cfg.set_by_path("data.mesh_meta_path", meta)
    cfg.set_by_path("data.grid_dir", str(tmp_path / "grids"))
    with pytest.raises(ValueError, match="is empty"):
        fit_grids(cfg)
    cfg.set_by_path("data.mesh_meta_path", "PLACEHOLDER")
    with pytest.raises(ValueError, match="mesh_meta_path"):
        fit_grids(cfg)
