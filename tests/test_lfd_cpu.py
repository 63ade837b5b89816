"""CPU: the light field distance's fixed parts (geometry/lfd.py) and its numpy restatement (oracle/lfd_oracle.py): the
dodecahedron's rotation group and view permutations, the camera-set rotation table against its generator, descriptor
invariances on simple silhouettes, and the distance's group properties on descriptors and on two small meshes."""
import numpy as np
import pytest

from helpers import ROOT  # noqa: F401  (puts the repository on sys.path)
from oracle import lfd_oracle as lo


def _lfd():
    from meshdiffusion_b200.geometry import lfd
    return lfd


def _vertices20():
    return np.concatenate([lo.VERTS, -lo.VERTS])


def test_rotation_group_is_the_dodecahedron_group():
    G = lo.icosahedral_group()
    assert G.shape == (60, 3, 3)
    assert np.abs(G[0] - np.eye(3)).max() == 0

    def find(m):
        k = [i for i, g in enumerate(G) if np.abs(g - m).max() < 1e-9]
        assert len(k) == 1
        return k[0]

    for a in G:
        find(a.T)  # inverse
        for b in G:
            find(a @ b)  # closure
    V = _vertices20()
    for g in G:
        img = V @ g.T
        assert all(np.abs(V - x).max(1).min() < 1e-9 for x in img)
    perms = lo.permutations(G)
    assert len({tuple(p) for p in perms}) == 60
    assert all(sorted(p) == list(range(10)) for p in perms)
    np.testing.assert_array_equal(_lfd().PERMUTATIONS, perms)
    assert _lfd().PERMUTATIONS.dtype == np.int8


def test_rotation_table_matches_its_generator():
    R = _lfd().ROTATIONS
    assert R.shape == (10, 3, 3)
    assert np.abs(lo.generate_rotations() - R).max() <= 1e-15
    assert np.abs(R[0] - np.eye(3)).max() == 0
    for r in R:
        assert np.abs(r @ r.T - np.eye(3)).max() < 1e-14
        assert abs(np.linalg.det(r) - 1) < 1e-14


def test_module_mvps_equal_the_oracle_bitwise():
    lfd = _lfd()
    rng = np.random.default_rng(0)
    v = rng.normal(size=(50, 3)).astype(np.float32)
    c, s = lo.centre_scale(v)
    got = lfd.camera_mvps(c[None], np.array([s]))[0]
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got.view(np.uint32), lo.mvps(lfd.ROTATIONS, c, s).view(np.uint32))
    # the rows are an orthonormal frame scaled by 0.9 s, 0.9 s, 0.5 s: the unit sphere around c fits the image
    F = lfd.FRAMES
    np.testing.assert_allclose(np.einsum("vij,vkj->vik", F, F), np.broadcast_to(np.eye(3), F.shape), atol=1e-14)


def _disk(res, cx, cy, r):
    y, x = np.mgrid[:res, :res] + 0.5
    return (x - cx) ** 2 + (y - cy) ** 2 <= r * r


def test_descriptors_are_invariant_to_right_angle_rotations_and_mirrors():
    res = 64
    rect = np.zeros((res, res), bool)
    rect[13:40, 20:31] = True
    for img in (_disk(res, 30.5, 33.0, 17.3), rect):
        base, n = lo.descriptor(img)
        assert n == int(img.sum()) and base[:45].any() and not base[45:].any()
        for other in (np.rot90(img), np.rot90(img, 2), np.fliplr(img), np.flipud(img)):
            d, _ = lo.descriptor(other)
            assert np.abs(d.astype(int) - base.astype(int)).max() <= 1, (base, d)


def test_empty_and_single_pixel_silhouettes():
    d, n = lo.descriptor(np.zeros((40, 40), bool))
    assert n == 0 and not d.any()
    one = np.zeros((40, 40), bool)
    one[7, 29] = True
    d, n = lo.descriptor(one)
    assert n == 1 and d.shape == (48,)


def test_oracle_distance_group_properties():
    perms = _lfd().PERMUTATIONS
    rng = np.random.default_rng(1)
    A = rng.integers(0, 256, (10, 10, 48), dtype=np.uint8)
    B = rng.integers(0, 256, (10, 10, 48), dtype=np.uint8)
    assert lo.lfd(A, A, perms) == 0
    assert lo.lfd(A, B, perms) == lo.lfd(B, A, perms) > 0
    for g in (1, 17, 59):
        assert lo.lfd(A, A[:, perms[g]], perms) == 0
        assert lo.lfd(A[::-1], A[:, perms[g]], perms) == 0  # light fields in another order as well
        assert lo.lfd(A[:, perms[g]], B, perms) == lo.lfd(A, B, perms)


def _torus(R=0.6, r=0.25, nu=16, nv=8):
    u, v = np.meshgrid(np.arange(nu) * 2 * np.pi / nu, np.arange(nv) * 2 * np.pi / nv, indexing="ij")
    p = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], -1).reshape(-1, 3)
    f = []
    for i in range(nu):
        for j in range(nv):
            a, b, c, d = i * nv + j, (i + 1) % nu * nv + j, (i + 1) % nu * nv + (j + 1) % nv, i * nv + (j + 1) % nv
            f += [(a, b, c), (a, c, d)]
    return p.astype(np.float32), np.array(f)


def _box(h=(0.5, 0.3, 0.15)):
    p = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32) * np.float32(h)
    f = np.array([(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6),
                  (0, 6, 4), (1, 5, 7), (1, 7, 3)])
    return p, f


@pytest.mark.parametrize("shape", ["torus", "box"])
def test_a_group_rotation_of_a_mesh_is_near_it(shape):
    lfd = _lfd()
    S, T = (_torus(), _box()) if shape == "torus" else (_box(), _torus())
    g = lo.icosahedral_group()[7]
    gS = ((S[0].astype(np.float64) @ g.T).astype(np.float32), S[1])
    d = [lo.mesh_descriptors(v, f, lfd.ROTATIONS, res=64) for v, f in (S, gS, T)]
    assert all(e == 0 for _, e in d)
    near = lo.lfd(d[0][0], d[1][0], lfd.PERMUTATIONS)
    far = lo.lfd(d[0][0], d[2][0], lfd.PERMUTATIONS)
    assert near < 0.2 * far, (near, far)
