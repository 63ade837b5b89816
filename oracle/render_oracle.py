"""Float32 numpy restatement of the preview shading kernel (`mdb_render_shade`, meshdiffusion_b200/csrc/raster.cu), plus a
float64 SH projection of a lat-long radiance map and the sRGB threshold table the kernel encodes with.

The face ids come from `raster_oracle.rasterize` at res * ssaa. Every product, sum, quotient and square root is a float32
numpy operation, rounded on its own, in the kernel's order, so the bytes match the kernel's. Pure numpy: also runs
without a GPU.
"""
import numpy as np

from . import raster_oracle as ro

F32 = np.float32
NORMAL_THRESHOLD = F32(0.1)
# real SH basis constants, l <= 2
_C0, _C1, _C2, _C20, _C22 = (F32(0.28209479177387814), F32(0.4886025119029199), F32(1.0925484305920792),
                             F32(0.31539156525252005), F32(0.5462742152960396))


def srgb_to_linear(s):
    s = np.asarray(s, np.float64)
    return np.where(s <= 0.04045, s / 12.92, ((s + 0.055) / 1.055) ** 2.4)


def srgb_thresholds():
    """fp32 [255]: code k (1..255) starts where sRGB(x) reaches (k - 0.5) / 255; computed in float64."""
    return srgb_to_linear((np.arange(1, 256) - 0.5) / 255).astype(F32)


def encode_srgb(x, thresholds=None):
    """uint8 codes of linear values x: the number of thresholds each one reaches (NaN -> 0)."""
    t = srgb_thresholds() if thresholds is None else np.asarray(thresholds, F32)
    x = np.asarray(x, F32)
    code = np.searchsorted(t, x, side="right")
    return np.where(np.isnan(x), 0, code).astype(np.uint8)


def sh9_basis(d):
    """float64 [..., 9] real SH of unit directions d [..., 3] in the kernel's order."""
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    c0, c1, c2 = 0.5 / np.sqrt(np.pi), np.sqrt(3 / (4 * np.pi)), 0.5 * np.sqrt(15 / np.pi)
    c20, c22 = 0.25 * np.sqrt(5 / np.pi), 0.25 * np.sqrt(15 / np.pi)
    return np.stack([np.full_like(x, c0), c1 * y, c1 * z, c1 * x, c2 * x * y, c2 * y * z, c20 * (3 * z * z - 1),
                     c2 * x * z, c22 * (x * x - y * y)], -1)


def latlong_dirs(h, w):
    """float64 directions [h, w, 3] and solid angles [h, w] of the texel centres of an h x w lat-long map."""
    theta = np.pi * (np.arange(h) + 0.5) / h
    phi = 2 * np.pi * ((np.arange(w) + 0.5) / w - 0.5)
    t, p = np.meshgrid(theta, phi, indexing="ij")
    d = np.stack([np.sin(t) * np.sin(p), np.cos(t), -np.sin(t) * np.cos(p)], -1)
    return d, np.sin(t) * (np.pi / h) * (2 * np.pi / w)


def sh9_irradiance(latlong):
    """float64 [9, 3] SH coefficients of irradiance / pi for a radiance map [h, w, 3]."""
    L = np.asarray(latlong, np.float64)
    d, dw = latlong_dirs(L.shape[0], L.shape[1])
    coef = np.einsum("hwk,hw,hwc->kc", sh9_basis(d), dw, L)
    band = np.array([1.0, 2 / 3, 2 / 3, 2 / 3, 0.25, 0.25, 0.25, 0.25, 0.25])  # A_l / pi: pi, 2 pi / 3, pi / 4
    return coef * band[:, None]


def _safe_normalize(v):
    l = np.sqrt(np.fmax(_dot(v, v), F32(1e-20)))
    return v / l[..., None]


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _interp(b, a):
    """(b0 a0 + b1 a1) + b2 a2 for b [N, 3], a [N, 3 vertices, 3]."""
    return (b[:, 0, None] * a[:, 0] + b[:, 1, None] * a[:, 1]) + b[:, 2, None] * a[:, 2]


def shade_fragments(verts, v_nrm, faces, mvp, campos, fres, face, px, py, sh, kd):
    """Linear RGB [N, 3] of faces `face` [N] at sub-pixel centres (px, py) [N], and a drawn flag [N]."""
    verts, v_nrm = np.asarray(verts, F32), np.asarray(v_nrm, F32)
    tri = np.asarray(faces, np.int64)[face]                                  # [N, 3]
    x, y, _, area, drawn, _ = ro.setup(verts, tri, mvp, fres)
    with np.errstate(all="ignore"):
        e = np.stack([ro.edge_fn(x[:, 1], y[:, 1], x[:, 2], y[:, 2], px, py), ro.edge_fn(x[:, 2], y[:, 2], x[:, 0], y[:, 0], px, py),
                      ro.edge_fn(x[:, 0], y[:, 0], x[:, 1], y[:, 1], px, py)], -1)
        p, n = verts[tri], v_nrm[tri]                                        # [N, 3, 3]
        w = ro.mvp_rows(mvp, p)[..., 3]
        q = (e / area[:, None]) / w
        qs = (q[:, 0] + q[:, 1]) + q[:, 2]
        b = q / qs[:, None]
        pos = _interp(b, p)
        smooth = _safe_normalize(_interp(b, n))
        view = _safe_normalize(np.asarray(campos, F32)[None] - pos)
        geom = _safe_normalize(_cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]))
        flip = ~(_dot(geom, view) > 0)
        smooth = np.where(flip[:, None], -smooth, smooth)
        geom = np.where(flip[:, None], -geom, geom)
        t = np.fmin(np.fmax(_dot(view, smooth) / NORMAL_THRESHOLD, F32(0)), F32(1))
        s = geom + t[:, None] * (smooth - geom)
        X, Y, Z = s[:, 0], s[:, 1], s[:, 2]
        basis = [np.full_like(X, _C0), _C1 * Y, _C1 * Z, _C1 * X, (_C2 * X) * Y, (_C2 * Y) * Z,
                 _C20 * (F32(3) * (Z * Z) - F32(1)), (_C2 * X) * Z, _C22 * (X * X - Y * Y)]
        sh = np.asarray(sh, F32).reshape(9, 3)
        E = sh[0][None] * basis[0][:, None]
        for i in range(1, 9):
            E = E + sh[i][None] * basis[i][:, None]
        col = np.asarray(kd, F32)[None] * np.fmax(E, F32(0))
    return col.astype(F32), drawn


def shade(verts, v_nrm, faces, mvp, campos, res, ssaa, face_id, sh, kd, bg, thresholds=None):
    """One job -> uint8 [res, res, 3], as mdb_render_shade computes it from face_id [res * ssaa, res * ssaa]."""
    sres = res * ssaa
    face_id = np.asarray(face_id)
    assert face_id.shape == (sres, sres)
    col = np.broadcast_to(np.asarray(bg, F32), (sres, sres, 3)).copy()
    rows, cols = np.nonzero(face_id >= 0)
    if rows.size:
        c, drawn = shade_fragments(verts, v_nrm, faces, mvp, campos, F32(sres), face_id[rows, cols],
                                   cols.astype(F32) + F32(0.5), rows.astype(F32) + F32(0.5), sh, kd)
        col[rows[drawn], cols[drawn]] = c[drawn]
    acc = np.zeros((res, res, 3), F32)
    for a in range(ssaa):
        for b in range(ssaa):
            acc = acc + col[a::ssaa, b::ssaa]
    return encode_srgb(acc / F32(ssaa * ssaa), thresholds)


def render(verts, faces, v_nrm, mvp, campos, res, ssaa, sh, kd, bg):
    """Rasterize at res * ssaa with raster_oracle, then shade: -> (uint8 [res, res, 3], face_id, n_behind)."""
    _, face_id, behind = ro.rasterize(verts, faces, mvp, res * ssaa)
    return shade(verts, v_nrm, faces, mvp, campos, res, ssaa, face_id, sh, kd, bg), face_id, behind
