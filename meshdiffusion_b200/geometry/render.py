"""Shaded previews of meshes: the image nvdiffrec/eval.py writes next to every generated mesh "for fast sanity check".

eval.py renders each raw marching-tets mesh once with nvdiffrast: the `'diffuse'` bsdf with kd = (0.75, 0.3, 0.6), the
environment light of configs/res64.json, a white background and the display camera `rotate_scene(angle_ind)` at
1000 x 1000. Here the same picture comes from the library's own kernels (csrc/raster.cu):

* `view_camera` -- eval.py's display camera (model-view and model-view-projection);
* `sh9_irradiance` -- the diffuse part of an environment light: the 9-term SH projection of a lat-long radiance map,
  the quantity nvdiffrec's prefiltered diffuse cube holds (irradiance / pi);
* `render_meshes` -- a face-id pass at res * ssaa (`mdb_raster_depth`) and the shading pass (`mdb_render_shade`):
  perspective-correct normals, nvdiffrec's two-sided shading normal, kd * E(n) / pi, a box resolve and sRGB;
* `read_hdr` / `write_png` -- Radiance `.hdr` in, 8-bit RGB PNG out, with numpy and the standard library only.

Without `render.envmap` the light is a small procedural sky (`default_envmap`) projected the same way.
"""
import struct
import zlib

import numpy as np
import torch

from .. import _native
from . import singleview

EVAL_RADIUS = 3.0                # RADIUS of nvdiffrec/eval.py (fit_singleview.py's validation camera uses 2.0)
DEFAULT_VIEW = 25                # eval.py --angle-ind default
DEFAULT_RES = 1000               # train_res of configs/res64.json (display_res defaults to it)
DEFAULT_SSAA = 2
KD = (0.75, 0.3, 0.6)            # eval.py's diffuse material
BACKGROUND = (1.0, 1.0, 1.0)     # "background": "white" of configs/res64.json (linear; sRGB white)
MAX_SSAA = 4
MAX_RASTER_RES = 16384


def view_camera(view, res=DEFAULT_RES, radius=EVAL_RADIUS):
    """(mv, mvp) fp32 [4, 4] of eval.py's `rotate_scene(FLAGS, view)` for a square res x res image. With
    `radius=singleview.RADIUS` the mvp is bitwise `singleview.view_mvp(view, res)`."""
    ang = (view / singleview.VIEWS_PER_TURN) * np.pi * 2
    mv = singleview._translate(0, 0, -radius) @ (singleview._rotate_x(-0.4) @ singleview._rotate_y(ang))
    return mv, singleview._perspective(singleview.FOVY, res / res, singleview.NEAR, singleview.FAR) @ mv


def camera_position(mv):
    """World-space camera position fp32 [3]: the translation of the inverse model-view (eval.py's `campos`)."""
    return torch.linalg.inv(torch.as_tensor(mv, dtype=torch.float64))[:3, 3].float()


# ---- light ---------------------------------------------------------------------------------------------------------

def latlong_directions(h, w):
    """float64 unit directions [h, w, 3] and solid angles [h, w] of the texel centres of an h x w lat-long map, in nvdiffrec's
    latlong_to_cubemap convention: theta = pi (i + 1/2) / h, phi = 2 pi ((j + 1/2) / w - 1/2),
    d = (sin theta sin phi, cos theta, -sin theta cos phi)."""
    theta = np.pi * (np.arange(h) + 0.5) / h
    phi = 2 * np.pi * ((np.arange(w) + 0.5) / w - 0.5)
    t, p = np.meshgrid(theta, phi, indexing="ij")
    d = np.stack([np.sin(t) * np.sin(p), np.cos(t), -np.sin(t) * np.cos(p)], -1)
    return d, np.sin(t) * (np.pi / h) * (2 * np.pi / w)


def _sh9(d):
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    c0, c1, c2 = 0.5 / np.sqrt(np.pi), np.sqrt(3 / (4 * np.pi)), 0.5 * np.sqrt(15 / np.pi)
    c20, c22 = 0.25 * np.sqrt(5 / np.pi), 0.25 * np.sqrt(15 / np.pi)
    return np.stack([np.full_like(x, c0), c1 * y, c1 * z, c1 * x, c2 * x * y, c2 * y * z, c20 * (3 * z * z - 1),
                     c2 * x * z, c22 * (x * x - y * y)], -1)


# clamped-cosine convolution per band (pi, 2 pi / 3, pi / 4), divided by pi
_BAND = np.array([1.0, 2 / 3, 2 / 3, 2 / 3, 0.25, 0.25, 0.25, 0.25, 0.25])


def sh9_irradiance(latlong):
    """float64 [9, 3]: SH coefficients (order Y00, Y1-1, Y10, Y11, Y2-2, Y2-1, Y20, Y21, Y22) of irradiance / pi for a
    lat-long radiance map [h, w, 3], each texel weighted by its solid angle. `mdb_render_shade` takes them as they are."""
    L = np.asarray(latlong, np.float64)
    if L.ndim != 3 or L.shape[2] < 3:
        raise ValueError(f"expected a lat-long map [h, w, 3], got {L.shape}")
    d, dw = latlong_directions(L.shape[0], L.shape[1])
    return np.einsum("hwk,hw,hwc->kc", _sh9(d), dw, L[..., :3]) * _BAND[:, None]


def default_envmap(h=64, w=128):
    """A procedural lat-long radiance map [h, w, 3] for when no `.hdr` is given: a sky over a darker ground, blended across
    the horizon, and one soft key light above and in front of the default view (its camera sits at -z, above the
    object)."""
    d, _ = latlong_directions(h, w)
    up = np.clip(d[..., 1] / 0.2 * 0.5 + 0.5, 0, 1)[..., None]
    sky, ground = np.array([0.70, 0.75, 0.85]), np.array([0.30, 0.27, 0.25])
    L = ground * (1 - up) + sky * up
    key = np.array([0.45, 0.75, -0.5])
    key /= np.linalg.norm(key)
    lobe = np.exp((d @ key - 1) / 0.02)[..., None]
    return L + 6.0 * np.array([1.0, 0.97, 0.92]) * lobe


def environment_light(envmap=None):
    """float64 [9, 3] irradiance coefficients of the `.hdr` at `envmap`, or of `default_envmap()` when it is None."""
    return sh9_irradiance(read_hdr(envmap) if envmap else default_envmap())


def srgb_thresholds():
    """fp32 [255], ascending: output code k (1..255) starts at the linear value whose sRGB is (k - 0.5) / 255, so the code
    of x is the number of thresholds it reaches: the reference's rint(clip(srgb(x), 0, 1) * 255). Computed in float64."""
    s = (np.arange(1, 256) - 0.5) / 255
    return np.where(s <= 0.04045, s / 12.92, ((s + 0.055) / 1.055) ** 2.4).astype(np.float32)


# ---- files ---------------------------------------------------------------------------------------------------------

def read_hdr(path):
    """Radiance RGBE `.hdr` -> float32 [h, w, 3], top row first. Header, a `-Y h +X w` resolution line, then flat or
    new-style run-length scanlines; a pixel decodes as m * 2^(e - 136), and 0 when e = 0 (rgbe.c)."""
    with open(path, "rb") as fh:
        data = fh.read()
    if not data.startswith(b"#?"):
        raise ValueError(f"{path}: not a Radiance file")
    pos = 0
    while True:
        nl = data.find(b"\n", pos)
        if nl < 0:
            raise ValueError(f"{path}: truncated header")
        line, pos = data[pos:nl].strip(), nl + 1
        if not line:
            break
        if line.startswith(b"FORMAT=") and line != b"FORMAT=32-bit_rle_rgbe":
            raise ValueError(f"{path}: unsupported {line.decode(errors='replace')}")
    nl = data.find(b"\n", pos)
    parts = data[pos:nl].split()
    if len(parts) != 4 or parts[0] != b"-Y" or parts[2] != b"+X":
        raise ValueError(f"{path}: unsupported resolution line {data[pos:nl]!r}")
    h, w = int(parts[1]), int(parts[3])
    buf = np.frombuffer(data, np.uint8, offset=nl + 1)
    out = np.empty((h, w, 4), np.uint8)
    p = 0
    for row in range(h):
        head = buf[p:p + 4]
        if not (8 <= w <= 0x7fff and head.size == 4 and head[0] == 2 and head[1] == 2 and not head[2] & 0x80):
            if p + 4 * w > buf.size:
                raise ValueError(f"{path}: truncated scanline {row}")
            out[row] = buf[p:p + 4 * w].reshape(w, 4)
            p += 4 * w
            continue
        if (int(head[2]) << 8 | int(head[3])) != w:
            raise ValueError(f"{path}: scanline {row} has the wrong width")
        p += 4
        for ch in range(4):
            x = 0
            while x < w:
                if p >= buf.size:
                    raise ValueError(f"{path}: truncated scanline {row}")
                n = int(buf[p])
                if n > 128:  # a run of n - 128 copies of the next byte
                    n -= 128
                    if n > w - x or p + 1 >= buf.size:
                        raise ValueError(f"{path}: bad run in scanline {row}")
                    out[row, x:x + n, ch] = buf[p + 1]
                    p += 2
                else:        # n literal bytes
                    if n == 0 or n > w - x or p + 1 + n > buf.size:
                        raise ValueError(f"{path}: bad literal in scanline {row}")
                    out[row, x:x + n, ch] = buf[p + 1:p + 1 + n]
                    p += 1 + n
                x += n
    e = out[..., 3].astype(np.int32)
    rgb = np.ldexp(out[..., :3].astype(np.float32), (e - 136)[..., None])
    return np.where((e == 0)[..., None], np.float32(0), rgb).astype(np.float32)


def write_png(path, rgb, level=1):
    """uint8 [h, w, 3] -> an 8-bit RGB PNG (no filtering, zlib `level`). Level 1 compresses a 1000 x 1000 preview about
    twice as fast as zlib's default 6, and the file is under 5% larger."""
    rgb = np.ascontiguousarray(np.asarray(rgb, np.uint8))
    if rgb.ndim != 3 or rgb.shape[2] != 3:
        raise ValueError(f"expected uint8 [h, w, 3], got {rgb.shape}")
    h, w, _ = rgb.shape
    raw = np.zeros((h, 1 + 3 * w), np.uint8)  # filter type 0 per row
    raw[:, 1:] = rgb.reshape(h, 3 * w)

    def chunk(tag, body):
        return struct.pack(">I", len(body)) + tag + body + struct.pack(">I", zlib.crc32(tag + body) & 0xffffffff)

    with open(path, "wb") as fh:
        fh.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
                 + chunk(b"IDAT", zlib.compress(raw.tobytes(), level)) + chunk(b"IEND", b""))
    return path


# ---- rendering -----------------------------------------------------------------------------------------------------

def _shade_packed(verts, v_nrm, faces, vert_off, face_off, job_mesh, mvp, campos, res, ssaa, face_id, params, out):
    sh, kd, bg, thr = params
    _native.check(_native.lib().mdb_render_shade(
        _native.ptr(verts), _native.ptr(v_nrm), _native.ptr(faces), _native.ptr(vert_off), _native.ptr(face_off),
        _native.ptr(job_mesh), _native.ptr(mvp), _native.ptr(campos), job_mesh.shape[0], res, ssaa, _native.ptr(face_id),
        _native.ptr(sh), _native.ptr(kd), _native.ptr(bg), _native.ptr(thr), _native.ptr(out), _native.current_stream()))


def render_meshes(meshes, normals, views=(DEFAULT_VIEW,), res=DEFAULT_RES, ssaa=DEFAULT_SSAA, light=None):
    """Preview images of every mesh from every view -> uint8 [M, V, res, res, 3] on the meshes' CUDA device.

    meshes: list of M (verts fp32 [Nv, 3], faces int [F, 3]); normals: list of M smooth vertex normals [Nv, 3]
    (mesh_ops.auto_normals); views: eval.py display views (`view_camera`); light: [9, 3] irradiance coefficients
    (`sh9_irradiance`), default `environment_light()`. The faces are rasterized at res * ssaa and every output pixel
    averages its ssaa x ssaa sub-pixels before the sRGB step. Row 0 is the top of the picture. Raises if a triangle has a
    vertex at w <= 0 (there is no near-plane clipping)."""
    res, ssaa = int(res), int(ssaa)
    if not 1 <= ssaa <= MAX_SSAA:
        raise ValueError(f"ssaa must be in [1, {MAX_SSAA}], got {ssaa}")
    if not 1 <= res * ssaa <= MAX_RASTER_RES:
        raise ValueError(f"res * ssaa must be in [1, {MAX_RASTER_RES}], got {res} * {ssaa}")
    if len(normals) != len(meshes):
        raise ValueError("one normal array per mesh")
    views = tuple(int(v) for v in views)
    M, V = len(meshes), len(views)
    dev = meshes[0][0].device
    cams = [view_camera(v, res) for v in views]
    mvps = torch.stack([mvp for _, mvp in cams])
    cam = torch.stack([camera_position(mv) for mv, _ in cams]).to(dev).repeat(M, 1).contiguous()
    verts, faces, vert_off, face_off = singleview._pack(meshes, dev)
    v_nrm = torch.cat([n.reshape(-1, 3) for n in normals]).to(dev, torch.float32).contiguous()
    if v_nrm.shape != verts.shape:
        raise ValueError("every mesh needs one normal per vertex")
    job_mesh, mvp = singleview._jobs(M, mvps, dev)
    light = environment_light() if light is None else light
    f32 = dict(device=dev, dtype=torch.float32)
    params = (torch.as_tensor(np.asarray(light, np.float64).reshape(9, 3), **f32).contiguous(), torch.tensor(KD, **f32),
              torch.tensor(BACKGROUND, **f32), torch.from_numpy(srgb_thresholds()).to(dev))
    out = torch.empty(M * V, res, res, 3, device=dev, dtype=torch.uint8)
    sres = res * ssaa
    step = max(1, singleview._MAX_JOB_PIXELS // (sres * sres))
    for j0 in range(0, M * V, step):
        jm, mv = job_mesh[j0:j0 + step].contiguous(), mvp[j0:j0 + step].contiguous()
        _, face_id = singleview._raster_packed(verts, faces, vert_off, face_off, jm, mv, sres)
        _shade_packed(verts, v_nrm, faces, vert_off, face_off, jm, mv, cam[j0:j0 + step], res, ssaa, face_id, params,
                      out[j0:j0 + step])
    return out.view(M, V, res, res, 3)
