"""CPU: the float32 shading oracle on hand-built scenes (uniform colour under a constant light, upright images, two-sided
shading, supersampling of fully covered pixels), the SH projection of lat-long maps, the `.hdr` reader, the PNG writer,
the shading entry point's size checks, and `--mode=export`'s command line."""
import os
import struct
import zlib

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import render_oracle as rdo

KD = (0.75, 0.3, 0.6)
WHITE = (1.0, 1.0, 1.0)
QUAD_V = np.array([[-0.6, -0.6, 0], [0.6, -0.6, 0], [0.6, 0.6, 0], [-0.6, 0.6, 0]], np.float32)
QUAD_F = np.array([[0, 1, 2], [0, 2, 3]])


def _front_camera(res):
    """A camera on +z at distance 3 looking at the origin: (mvp, campos)."""
    from meshdiffusion_b200.geometry import singleview as sv
    mv = sv._translate(0, 0, -3.0)
    mvp = sv._perspective(sv.FOVY, 1.0, sv.NEAR, sv.FAR) @ mv
    return mvp.numpy(), np.array([0, 0, 3.0], np.float32)


def _srgb_code(x):
    x = np.clip(np.asarray(x, np.float64), 0, 1)
    s = np.where(x <= 0.0031308, x * 12.92, 1.055 * x ** (1 / 2.4) - 0.055)
    return s * 255


def _light():
    from meshdiffusion_b200.geometry import render
    return render.environment_light().astype(np.float32)


def test_thresholds_and_encoding_match_the_reference_rounding():
    from meshdiffusion_b200.geometry import render
    t = render.srgb_thresholds()
    assert t.dtype == np.float32 and t.shape == (255,) and (np.diff(t) > 0).all()
    np.testing.assert_array_equal(t, rdo.srgb_thresholds())
    x = np.random.default_rng(0).uniform(-0.1, 1.2, 200000).astype(np.float32)
    want = _srgb_code(x)
    clear = np.abs(want - np.floor(want) - 0.5) > 1e-4  # away from exact halves, where rint and the table may differ
    np.testing.assert_array_equal(rdo.encode_srgb(x)[clear], np.rint(want[clear]).astype(np.uint8))
    assert rdo.encode_srgb(np.array([np.nan, -1, 0, 1, 5], np.float32)).tolist() == [0, 0, 0, 255, 255]


def test_view_camera_matches_view_mvp_and_eval_campos():
    from meshdiffusion_b200.geometry import render, singleview
    for v in (0, 13, 25, 49):
        _, mvp = render.view_camera(v, 1000, radius=singleview.RADIUS)
        assert torch.equal(mvp, singleview.view_mvp(v, 1000))
    mv, _ = render.view_camera(25, 1000)
    cam = render.camera_position(mv)
    # eval.py's default view: radius 3, pitched up by 0.4 rad, on the -z side after half a turn
    np.testing.assert_allclose(cam.numpy(), [0, 3 * np.sin(0.4), -3 * np.cos(0.4)], atol=1e-5)


def test_flat_quad_under_constant_light_is_one_colour():
    res = 32
    mvp, cam = _front_camera(res)
    L = np.array([0.8, 0.9, 0.7])
    sh = rdo.sh9_irradiance(np.broadcast_to(L, (32, 64, 3)))
    nrm = np.tile(np.array([[0, 0, 1]], np.float32), (4, 1))
    img, face_id, behind = rdo.render(QUAD_V, QUAD_F, nrm, mvp, cam, res, 2, sh.astype(np.float32), KD, WHITE)
    assert behind == 0 and img.dtype == np.uint8 and img.shape == (res, res, 3)
    full = (face_id >= 0).reshape(res, 2, res, 2).all((1, 3))
    assert 100 < full.sum() < res * res
    colours = np.unique(img[full], axis=0)
    want = _srgb_code(np.array(KD) * L)
    assert (np.abs(want - np.floor(want) - 0.5) > 0.05).all()
    np.testing.assert_array_equal(colours, np.rint(want)[None].astype(np.uint8))
    empty = (face_id < 0).reshape(res, 2, res, 2).all((1, 3))
    assert (img[empty] == 255).all() and empty[0, 0]


def test_triangle_above_the_origin_is_in_the_top_half():
    from meshdiffusion_b200.geometry import render
    res = 48
    mv, mvp = render.view_camera(25, res)
    cam = render.camera_position(mv).numpy()
    for y0, top in ((0.3, True), (-0.6, False)):
        v = np.array([[-0.2, y0, 0], [0.2, y0, 0], [0, y0 + 0.3, 0]], np.float32)
        n = np.tile(np.array([[0, 1, 0]], np.float32), (3, 1))
        img, face_id, _ = rdo.render(v, np.array([[0, 1, 2]]), n, mvp.numpy(), cam, res, 1, _light(), KD, WHITE)
        rows = np.nonzero((img != 255).any(-1))[0]
        assert rows.size and (face_id >= 0).any()
        assert (rows < res // 2).all() if top else (rows >= res // 2).all()


def test_back_facing_quad_is_shaded_like_the_front_facing_one():
    res = 24
    mvp, cam = _front_camera(res)
    sh = _light()
    front, _, _ = rdo.render(QUAD_V, QUAD_F, np.tile([[0, 0, 1]], (4, 1)).astype(np.float32), mvp, cam, res, 2, sh, KD, WHITE)
    back, _, _ = rdo.render(QUAD_V, QUAD_F[:, ::-1], np.tile([[0, 0, -1]], (4, 1)).astype(np.float32), mvp, cam, res, 2, sh,
                            KD, WHITE)
    assert (front != 255).any()
    np.testing.assert_array_equal(front, back)


def test_supersampling_keeps_fully_covered_pixels():
    res = 20
    mvp, cam = _front_camera(res)
    sh = _light()
    nrm = np.tile(np.array([[0, 0, 1]], np.float32), (4, 1))
    quad = QUAD_V * np.float32(0.9)  # edges that cut pixels: X = 5.65 and 14.35
    imgs, full = [], np.ones((res, res), bool)
    for s in (1, 2, 3):
        img, face_id, _ = rdo.render(quad, QUAD_F, nrm, mvp, cam, res, s, sh, KD, WHITE)
        imgs.append(img)
        full &= (face_id >= 0).reshape(res, s, res, s).all((1, 3))
    assert full.sum() > 50
    for img in imgs[1:]:
        np.testing.assert_array_equal(img[full], imgs[0][full])
    assert (imgs[1] != imgs[0]).any()  # the edges do change


def test_sh_projection_of_a_constant_map():
    from meshdiffusion_b200.geometry import render
    L = np.array([0.5, 1.0, 2.0])
    sh = render.sh9_irradiance(np.broadcast_to(L, (48, 96, 3)))
    np.testing.assert_allclose(sh, rdo.sh9_irradiance(np.broadcast_to(L, (48, 96, 3))), rtol=1e-12, atol=1e-15)
    # E / pi of a constant radiance L is L: c00 Y00 = L; midpoint quadrature of the sphere is good to ~1e-3
    np.testing.assert_allclose(sh[0] * 0.5 / np.sqrt(np.pi), L, rtol=2e-3)
    # the rest vanish: exactly by symmetry, except the two l = 2 terms that see the map's polar axis (y), which vanish to
    # the quadrature error in theta
    assert np.abs(np.delete(sh, [0, 6, 8], axis=0)).max() < 1e-12
    assert (np.abs(sh[[6, 8]]) < 1e-3 * L).all()


def test_sh_projection_of_one_bright_texel_is_the_clamped_cosine_lobe():
    from meshdiffusion_b200.geometry import render
    h, w, i, j, P = 32, 64, 9, 40, 50.0
    m = np.zeros((h, w, 3))
    m[i, j] = P
    sh = render.sh9_irradiance(m)
    d, dw = render.latlong_directions(h, w)
    light = d[i, j]
    assert light[1] > 0.5  # texel (9, 40) is above the horizon
    n = np.random.default_rng(1).normal(size=(500, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    got = rdo.sh9_basis(n) @ sh[:, 0]
    cos = n @ light
    scale = P * dw[i, j] / np.pi
    # the exact SH9 truncation of max(cos, 0) / pi: (1 + 2 t + 5/8 (3 t^2 - 1)) / 4 per unit of P dw
    np.testing.assert_allclose(got, scale * (1 + 2 * cos + 0.625 * (3 * cos ** 2 - 1)) / 4, rtol=1e-9, atol=1e-12 * scale)
    # which stays within 10% of the lobe's peak of the clamped cosine itself
    assert np.abs(got - scale * np.maximum(cos, 0)).max() < 0.1 * scale


def _rgbe(rgb):
    """float [..., 3] -> RGBE bytes as rgbe.c's float2rgbe writes them."""
    rgb = np.asarray(rgb, np.float64)
    v = rgb.max(-1)
    mant, ex = np.frexp(v)
    scale = np.where(v < 1e-32, 0, mant * 256 / np.where(v == 0, 1, v))
    out = np.zeros(rgb.shape[:-1] + (4,), np.uint8)
    out[..., :3] = np.where(v[..., None] < 1e-32, 0, np.floor(rgb * scale[..., None]))
    out[..., 3] = np.where(v < 1e-32, 0, ex + 128)
    return out


def _rle_channel(vals):
    """New-style run-length encoding of one channel of a scanline: runs of 3 or more, literals otherwise."""
    out, k = bytearray(), 0
    while k < len(vals):
        r = 1
        while k + r < len(vals) and vals[k + r] == vals[k] and r < 127:
            r += 1
        if r >= 3:
            out += bytes([128 + r, vals[k]])
            k += r
            continue
        start = k
        while k < len(vals) and k - start < 128 and not (k + 2 < len(vals) and vals[k] == vals[k + 1] == vals[k + 2]):
            k += 1
        out += bytes([k - start]) + bytes(vals[start:k])
    return bytes(out)


def test_read_hdr_flat_and_run_length_scanlines(tmp_path):
    from meshdiffusion_b200.geometry import render
    h, w = 4, 12
    rng = np.random.default_rng(5)
    img = rng.uniform(0, 8, (h, w, 3))
    img[1, 2:9] = [0.25, 1.5, 3.0]     # a run in every channel
    img[2, :] = 0.0                    # e = 0 decodes to 0
    img[3, 5] = [1e3, 1e-2, 1.0]
    px = _rgbe(img)
    body = bytearray(px[0].tobytes())  # row 0 flat
    for r in range(1, h):              # rows 1..3 new-style RLE
        body += bytes([2, 2, w >> 8, w & 255])
        for ch in range(4):
            body += _rle_channel(list(px[r, :, ch]))
    assert any(b > 128 for b in body[4 * w:])  # the encoding has runs
    path = tmp_path / "t.hdr"
    path.write_bytes(b"#?RADIANCE\n# test\nFORMAT=32-bit_rle_rgbe\nEXPOSURE=1.0\n\n" + f"-Y {h} +X {w}\n".encode() + bytes(body))
    got = render.read_hdr(str(path))
    m, e = px[..., :3].astype(np.float64), px[..., 3:].astype(np.int64)
    want = np.where(e == 0, 0.0, m * np.exp2(e - 136.0)).astype(np.float32)
    assert got.dtype == np.float32 and got.shape == (h, w, 3)
    np.testing.assert_array_equal(got, want)
    assert (got[2] == 0).all()
    assert (np.abs(got - img) <= img.max(-1, keepdims=True) * 2 ** -7).all()  # 8 bits of mantissa shared by a pixel
    # narrower than 8 pixels: always flat
    path2 = tmp_path / "narrow.hdr"
    path2.write_bytes(b"#?RGBE\n\n-Y 2 +X 3\n" + px[:2, :3].tobytes())
    np.testing.assert_array_equal(render.read_hdr(str(path2)), want[:2, :3])
    path3 = tmp_path / "bad.hdr"
    path3.write_bytes(b"#?RADIANCE\n\n+Y 2 +X 3\n")
    with pytest.raises(ValueError, match="resolution"):
        render.read_hdr(str(path3))


def test_write_png_round_trip(tmp_path):
    from meshdiffusion_b200.geometry import render
    rgb = np.random.default_rng(2).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    path = render.write_png(str(tmp_path / "x.png"), rgb)
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(tag + body) & 0xffffffff
        chunks.append((tag, body))
        pos += 12 + n
    assert [t for t, _ in chunks] == [b"IHDR", b"IDAT", b"IEND"]
    assert struct.unpack(">IIBBBBB", chunks[0][1]) == (53, 37, 8, 2, 0, 0, 0)
    raw = np.frombuffer(zlib.decompress(chunks[1][1]), np.uint8).reshape(37, 1 + 53 * 3)
    assert (raw[:, 0] == 0).all()
    np.testing.assert_array_equal(raw[:, 1:].reshape(37, 53, 3), rgb)


def test_default_light_is_positive_and_brighter_from_above():
    from meshdiffusion_b200.geometry import render
    sh = render.environment_light()
    assert sh.shape == (9, 3)
    n = np.random.default_rng(3).normal(size=(2000, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    E = rdo.sh9_basis(n) @ sh
    assert (E > 0).all()
    assert E[n[:, 1] > 0.9].mean() > 1.5 * E[n[:, 1] < -0.9].mean()


def test_shade_entry_point_checks_sizes_before_launching():
    """The checks run before anything is enqueued (so this needs no GPU)."""
    from meshdiffusion_b200 import _native
    L = _native.lib()
    args = [None] * 8

    def call(n_jobs, res, ssaa):
        return L.mdb_render_shade(*args, n_jobs, res, ssaa, None, None, None, None, None, None, None)

    assert call(0, 64, 2) == 0
    for n_jobs, res, ssaa, msg in ((1, 64, 0, b"ssaa"), (1, 64, 5, b"ssaa"), (1, 8192, 3, b"16384"), (1, 0, 1, b"resolution"),
                                   (70000, 64, 1, b"jobs")):
        assert call(n_jobs, res, ssaa) != 0
        assert msg in L.mdb_last_error()


def test_export_mode_parses_and_default_config_has_no_render_options():
    import main_diffusion
    cfg_path, mode, overrides = main_diffusion.parse_args([f"--config={ROOT}/configs/res64.py", "--mode=export",
                                                           "--config.render.views=(0, 25)", "--config.render.res=256",
                                                           "--config.render.ssaa=3", "--config.render.envmap=/x/env.hdr"])
    assert mode == "export"
    assert dict(overrides) == {"render.views": (0, 25), "render.res": 256, "render.ssaa": 3, "render.envmap": "/x/env.hdr"}
    from meshdiffusion_b200.diffusion import export
    for name in ("res64", "res128"):
        cfg = main_diffusion.load_config_file(os.path.join(ROOT, "configs", f"{name}.py"))
        assert cfg.render == {}  # the reference's empty `render` group
        assert export._render_options(cfg) == ((25,), 1000, 2, None)
        for dotted, value in overrides:
            cfg.set_by_path(dotted, value)
        assert export._render_options(cfg) == ((0, 25), 256, 3, "/x/env.hdr")
