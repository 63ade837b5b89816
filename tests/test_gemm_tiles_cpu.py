"""Tile shape of the forward GEMM launches (mdb_unet_gemm_tiles), from GPU-less plans: what tools/bench_gemm_ops.py groups
launches by for its per-tile fit."""
import ctypes

import pytest

from helpers import full_config


def _tiles(name, precision, batch):
    """{launch name: (work items, split-K factor, k-steps per tile, most k-steps per entry, BLOCK_N)} of a dry plan."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(full_config(name, precision)), batch, precision, training=False)
    h = ctypes.c_void_p()
    _native.check(L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)))
    try:
        ng = ctypes.c_int()
        _native.check(L.mdb_unet_info(h, None, None, ctypes.byref(ng), None))
        rows = {}
        for i in range(ng.value):
            nm = ctypes.c_char_p()
            v = [ctypes.c_int() for _ in range(5)]
            _native.check(L.mdb_unet_gemm_ops(h, i, ctypes.byref(nm), None, None))
            _native.check(L.mdb_unet_gemm_tiles(h, i, *[ctypes.byref(x) for x in v]))
            rows[nm.value.decode()] = tuple(x.value for x in v)
        assert L.mdb_unet_gemm_tiles(h, ng.value, None, None, None, None, None) != 0
        assert b"out of range" in L.mdb_last_error()
        return rows
    finally:
        L.mdb_unet_destroy(h)


@pytest.mark.parametrize("precision", ["bf16", "tf32", "bf16x3"])
def test_res64_halo_convolutions(precision):
    """At batch 32 the 64^3 convolutions of the first and last level are 32 * 64^3 / 128 = 65 536 tiles of 128 columns;
    27 taps in entries of three k-steps, over 256 input channels (conv0 of the last level, the concatenation with the
    skip) or 128 (conv1 of the first level)."""
    rows = _tiles("res64", precision, 32)
    per_64_channels = 1 if precision != "tf32" else 2  # a k-step covers 64 bf16 or 32 tf32 channels
    for name in ("res49.conv0", "res52.conv0"):
        assert rows[name] == (65536, 1, 4 * 27 * per_64_channels, 3, 128), (name, rows[name])
    for name in ("res4.conv1", "res5.conv1"):
        assert rows[name] == (65536, 1, 2 * 27 * per_64_channels, 3, 128), (name, rows[name])
    for work, splits, ksteps, entry_ksteps, block_n in rows.values():
        assert work > 0 and splits >= 1 and ksteps >= 1 and 1 <= entry_ksteps <= 5 and block_n in (32, 128)
