"""CPU: the shared library builds for sm_90a, loads, and exports every symbol the header declares (no compute)."""
import ctypes
import os
import re

from helpers import ROOT, tiny_config


def _declared():
    text = open(os.path.join(ROOT, "include", "meshdiff_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(mdb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from meshdiffusion_b200 import _native
    L = _native.lib()
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} is declared in include/meshdiff_b200.h but not exported"
    assert set(names) == set(_native.SIGNATURES), "ctypes signature table and header disagree"
    assert L.mdb_version() == 100


def test_sass_contains_wgmma_and_tma():
    """The .so must carry Hopper warpgroup-MMA / TMA SASS (HGMMA, UTMALDG) and no other architecture, i.e. it really is the
    sm_90a path."""
    import shutil
    import subprocess
    from meshdiffusion_b200 import _native
    _native.lib()
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", _native.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"arch = (sm_\w+)", sass))
    assert archs == {"sm_90a"}, archs
    for mnemonic in ("HGMMA", "UTMALDG"):
        assert mnemonic in sass, f"{mnemonic} missing from the SASS"


def test_dry_plan_errors_are_reported_not_thrown():
    from meshdiffusion_b200 import _native
    L = _native.lib()
    cfg = _native.UNetConfigC()
    cfg.image_size, cfg.nf, cfg.n_levels = 60, 128, 5  # 60 is not divisible by 2^4
    for i, v in enumerate([1, 1, 2, 4, 4]):
        cfg.ch_mult[i] = v
    cfg.num_res_blocks, cfg.level0_blocks, cfg.n_attn, cfg.num_channels, cfg.stem_ksize = 3, -1, 0, 4, 3
    cfg.max_batch = 1
    h = ctypes.c_void_p()
    rc = L.mdb_unet_create_dry(ctypes.byref(cfg), ctypes.byref(h))
    assert rc != 0 and b"image_size" in L.mdb_last_error()


def test_dry_plan_refuses_to_run():
    """The steps of a dry plan hold null pointers: the entry points that would run it report an error before anything is
    enqueued (so this needs no GPU)."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    cfg = ddpm._config_c(ddpm.arch_from_config(tiny_config("res64", "bf16")), 1, "bf16")
    h = ctypes.c_void_p()
    _native.check(L.mdb_unet_create_dry(ctypes.byref(cfg), ctypes.byref(h)))
    try:
        assert L.mdb_unet_commit(h, None) != 0
        assert b"a dry plan cannot run" in L.mdb_last_error()
        assert L.mdb_unet_forward(h, None, None, None, 1, None) != 0
        assert b"a dry plan cannot run" in L.mdb_last_error()
    finally:
        L.mdb_unet_destroy(h)


def test_groupnorm_entry_points_refuse_null_stats():
    """The GroupNorm kernels derive mean / rstd from `stats` and have no other source of them: a NULL `stats` is an error
    reported before anything is launched (so this needs no GPU)."""
    from meshdiffusion_b200 import _native
    L = _native.lib()
    B, V, C = 1, 8, 32
    assert L.mdb_groupnorm_act(None, None, None, None, None, B, V, C, 1, 0, None) != 0
    assert b"stats" in L.mdb_last_error()
    assert L.mdb_groupnorm_act_backward(None, None, None, None, None, None, None, None, None, B, V, C, 1, 0.0, 0, None) != 0
    assert b"stats" in L.mdb_last_error()
    for precision in (0, 2):
        assert L.mdb_groupnorm_act_backward_prec(None, None, None, None, None, None, None, None, None, B, V, C, 1, 0.0, 0,
                                                 precision, None) != 0
        assert b"stats" in L.mdb_last_error()
