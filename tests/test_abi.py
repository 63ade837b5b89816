"""CPU: the shared library builds for sm_90a, loads, and exports every symbol the header declares (no compute)."""
import ctypes
import os
import re

from helpers import ROOT


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
