"""Operand ring depth of every forward GEMM launch, from GPU-less plans (mdb_unet_gemm_slots).

The accumulator staging of the implicit-GEMM epilogue takes 64 columns at a time, so the rings get the room for a third
weight slot in split-bf16 halo convolutions (a k-step's W_hi and W_lo tiles, 32 KB, may then be two k-steps ahead of
the MMAs instead of one) and a third A slot in bf16 / tf32 ones."""
import ctypes

import pytest

from helpers import full_config

SMEM_LIMIT = 232448  # the opt-in dynamic shared memory per block on sm_90


def _plan(name, precision):
    """[(launch name, A slots, B slots, dynamic shared memory bytes)] of a dry inference plan at batch 1."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(full_config(name, precision)), 1, precision, training=False)
    h = ctypes.c_void_p()
    _native.check(L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)))
    try:
        ng = ctypes.c_int()
        _native.check(L.mdb_unet_info(h, None, None, ctypes.byref(ng), None))
        rows = []
        for i in range(ng.value):
            nm, a, b, sm = ctypes.c_char_p(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
            _native.check(L.mdb_unet_gemm_ops(h, i, ctypes.byref(nm), None, None))
            _native.check(L.mdb_unet_gemm_slots(h, i, ctypes.byref(a), ctypes.byref(b), ctypes.byref(sm)))
            rows.append((nm.value.decode(), a.value, b.value, sm.value))
        return rows
    finally:
        L.mdb_unet_destroy(h)


def _multi_step_launches(name, monkeypatch):
    """Names of the launches whose load-table entries carry three or more k-steps (the halo convolutions). With the A
    ring held at two slots the picker adds B slots until they cover two entries' k-steps, and a bf16 plan has room for
    all of them: six or more B slots mean at least three k-steps per entry."""
    with monkeypatch.context() as m:
        m.setenv("MDB_MAX_STAGES", "2")
        m.delenv("MDB_MAX_BSLOTS", raising=False)
        return {nm for nm, a, b, _ in _plan(name, "bf16") if b >= 6}


@pytest.mark.parametrize("name", ["res64", "res128"])
def test_halo_convolutions_get_the_deeper_rings(name, monkeypatch):
    monkeypatch.delenv("MDB_MAX_STAGES", raising=False)
    monkeypatch.delenv("MDB_MAX_BSLOTS", raising=False)
    halo = _multi_step_launches(name, monkeypatch)
    assert len(halo) > 0
    for precision in ("bf16", "tf32", "bf16x3"):
        rows = _plan(name, precision)
        assert halo <= {r[0] for r in rows}
        for nm, a, b, smem in rows:
            assert smem <= SMEM_LIMIT, (precision, nm, smem)
            assert a >= 2 and b >= 2, (precision, nm, a, b)
            if nm in halo:
                if precision == "bf16x3":
                    assert b >= 3, (precision, nm, a, b)
                else:
                    assert a >= 3, (precision, nm, a, b)


@pytest.mark.parametrize("name", ["res64", "res128"])
@pytest.mark.parametrize("precision", ["bf16", "tf32", "bf16x3"])
def test_bslot_cap(name, precision, monkeypatch):
    monkeypatch.delenv("MDB_MAX_STAGES", raising=False)
    monkeypatch.setenv("MDB_MAX_BSLOTS", "2")
    for nm, a, b, smem in _plan(name, precision):
        assert b == 2, (nm, a, b)
        assert smem <= SMEM_LIMIT, (nm, smem)
