"""Host-side checks of the training (forward + backward) plan: built GPU-less through mdb_unet_create_dry."""
import ctypes

import pytest

from helpers import engine_report, full_config, tiny_config


def _dry(cfg, batch, training):
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(cfg), batch, "bf16", training=training)
    h = ctypes.c_void_p()
    _native.check(L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)))
    arena, n = ctypes.c_longlong(), L.mdb_unet_num_params(h)
    _native.check(L.mdb_unet_info(h, None, ctypes.byref(arena), None, None))
    L.mdb_unet_destroy(h)
    return arena.value, n


@pytest.mark.parametrize("name,batch", [("tiny", 3), ("res64", 1), ("res128", 1)])
def test_training_plan_builds_and_frees_everything(name, batch):
    """The backward emitters must hand every activation / gradient / scratch block back to the arena (the builder
    throws on a leak), and the plan must not change the parameter table."""
    cfg = tiny_config("res64", "bf16") if name == "tiny" else full_config(name, "bf16")
    a_inf, n_inf = _dry(cfg, batch, False)
    a_trn, n_trn = _dry(cfg, batch, True)
    assert n_inf == n_trn
    assert a_trn > a_inf
    if name == "res64":
        assert a_trn < 3.5 * 2 ** 30, "res64 training arena grew beyond 3.5 GB per sample"


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("name,batch", [("tiny", 3), ("res64", 1), ("res128", 1)])
def test_dry_training_plan_answers_backward_queries(name, batch, precision):
    """The dry plan is built by the engine's own builders, so without a GPU it knows the backward launches and after
    which of them each parameter gradient is final."""
    cfg = tiny_config("res64", "bf16") if name == "tiny" else full_config(name, "bf16")
    r = engine_report(cfg, batch, precision, training=True)
    n, ready = r["n_bwd_steps"], r["grad_ready"]
    assert n > 0 and r["bwd_flops"] > 0
    # never written by the backward: the grid mask, the coordinates and the pos_layer weight (ddpm_res64.py:148 feeds
    # coords * 0); res128 has no pos bias either
    never = {"mask", "pos_layer.weight"} | ({"pos_layer.bias"} if name == "res128" else {"coords"})
    assert {k for k, v in ready.items() if v == 0} == never
    assert all(1 <= v <= n for k, v in ready.items() if k not in never)
    # the time-embedding backward is the last launch
    temb = [k for k in ready if k.split(".")[:2] in (["all_modules", "0"], ["all_modules", "1"])]
    assert len(temb) == 4 and all(ready[k] == n for k in temb)
    # the head's emitter runs first: the head conv and its GroupNorm are final before any other gradient
    head = max(int(k.split(".")[1]) for k in ready if k.startswith("all_modules."))
    first = min(v for v in ready.values() if v)
    assert {k for k, v in ready.items() if v == first} == {f"all_modules.{m}.{p}" for m in (head - 1, head) for p in ("weight", "bias")}


def test_training_engine_refuses_tf32():
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    cfg = tiny_config("res64", "tf32")
    c = ddpm._config_c(ddpm.arch_from_config(cfg), 1, "tf32", training=True)
    h = ctypes.c_void_p()
    assert L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)) != 0
    assert b"bf16" in L.mdb_last_error()
