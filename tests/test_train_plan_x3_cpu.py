"""Host-side checks of the split-bf16 (bf16x3) training plan and of how the score network selects its training operand
mode: plans are built GPU-less through mdb_unet_create_dry."""
import ctypes

import pytest

from helpers import full_config, tiny_config


def _dry(cfg, batch, precision, training=True):
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(cfg), batch, precision, training=training)
    h = ctypes.c_void_p()
    _native.check(L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)))
    try:
        arena = ctypes.c_longlong()
        _native.check(L.mdb_unet_info(h, None, ctypes.byref(arena), None, None))
        table = []
        for i in range(L.mdb_unet_num_params(h)):
            name, numel = ctypes.c_char_p(), ctypes.c_longlong()
            _native.check(L.mdb_unet_param_info(h, i, ctypes.byref(name), ctypes.byref(numel), None, None))
            table.append((name.value.decode(), numel.value))
        return arena.value, table
    finally:
        L.mdb_unet_destroy(h)


@pytest.mark.parametrize("name,batch", [("tiny", 3), ("res64", 1), ("res128", 1)])
def test_x3_training_plan_builds_and_frees_everything(name, batch):
    """Every activation / gradient / scratch block of the split-bf16 plan goes back to the arena (the builder throws on a
    leak), and the parameter table is the bf16 plan's."""
    cfg = tiny_config("res64", "bf16") if name == "tiny" else full_config(name, "bf16")
    a_bf16, t_bf16 = _dry(cfg, batch, "bf16")
    a_x3, t_x3 = _dry(cfg, batch, "bf16x3")
    a_inf, _ = _dry(cfg, batch, "bf16x3", training=False)
    assert t_x3 == t_bf16
    assert a_x3 > a_inf
    print(f"{name} B{batch}: training arena bf16 {a_bf16 / 2 ** 30:.3f} GB, bf16x3 {a_x3 / 2 ** 30:.3f} GB "
          f"({a_x3 / a_bf16:.2f}x)")
    if name == "res64":
        # split-bf16 tensors are twice the bytes; fp32 scratch (attention logits, split-K partials) is not
        assert a_x3 <= 2.2 * a_bf16


def test_score_net_training_mode_from_config():
    from meshdiffusion_b200.diffusion.models import ddpm
    cfg = tiny_config("res64", "bf16x3")
    assert ddpm.ScoreNet(cfg).train_precision == "bf16"  # default: the bf16 plan
    cfg.training.compute_dtype = "bf16x3"
    net = ddpm.ScoreNet(cfg)
    assert net.train_precision == "bf16x3"
    assert net.precision == "bf16x3"  # the inference mode is model.compute_dtype, independent of the training one
    for bad in ("tf32", "fp16"):
        cfg.training.compute_dtype = bad
        with pytest.raises(ValueError, match="training.compute_dtype"):
            ddpm.ScoreNet(cfg)


def test_x3_training_engine_refuses_tf32_still():
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(tiny_config("res64", "tf32")), 1, "tf32", training=True)
    h = ctypes.c_void_p()
    assert L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)) != 0
    assert b"bf16x3" in L.mdb_last_error()


def test_precision_entry_points_are_exported():
    from meshdiffusion_b200 import _native
    L = _native.lib()
    for name in ("mdb_conv3d_backward_prec", "mdb_groupnorm_act_backward_prec"):
        assert name in _native.SIGNATURES
        assert getattr(L, name) is not None
