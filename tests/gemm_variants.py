"""Shared by test_gemm_probe_cpu.py and test_gpu_gemm_variants.py: the probe descriptions of the implicit-GEMM variants the
score network launches, their error gates, the operand rounding of the fp64 references and the engine's dry report.

Error metric everywhere: max |out - ref| / max |ref|, ref in fp64 from the operands as the kernel sees them (bf16-rounded,
or hi + lo for split bf16; tf32 operands stay fp32 in memory and are rounded inside the tensor core)."""
import ctypes

import torch

PRECISIONS = ("bf16", "bf16x3", "tf32")
PREC_ID = {"bf16": 0, "tf32": 1, "bf16x3": 2}
# Gates per family, from the gates of test_gpu_conv.py (tf32 2e-3, bf16 2e-2, bf16x3 1e-4) tightened to what the errors
# measured on an H100 SXM (700 W) support, about twice the largest of them: bf16 5.0e-3 (split-K vs S = 1; output
# rounding alone is 2^-9 of the largest value), bf16x3 2.0e-5, tf32 9.2e-4 (P.v; tf32 operands are rounded inside the
# tensor core, which the fp32 reference does not model). Statistics are held to the same gates.
_GATE = {"tf32": 2e-3, "bf16": 1e-2, "bf16x3": 5e-5}
GATES = {family: dict(_GATE) for family in ("split", "upsample", "attn", "nin")}
# GroupNorm backward (bf16 / split bf16 only). Largest errors measured on the same H100: bf16 8.8e-3 (dx, fused vs
# two-pass under dropout: dy rounded to bf16 at different points), so the bf16 gate of test_gpu_conv.py stays; bf16x3
# 1.9e-5, tightened like the others.
GATES["gnb"] = {"bf16": 2e-2, "bf16x3": 5e-5}
SENTINEL = 7.0  # exact in bf16 and fp32
GUARD = 4096    # sentinel elements on each side of an output


def rel_err(out, ref):
    out, ref = out.double(), ref.double()
    return (out - ref).abs().max().item() / max(ref.abs().max().item(), 1e-300)


def parts(precision):
    return 2 if precision == "bf16x3" else 1


def act_dtype(precision):
    return torch.float32 if precision == "tf32" else torch.bfloat16


def as_operand(x, precision):
    """x (float) as the kernel reads it, in fp64: bf16-rounded, hi + lo of split bf16, or fp32."""
    x = x.float()
    if precision == "tf32":
        return x.double()
    hi = x.to(torch.bfloat16)
    if precision == "bf16":
        return hi.double()
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi.double() + lo.double()


def pack_rows(x, precision):
    """Rows [..., W] (float) -> operand-format rows [..., W * parts]: split bf16 is [W hi | W lo]."""
    x = x.float()
    if precision == "tf32":
        return x.contiguous()
    hi = x.to(torch.bfloat16)
    if precision == "bf16":
        return hi.contiguous()
    lo = (x - hi.float()).to(torch.bfloat16)
    return torch.cat([hi, lo], dim=-1).contiguous()


def unpack_rows(y, precision, W):
    """Operand-format rows [..., W * parts] -> fp64 [..., W]."""
    if precision == "bf16x3":
        return y[..., :W].double() + y[..., W:2 * W].double()
    return y[..., :W].double()


def guarded(n, dtype, device="cuda"):
    """(buffer, view of its n middle elements): the view sits between two sentinel-filled guard regions."""
    buf = torch.full((GUARD + n + GUARD,), SENTINEL, dtype=dtype, device=device)
    return buf, buf[GUARD:GUARD + n]


def guards_intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())


def _p(t):
    if t is None:
        return None
    return t.data_ptr() if isinstance(t, torch.Tensor) else t


def src(t, C, X, Y=1, Z=1, ld=0):
    from meshdiffusion_b200 import _native
    return _native.GemmSrcC(_p(t), C, X, Y, Z, ld)


def desc(precision, kind, srcs, n, grid, batch_plan, batch=0, **kw):
    """mdb_gemm_probe_desc: `srcs` are GemmSrcC (or (tensor, C, X, Y, Z[, ld]) tuples); tensors in `kw` become pointers.
    The output defaults to dense NDHWC rows of n channels."""
    from meshdiffusion_b200 import _native
    d = _native.GemmProbeDescC()
    d.precision, d.kind, d.n, d.batch_plan, d.batch = PREC_ID[precision], kind, n, batch_plan, batch
    d.x, d.y, d.z = grid
    d.n_src = len(srcs)
    for i, s in enumerate(srcs):
        d.src[i] = s if isinstance(s, _native.GemmSrcC) else src(*s)
    V = grid[0] * grid[1] * grid[2]
    d.osx, d.osy, d.osz, d.osb, d.lo_off = n, n * grid[0], n * grid[0] * grid[1], n * V, -1
    d.ksize, d.stride = 3, 1
    extra = kw.pop("extra", [])
    d.n_extra = len(extra)
    for i, s in enumerate(extra):
        d.extra[i] = s if isinstance(s, _native.GemmSrcC) else src(*s)
    for k, v in kw.items():
        setattr(d, k, _p(v) if isinstance(v, torch.Tensor) else v)
    return d


def probe(d, stream=None):
    """Runs (or with d.dry describes) one probe; returns its report as a tuple (work items, splits, k-steps, most k-steps
    per entry, BLOCK_N, FLOPs, fill bytes)."""
    from meshdiffusion_b200 import _native
    L = _native.lib()
    r = _native.GemmProbeReportC()
    _native.check(L.mdb_gemm_probe(ctypes.byref(d), ctypes.byref(r), stream))
    return report_tuple(r)


def report_tuple(r):
    return (r.work_items, r.splits, r.ksteps, r.entry_ksteps, r.block_n, r.flops, r.fill_bytes)


def engine_tiles(cfg, batch, precision):
    """{forward GEMM launch name: report tuple} of a GPU-less inference plan (mdb_unet_gemm_tiles + mdb_unet_gemm_ops)."""
    from meshdiffusion_b200 import _native
    from meshdiffusion_b200.diffusion.models import ddpm
    L = _native.lib()
    c = ddpm._config_c(ddpm.arch_from_config(cfg), batch, precision, training=False)
    h = ctypes.c_void_p()
    _native.check(L.mdb_unet_create_dry(ctypes.byref(c), ctypes.byref(h)))
    try:
        ng = ctypes.c_int()
        _native.check(L.mdb_unet_info(h, None, None, ctypes.byref(ng), None))
        rows = {}
        for i in range(ng.value):
            nm, fl, fb = ctypes.c_char_p(), ctypes.c_double(), ctypes.c_double()
            v = [ctypes.c_int() for _ in range(5)]
            _native.check(L.mdb_unet_gemm_ops(h, i, ctypes.byref(nm), ctypes.byref(fl), ctypes.byref(fb)))
            _native.check(L.mdb_unet_gemm_tiles(h, i, *[ctypes.byref(x) for x in v]))
            rows[nm.value.decode()] = tuple(x.value for x in v) + (fl.value, fb.value)
        return rows
    finally:
        L.mdb_unet_destroy(h)


# ---------------------------------------------------------------------------------------------------- the cases
# Each case can name the engine launch it mirrors: (config "full" | "tiny", launch name); test_gemm_probe_cpu.py checks
# that the dry probe of the case reports that launch's tiles, FLOPs and fill bytes at the case's batch and precision.

# split-K convolutions: B (planned), Cin, N, R (input grid), stride; terms = bias, per-sample bias, residual, statistics
SPLIT_CASES = [
    dict(id="conv0_c256_r8", B=1, Cin=256, N=256, R=8, stride=1, terms=False),
    dict(id="conv0_c256_r8_terms", B=1, Cin=256, N=256, R=8, stride=1, terms=True),
    dict(id="tile4442_b3", B=3, Cin=256, N=256, R=4, stride=1, terms=True, launch=(2, 3)),
    dict(id="n96", B=1, Cin=256, N=96, R=8, stride=1, terms=True),
    dict(id="stride2", B=1, Cin=256, N=256, R=8, stride=2, terms=True),
    dict(id="dgrad_addend", B=1, Cin=256, N=256, R=8, stride=1, dgrad=True),
    dict(id="k5", B=1, Cin=64, N=64, R=8, stride=1, k=5, terms=True),
    dict(id="res22_conv0", B=1, Cin=512, N=512, R=4, stride=1, terms="conv0", mirror=("full", "res22.conv0")),
    dict(id="res22_conv1", B=1, Cin=512, N=512, R=4, stride=1, terms="conv1", mirror=("full", "res22.conv1")),
    dict(id="down21", B=1, Cin=512, N=512, R=8, stride=2, terms="down", mirror=("full", "down21")),
    dict(id="tiny_res3_conv0", B=2, Cin=32, N=32, R=16, stride=1, terms="conv0", mirror=("tiny", "res3.conv0")),
    dict(id="tiny_down4", B=2, Cin=32, N=32, R=16, stride=2, terms="down", mirror=("tiny", "down4")),
]

# sub-pixel upsample: low resolution r, channels C, planned batch B (launched at B and, for B > 1, at B - 1)
UP_CASES = [dict(id=f"r{r}_c{C}_b{B}", r=r, C=C, B=B) for r in (4, 8, 16) for C in (128, 256) for B in (1, 3)]
UP_MIRRORS = [dict(r=4, C=512, B=1, mirror=("full", "up32")), dict(r=8, C=512, B=1, mirror=("full", "up37")),
              dict(r=8, C=64, B=2, mirror=("tiny", "up13"))]

# attention core: (V, C, B planned)
ATTN_CASES = [dict(id="v64_c512_b1", V=64, C=512, B=1, mirror=("full", "attn26")),
              dict(id="v64_c512_b3", V=64, C=512, B=3, mirror=("full", "attn26")),
              dict(id="v512_c64_b2", V=512, C=64, B=2, mirror=("tiny", "attn6")),
              dict(id="v512_c256_b2", V=512, C=256, B=2),
              dict(id="v4096_c256_b1", V=4096, C=256, B=1, mirror=("full", "attn12"))]

# fused NIN shortcut of Conv_1: (C0, C1 -> N) at R, batch 2
NIN_CASES = [dict(id="c512_256_to_256_r8", C0=512, C1=256, N=256, R=8, B=2),
             dict(id="c128_128_to_128_r16", C0=128, C1=128, N=128, R=16, B=2),
             dict(id="c64_32_to_32_r16", C0=64, C1=32, N=32, R=16, B=2, mirror=("tiny", "res14.conv1")),
             dict(id="c512_512_to_512_r4", C0=512, C1=512, N=512, R=4, B=1, mirror=("full", "res28.conv1"))]


def split_desc(case, precision, splits, tensors=None, batch=0):
    """Probe description of a SPLIT_CASES entry (tensors: the dict test_gpu_gemm_variants.py allocates, None = dry)."""
    from meshdiffusion_b200 import _native
    t = tensors or {}
    B, Cin, N, R, stride = case["B"], case["Cin"], case["N"], case["R"], case["stride"]
    Ro = R // stride
    kind = _native.PROBE_CONV_DGRAD if case.get("dgrad") else _native.PROBE_CONV
    terms = case.get("terms")
    kw = dict(ksize=case.get("k", 3), stride=stride, splits=splits, out=t.get("out"), w=t.get("w"))
    if terms is True or terms in ("conv0", "conv1", "down"):
        kw.update(bias=t.get("bias"), stats=t.get("stats"))
    if terms is True or terms == "conv0":
        kw.update(rowbias=t.get("rowbias"), rowbias_ld=N)
    if terms is True or terms == "conv1" or case.get("dgrad"):
        kw.update(residual=t.get("res"), res_ld=N, res_batch_stride=Ro ** 3 * N)
    if tensors is None:
        kw["dry"] = 1
    return desc(precision, kind, [(t.get("x"), Cin, R, R, R)], N, (Ro, Ro, Ro), B, batch, **kw)


def nin_desc(case, precision, tensors=None, batch=0, splits=-1):
    from meshdiffusion_b200 import _native
    t = tensors or {}
    B, C0, C1, N, R = case["B"], case["C0"], case["C1"], case["N"], case["R"]
    kw = dict(out=t.get("out"), w=t.get("w1"), w_extra=t.get("wn"), bias=t.get("bias"), stats=t.get("stats"),
              extra=[(t.get("h"), C0, R, R, R), (t.get("skip"), C1, R, R, R)], splits=splits)
    if tensors is None:
        kw["dry"] = 1
    return desc(precision, _native.PROBE_CONV, [(t.get("a2"), N, R, R, R)], N, (R, R, R), B, batch, **kw)


def nin_slot_desc(V_grid, C, B, i, precision, tensors=None, batch=0):
    """attn*.nin<i>: hn [B][R^3][C] @ W_i [C][C] + b_i written to slot i of the qkv rows (pitch 3C)."""
    from meshdiffusion_b200 import _native
    t = tensors or {}
    R = V_grid
    V = R ** 3
    es = 4 if precision == "tf32" else 2
    out = t["qkv"].data_ptr() + i * C * es if tensors else None
    kw = dict(out=out, w=t.get("w"), w_in_out=1, bias=t.get("b"), osx=3 * C, osy=3 * C * R, osz=3 * C * R * R,
              osb=3 * C * V, lo_off=-1)
    if tensors is None:
        kw["dry"] = 1
    return desc(precision, _native.PROBE_POINTWISE, [(t.get("hn"), C, R, R, R)], C, (R, R, R), B, batch, **kw)


def upsample_reports(r, C, B, precision):
    """Dry mdb_upsample_conv: the 8 parity ops' report tuples."""
    from meshdiffusion_b200 import _native
    L = _native.lib()
    reps = (_native.GemmProbeReportC * 8)()
    _native.check(L.mdb_upsample_conv(None, None, None, None, None, None, r, C, B, B, 0xFF, PREC_ID[precision], 1, reps,
                                      None))
    return [report_tuple(x) for x in reps]


def attention_reports(V, C, B, precision):
    """Dry mdb_attention_core: the (qk, pv) report tuples."""
    from meshdiffusion_b200 import _native
    L = _native.lib()
    reps = (_native.GemmProbeReportC * 2)()
    _native.check(L.mdb_attention_core(None, None, None, None, V, C, B, B, 15, PREC_ID[precision], 1, reps, None))
    return [report_tuple(x) for x in reps]


def upsample_probe_desc(r, C, B, par, precision):
    """The probe's own sub-pixel operand (add_conv_up2 at parity par), dry, with the engine's output strides."""
    from meshdiffusion_b200 import _native
    R = 2 * r
    return desc(precision, _native.PROBE_CONV_UP2, [(None, C, r, r, r)], C, (r, r, r), B, parity=par,
                osx=2 * C, osy=2 * R * C, osz=2 * R * R * C, osb=R ** 3 * C, lo_off=C, dry=1)


def fold_upconv(w):
    """fp64 fold of a 3^3 OIDHW weight into the 8 sub-pixel 2^3 kernels [8 (pz, py, px)][Cout][Cin][2][2][2]."""
    M = torch.tensor([[[1., 0., 0.], [0., 1., 1.]], [[1., 1., 0.], [0., 0., 1.]]], dtype=torch.float64, device=w.device)
    w = w.double()
    out = []
    for par in range(8):
        px, py, pz = par & 1, (par >> 1) & 1, par >> 2
        out.append(torch.einsum("ad,be,cf,oidef->oiabc", M[pz], M[py], M[px], w))
    return torch.stack(out)


def logits_desc(V, C, B, precision, tensors=None, batch=0):
    """attn*.qk through the probe: q (pitch 3C) times an activation B operand (k, the next C channels of the same rows),
    scaled by alpha = 1/sqrt(C), into fp32 logits [B][V][V] (an output grid of extent 1 in y and z)."""
    from meshdiffusion_b200 import _native
    t = tensors or {}
    es = 4 if precision == "tf32" else 2
    b_ptr = t["qkv"].data_ptr() + C * es if tensors else None
    kw = dict(b_ptr=b_ptr, b_k=C, b_n=V, b_row_stride=3 * C, b_batch_stride=V * 3 * C, out=t.get("S"), osx=V, osy=0,
              osz=0, osb=V * V, out_fp32=1, alpha=1.0 / C ** 0.5)
    if tensors is None:
        kw["dry"] = 1
    return desc(precision, _native.PROBE_ACT_B, [(t.get("qkv"), C, V, 1, 1, 3 * C)], V, (V, 1, 1), B, batch, **kw)


# GroupNorm-backward epilogue: a 3^3 data gradient (dy of Cout channels -> C0 + C1) whose result is dL/da of
# GroupNorm(+SiLU)(+dropout) over the concatenation of x0 (C0) and x1 (C1). 64 + 32 channels: 3 per group, and group 21
# holds channels 63-65, across the boundary.
GNB_CASES = [dict(id="one_src_c64", C0=64, C1=0, Cout=64, R=8),
             dict(id="two_src_64_32", C0=64, C1=32, Cout=64, R=8)]


def gnb_desc(case, precision, gnb, B_plan, tensors=None, batch=0, silu=1, dropout=0.0, seed=0):
    from meshdiffusion_b200 import _native
    t = tensors or {}
    C0, C1, Cout, R = case["C0"], case["C1"], case["Cout"], case["R"]
    N = C0 + C1
    kw = dict(ksize=3, splits=0, out=t.get("out"), w=t.get("w"), gnb=gnb, gn_x0=t.get("x0"), gn_c0=C0,
              gn_x1=t.get("x1") if C1 else None, gn_c1=C1, gn_stats0=t.get("stats0"),
              gn_stats1=t.get("stats1") if C1 else None, gn_gamma=t.get("gamma"), gn_beta=t.get("beta"),
              gn_silu=silu, gn_dropout=dropout, gn_seed=seed, gn_dx=t.get("dx"), gn_dgamma=t.get("dgamma"),
              gn_dbeta=t.get("dbeta"))
    if tensors is None:
        kw["dry"] = 1
    return desc(precision, _native.PROBE_CONV_DGRAD, [(t.get("dy"), Cout, R, R, R)], N, (R, R, R), B_plan, batch, **kw)
