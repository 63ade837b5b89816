"""The implicit-GEMM variants of the score network, one launch (or one engine composite) at a time, against fp64.

mdb_gemm_probe builds one GemmOp with the engine's builder calls; mdb_upsample_conv and mdb_attention_core run the engine's
own sub-pixel upsample and attention-core construction (unet.h). Families: split-K with its separate reduction kernel,
the 8-parity sub-pixel upsample, the attention core (q.k^T with an activation B operand and alpha, softmax rows, P.v
reading the probabilities inside the fp32 logits), the qkv projections at channel offsets, and Conv_1 with the fused NIN
shortcut. Every output sits between sentinel guard regions; what an op must not touch (other qkv slots, samples at or
past the launch batch, sites of parity classes not launched yet) is sentinel-filled and checked afterwards. An op
planned for more samples than it is launched at must equal, bit for bit, the op planned at the launch batch.

The references are fp64 (on the GPU, for speed) from the operands as the kernel reads them; the gates live in
gemm_variants.GATES, and test_gemm_probe_cpu.py checks that a plausible wrong answer misses each by 5x or more.
"""
import pytest
import torch
import torch.nn.functional as F

import gemm_variants as gv

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rows(x_ncdhw):
    """[B, C, Z, Y, X] -> [B, Z, Y, X, C] rows."""
    return x_ncdhw.permute(0, 2, 3, 4, 1).contiguous()


def _ncdhw(rows):
    return rows.permute(0, 4, 1, 2, 3).contiguous()


def _stats_err(words, ref, B):
    """Statistics [B][N][4] words vs (sum, sum of squares) over the voxels of the fp64 reference [B, N, ...]."""
    from meshdiffusion_b200 import ops
    got = ops.words_to_stats(words[:B].cpu())
    r = ref[:B].flatten(2)
    want = torch.stack([r.sum(-1), (r * r).sum(-1)], -1).cpu()
    return max(gv.rel_err(got[..., 0], want[..., 0]), gv.rel_err(got[..., 1], want[..., 1]))


# ------------------------------------------------------------------------------------------------ split-K
def _split_tensors(case, precision, seed=11):
    g = _gen(seed)
    B, Cin, N, R, stride = case["B"], case["Cin"], case["N"], case["R"], case["stride"]
    Ro = R // stride
    t = {}
    x = torch.randn(B, Cin, R, R, R, device=DEV, generator=g)
    t["x_ref"] = gv.as_operand(x, precision)
    t["x"] = gv.pack_rows(_rows(x), precision)
    k = case.get("k", 3)
    if case.get("dgrad"):  # forward weight [Cin (= dy channels)][N][3^3]
        w = torch.randn(Cin, N, k, k, k, device=DEV, generator=g) / (Cin * k ** 3) ** 0.5
    else:
        w = torch.randn(N, Cin, k, k, k, device=DEV, generator=g) / (Cin * k ** 3) ** 0.5
    t["w"] = w.contiguous()
    t["w_ref"] = gv.as_operand(w, precision)
    t["bias"] = torch.randn(N, device=DEV, generator=g)
    t["rowbias"] = torch.randn(B, N, device=DEV, generator=g)
    res = torch.randn(B, N, Ro, Ro, Ro, device=DEV, generator=g)
    t["res_ref"] = gv.as_operand(res, precision)
    t["res"] = gv.pack_rows(_rows(res), precision)
    return t


def _split_ref(case, t, B):
    stride, terms = case["stride"], case.get("terms")
    x, w = t["x_ref"][:B], t["w_ref"]
    if case.get("dgrad"):
        y = F.conv3d(x, w.transpose(0, 1).flip(2, 3, 4), padding=1)
    elif stride == 2:
        y = F.conv3d(F.pad(x, (0, 1, 0, 1, 0, 1)), w, stride=2)
    else:
        y = F.conv3d(x, w, padding=w.shape[-1] // 2)
    if terms is True or terms in ("conv0", "conv1", "down"):
        y = y + t["bias"].double().view(1, -1, 1, 1, 1)
    if terms is True or terms == "conv0":
        y = y + t["rowbias"][:B].double().view(B, -1, 1, 1, 1)
    if terms is True or terms == "conv1" or case.get("dgrad"):
        y = y + t["res_ref"][:B]
    return y


def _split_run(case, precision, t, splits, batch=0, batch_plan=None):
    """(output fp64 NCDHW over the planned batch, raw output rows, stats words, guards intact, splits used)."""
    c = dict(case, B=batch_plan or case["B"])
    B, N, Ro = c["B"], c["N"], c["R"] // c["stride"]
    n = B * Ro ** 3 * N * gv.parts(precision)
    buf, out = gv.guarded(n, gv.act_dtype(precision))
    stats = torch.zeros(B, N, 4, dtype=torch.int64, device=DEV)
    tt = dict(t, out=out, stats=stats)
    if B < case["B"]:  # a smaller plan over the first samples of the same tensors
        tt.update(x=t["x"][:B].contiguous(), rowbias=t["rowbias"][:B].contiguous(), res=t["res"][:B].contiguous())
    rep = gv.probe(gv.split_desc(c, precision, splits, tt, batch))
    torch.cuda.synchronize()
    rows = out.view(B, Ro, Ro, Ro, N * gv.parts(precision))
    return _ncdhw(gv.unpack_rows(rows, precision, N)), rows.clone(), stats, gv.guards_intact(buf), rep[1]


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.SPLIT_CASES, ids=lambda c: c["id"])
def test_split_k(case, precision):
    gate = gv.GATES["split"][precision]
    t = _split_tensors(case, precision)
    B = case["B"]
    ref = _split_ref(case, t, B)
    with_stats = case.get("terms") not in (False, None) and not case.get("dgrad")
    base, base_rows, _, ok, s1 = _split_run(case, precision, t, 0)
    assert ok and s1 == 1
    for S in (-1, 2, 3, 7, 10 ** 6):
        out, rows, stats, ok, used = _split_run(case, precision, t, S)
        err = gv.rel_err(out, ref)
        serr = _stats_err(stats, ref, B) if with_stats else 0.0
        agree = gv.rel_err(out, base)
        print(f"split {case['id']} {precision} S={S}->{used}: err {err:.3e} stats {serr:.3e} vs S=1 {agree:.3e}")
        assert ok, "the split-K reduction wrote outside the output"
        assert err < gate and serr < gate and agree < gate
        if S == 10 ** 6:
            assert 1 < used < S  # clamped to the op's k-groups
        _, rows2, stats2, _, _ = _split_run(case, precision, t, S)
        assert torch.equal(rows, rows2) and torch.equal(stats, stats2), "two launches at the same split factor differ"
    for b in case.get("launch", ()):
        # planned at B, launched at b: bitwise the op planned at b, and nothing written for samples >= b
        S = _split_run(case, precision, t, -1)[4]
        _, rows, stats, ok, _ = _split_run(case, precision, t, S, batch=b)
        _, rows_b, stats_b, _, _ = _split_run(case, precision, t, S, batch_plan=b)
        assert ok and torch.equal(rows[:b], rows_b) and torch.equal(stats[:b], stats_b), b
        assert bool((rows[b:] == gv.SENTINEL).all()) and not bool(stats[b:].any()), b


# ------------------------------------------------------------------------------------------------ sub-pixel upsample
def _upsample(x_rows, w, b, r, C, B_plan, batch, mask, precision):
    from meshdiffusion_b200 import _native
    L = _native.lib()
    R = 2 * r
    n = B_plan * R ** 3 * C * gv.parts(precision)
    buf, out = gv.guarded(n, gv.act_dtype(precision))
    stats = torch.zeros(B_plan, C, 4, dtype=torch.int64, device=DEV)
    w8 = torch.full((64 * C * C,), gv.SENTINEL, device=DEV)
    _native.check(L.mdb_upsample_conv(_native.ptr(x_rows), _native.ptr(w), _native.ptr(b), _native.ptr(w8),
                                      _native.ptr(out), _native.ptr(stats), r, C, B_plan, batch, mask,
                                      gv.PREC_ID[precision], 0, None, _native.current_stream()))
    torch.cuda.synchronize()
    return out.view(B_plan, R, R, R, C * gv.parts(precision)), stats, w8, gv.guards_intact(buf)


def _parity_sites(R, par):
    m = torch.zeros(R, R, R, dtype=torch.bool, device=DEV)
    px, py, pz = par & 1, (par >> 1) & 1, par >> 2
    m[pz::2, py::2, px::2] = True
    return m


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.UP_CASES, ids=lambda c: c["id"])
def test_subpixel_upsample(case, precision):
    gate = gv.GATES["upsample"][precision]
    r, C, B = case["r"], case["C"], case["B"]
    R = 2 * r
    g = _gen(21)
    x = torch.randn(B, C, r, r, r, device=DEV, generator=g)
    w = (torch.randn(C, C, 3, 3, 3, device=DEV, generator=g) / (C * 27) ** 0.5).contiguous()
    b = torch.randn(C, device=DEV, generator=g)
    xr = gv.pack_rows(_rows(x), precision)
    ref = F.conv3d(F.interpolate(gv.as_operand(x, precision), scale_factor=2, mode="nearest"), w.double(), b.double(),
                   padding=1)
    out, stats, w8, ok = _upsample(xr, w, b, r, C, B, 0, 0xFF, precision)
    got = _ncdhw(gv.unpack_rows(out, precision, C))
    err, serr = gv.rel_err(got, ref), _stats_err(stats, ref, B)
    ferr = gv.rel_err(w8.view(8, C, C, 2, 2, 2), gv.fold_upconv(w))
    print(f"upsample {case['id']} {precision}: err {err:.3e} stats {serr:.3e} fold {ferr:.3e}")
    assert ok and err < gate and serr < gate and ferr < 1e-6
    assert not bool((out == gv.SENTINEL).all(-1).any()), "a site of the output was not written"
    # each parity class writes its own sites and no other: launched one class at a time, in order
    if r == 4 or (C == 128 and B == 1):
        done = torch.zeros(R, R, R, dtype=torch.bool, device=DEV)
        for par in range(8):
            o, _, _, ok = _upsample(xr, w, b, r, C, B, 0, 1 << par, precision)
            sites = _parity_sites(R, par)
            written = ~(o == gv.SENTINEL).all(-1)
            assert ok and torch.equal(written, sites.expand_as(written)), par
            assert torch.equal(o[:, sites], out[:, sites]), par
            done |= sites
        assert bool(done.all())
    if B > 1:
        b_launch = B - 1
        o, st, _, ok = _upsample(xr, w, b, r, C, B, b_launch, 0xFF, precision)
        o_b, st_b, _, _ = _upsample(xr[:b_launch].contiguous(), w, b, r, C, b_launch, 0, 0xFF, precision)
        assert ok and torch.equal(o[:b_launch], o_b) and torch.equal(st[:b_launch], st_b)
        assert bool((o[b_launch:] == gv.SENTINEL).all()) and not bool(st[b_launch:].any())


# ------------------------------------------------------------------------------------------------ attention
def _attn_buffers(V, C, B, precision, qkv):
    p = gv.parts(precision)
    bufS, S = gv.guarded(B * V * V, torch.float32)
    bufO, O = gv.guarded(B * V * C * p, gv.act_dtype(precision))
    vT = torch.full((B * C * V * p,), gv.SENTINEL, dtype=gv.act_dtype(precision), device=DEV)
    return dict(qkv=qkv, S=S, O=O, vT=vT, bufS=bufS, bufO=bufO)


def _attn_run(bufs, V, C, B_plan, batch, stages, precision):
    from meshdiffusion_b200 import _native
    L = _native.lib()
    _native.check(L.mdb_attention_core(_native.ptr(bufs["qkv"]), _native.ptr(bufs["vT"]), _native.ptr(bufs["S"]),
                                       _native.ptr(bufs["O"]), V, C, B_plan, batch, stages, gv.PREC_ID[precision], 0,
                                       None, _native.current_stream()))
    torch.cuda.synchronize()


def _probabilities(S, V, B, precision):
    """The softmax's rows as P.v reads them: operand-format rows at the start of each fp32 row of S."""
    rows = S.view(B, V, V)
    if precision == "tf32":
        return rows.double()
    bf = rows.view(torch.bfloat16)  # [B][V][2V]
    return gv.unpack_rows(bf, precision, V)


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.ATTN_CASES, ids=lambda c: c["id"])
def test_attention_core(case, precision):
    gate = gv.GATES["attn"][precision]
    V, C, B = case["V"], case["C"], case["B"]
    g = _gen(31)
    qkv_f = torch.randn(B, V, 3 * C, device=DEV, generator=g)
    qkv = gv.pack_rows(qkv_f, precision)
    q, k, v = (gv.as_operand(qkv_f[..., i * C:(i + 1) * C], precision) for i in range(3))
    bufs = _attn_buffers(V, C, B, precision, qkv)
    _attn_run(bufs, V, C, B, 0, 1 | 2, precision)
    logits = bufs["S"].view(B, V, V).clone()
    ref_logits = q @ k.transpose(1, 2) / C ** 0.5
    e_l = gv.rel_err(logits, ref_logits)
    _attn_run(bufs, V, C, B, 0, 4, precision)
    P = _probabilities(bufs["S"], V, B, precision)
    e_p = gv.rel_err(P, torch.softmax(logits.double(), -1))
    _attn_run(bufs, V, C, B, 0, 8, precision)
    O = gv.unpack_rows(bufs["O"].view(B, V, C * gv.parts(precision)), precision, C)
    e_pv = gv.rel_err(O, P @ v)
    e_o = gv.rel_err(O, torch.softmax(ref_logits, -1) @ v)
    print(f"attention {case['id']} {precision}: logits {e_l:.3e} softmax {e_p:.3e} pv {e_pv:.3e} O {e_o:.3e}")
    assert gv.guards_intact(bufs["bufS"]) and gv.guards_intact(bufs["bufO"])
    # end to end, O carries the rounding of the logits through the softmax and that of the probabilities: two stages' gates
    assert e_l < gate and e_p < gate and e_pv < gate and e_o < 2 * gate
    if B > 1:
        b = B - 1
        big = _attn_buffers(V, C, B, precision, qkv)
        _attn_run(big, V, C, B, b, 15, precision)
        small = _attn_buffers(V, C, b, precision, qkv[:b].contiguous())
        _attn_run(small, V, C, b, 0, 15, precision)
        p = gv.parts(precision)
        assert torch.equal(big["O"][:b * V * C * p], small["O"]) and torch.equal(big["S"][:b * V * V], small["S"])
        assert bool((big["O"][b * V * C * p:] == gv.SENTINEL).all()) and bool((big["S"][b * V * V:] == gv.SENTINEL).all())


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.ATTN_CASES, ids=lambda c: c["id"])
def test_qkv_projections_at_channel_offsets(case, precision):
    """attn*.nin0-2: three launches write q, k and v into one qkv row of pitch 3C (split bf16: lo parts 3C further on);
    after each launch the slots not written yet are still sentinel."""
    gate = gv.GATES["attn"][precision]
    V, C, B = case["V"], case["C"], case["B"]
    R = round(V ** (1 / 3))
    g = _gen(41)
    hn = torch.randn(B, V, C, device=DEV, generator=g)
    hn_rows = gv.pack_rows(hn, precision)
    W = [(torch.randn(C, C, device=DEV, generator=g) / C ** 0.5).contiguous() for _ in range(3)]
    bias = [torch.randn(C, device=DEV, generator=g) for _ in range(3)]
    p = gv.parts(precision)
    buf, qkv = gv.guarded(B * V * 3 * C * p, gv.act_dtype(precision))
    rows = qkv.view(B, V, 3 * C * p)
    for i in range(3):
        gv.probe(gv.nin_slot_desc(R, C, B, i, precision, dict(qkv=qkv, hn=hn_rows, w=W[i], b=bias[i])))
        torch.cuda.synchronize()
        got = gv.unpack_rows(rows, precision, 3 * C)
        ref = gv.as_operand(hn, precision) @ gv.as_operand(W[i], precision) + bias[i].double()
        err = gv.rel_err(got[..., i * C:(i + 1) * C], ref)
        print(f"qkv {case['id']} {precision} slot {i}: err {err:.3e}")
        assert err < gate and gv.guards_intact(buf)
        for j in range(i + 1, 3):
            for part in range(p):
                sl = rows[..., part * 3 * C + j * C:part * 3 * C + (j + 1) * C]
                assert bool((sl == gv.SENTINEL).all()), (i, j, part)
    # once all three have run, every slot still holds its own projection (a later launch wrote no earlier slot)
    got = gv.unpack_rows(rows, precision, 3 * C)
    for i in range(3):
        ref = gv.as_operand(hn, precision) @ gv.as_operand(W[i], precision) + bias[i].double()
        assert gv.rel_err(got[..., i * C:(i + 1) * C], ref) < gate, i


# ------------------------------------------------------------------------------------------------ fused NIN shortcut
def _nin_run(case, precision, t, batch=0, batch_plan=None, splits=-1):
    c = dict(case, B=batch_plan or case["B"])
    B, N, R = c["B"], c["N"], c["R"]
    buf, out = gv.guarded(B * R ** 3 * N * gv.parts(precision), gv.act_dtype(precision))
    stats = torch.zeros(B, N, 4, dtype=torch.int64, device=DEV)
    tt = dict(t, out=out, stats=stats)
    if B < case["B"]:
        tt.update({k: t[k][:B].contiguous() for k in ("a2", "h", "skip")})
    rep = gv.probe(gv.nin_desc(c, precision, tt, batch, splits))
    torch.cuda.synchronize()
    rows = out.view(B, R, R, R, N * gv.parts(precision))
    return rows, stats, gv.guards_intact(buf), rep


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.NIN_CASES, ids=lambda c: c["id"])
def test_fused_nin_shortcut(case, precision):
    gate = gv.GATES["nin"][precision]
    B, C0, C1, N, R = case["B"], case["C0"], case["C1"], case["N"], case["R"]
    g = _gen(51)
    a2, h, skip = (torch.randn(B, c, R, R, R, device=DEV, generator=g) for c in (N, C0, C1))
    w1 = (torch.randn(N, N, 3, 3, 3, device=DEV, generator=g) / (N * 27) ** 0.5).contiguous()
    wn = (torch.randn(C0 + C1, N, device=DEV, generator=g) / (C0 + C1) ** 0.5).contiguous()
    bias = torch.randn(N, device=DEV, generator=g)  # Conv_1.bias + NIN_0.b, summed as the engine does at commit
    t = dict(a2=gv.pack_rows(_rows(a2), precision), h=gv.pack_rows(_rows(h), precision),
             skip=gv.pack_rows(_rows(skip), precision), w1=w1, wn=wn, bias=bias)
    rows, stats, ok, rep = _nin_run(case, precision, t)
    got = _ncdhw(gv.unpack_rows(rows, precision, N))
    raw = torch.cat([gv.as_operand(h, precision), gv.as_operand(skip, precision)], 1)
    ref = (F.conv3d(gv.as_operand(a2, precision), gv.as_operand(w1, precision), bias.double(), padding=1) +
           torch.einsum("bcxyz,cn->bnxyz", raw, gv.as_operand(wn, precision)))
    err, serr = gv.rel_err(got, ref), _stats_err(stats, ref, B)
    print(f"nin {case['id']} {precision} (splits {rep[1]}): err {err:.3e} stats {serr:.3e}")
    assert ok and err < gate and serr < gate
    if B > 1:
        b = B - 1
        # both at the split factor the engine plans for B (the plan at b may choose another one)
        S = rep[1]
        rows_p, st_p, ok, rep_p = _nin_run(case, precision, t, batch=b, splits=S)
        rows_b, st_b, _, rep_b = _nin_run(case, precision, t, batch_plan=b, splits=S)
        assert rep_p[1] == rep_b[1] == S
        assert torch.equal(rows_p[:b], rows_b) and torch.equal(st_p[:b], st_b)
        assert ok and gv.rel_err(_ncdhw(gv.unpack_rows(rows_p[:b], precision, N)), ref[:b]) < gate
        assert bool((rows_p[b:] == gv.SENTINEL).all()) and not bool(st_p[b:].any())


@pytest.mark.parametrize("precision", gv.PRECISIONS)
@pytest.mark.parametrize("case", gv.ATTN_CASES, ids=lambda c: c["id"])
def test_logits_through_the_probe(case, precision):
    """attn*.qk described to mdb_gemm_probe (activation B operand, alpha, fp32 output with y = z = 1): the same logits,
    bit for bit, as the engine's attention core, and nothing past the launch batch."""
    gate = gv.GATES["attn"][precision]
    V, C, B = case["V"], case["C"], case["B"]
    g = _gen(61)
    qkv_f = torch.randn(B, V, 3 * C, device=DEV, generator=g)
    qkv = gv.pack_rows(qkv_f, precision)
    q, k = (gv.as_operand(qkv_f[..., i * C:(i + 1) * C], precision) for i in range(2))
    b = B - 1 if B > 1 else B
    buf, S = gv.guarded(B * V * V, torch.float32)
    gv.probe(gv.logits_desc(V, C, B, precision, dict(qkv=qkv, S=S), batch=b))
    torch.cuda.synchronize()
    err = gv.rel_err(S[:b * V * V].view(b, V, V), (q @ k.transpose(1, 2) / C ** 0.5)[:b])
    print(f"logits probe {case['id']} {precision}: err {err:.3e}")
    assert err < gate and gv.guards_intact(buf) and bool((S[b * V * V:] == gv.SENTINEL).all())
    eng = _attn_buffers(V, C, B, precision, qkv)
    _attn_run(eng, V, C, B, b, 1 | 2, precision)
    assert torch.equal(S[:b * V * V], eng["S"][:b * V * V])


# ------------------------------------------------------------------------------------------------ GroupNorm backward
def _gnb_tensors(case, precision, B, seed=71):
    """Operands for B samples (the fused runs take the first samples): dy of the data gradient, the forward weight, the
    GroupNorm's raw inputs x0 / x1 with their statistics (from the operand values, as the forward GEMM leaves them),
    gamma and beta."""
    from meshdiffusion_b200 import ops
    g = _gen(seed)
    C0, C1, Cout, R = case["C0"], case["C1"], case["Cout"], case["R"]
    N = C0 + C1
    dy = torch.randn(B, Cout, R, R, R, device=DEV, generator=g)
    w = (torch.randn(Cout, N, 3, 3, 3, device=DEV, generator=g) / (Cout * 27) ** 0.5).contiguous()
    x = torch.randn(B, N, R, R, R, device=DEV, generator=g) * 1.5 + 0.3
    t = dict(dy_ref=gv.as_operand(dy, precision), dy=gv.pack_rows(_rows(dy), precision), w=w,
             w_ref=gv.as_operand(w, precision), x_ref=gv.as_operand(x, precision),
             gamma=torch.randn(N, device=DEV, generator=g) * 0.5 + 1.0, beta=torch.randn(N, device=DEV, generator=g) * 0.5)
    for name, lo, hi in (("0", 0, C0), ("1", C0, N)):
        if hi > lo:
            xs = x[:, lo:hi]
            t["x" + name] = gv.pack_rows(_rows(xs), precision)
            xr = gv.as_operand(xs, precision).flatten(2)
            t["stats" + name] = ops.stats_to_words(torch.stack([xr.sum(-1), (xr * xr).sum(-1)], -1)).to(DEV)
    return t


def _gnb_run(case, precision, t, gnb, B_plan, batch=0, silu=1, dropout=0.0, seed=5):
    """(dx fp64 NCDHW over the planned batch, raw dx rows, dgamma, dbeta, dx guards intact)."""
    C0, C1, R = case["C0"], case["C1"], case["R"]
    N = C0 + C1
    p = gv.parts(precision)
    tt = {k: (v[:B_plan].contiguous() if k in ("dy", "x0", "x1", "stats0", "stats1") else v) for k, v in t.items()}
    tt["out"] = torch.full((B_plan * R ** 3 * N * p,), gv.SENTINEL, dtype=gv.act_dtype(precision), device=DEV)
    buf, dx = gv.guarded(B_plan * R ** 3 * N * p, gv.act_dtype(precision))
    tt.update(dx=dx, dgamma=torch.full((N,), gv.SENTINEL, device=DEV), dbeta=torch.full((N,), gv.SENTINEL, device=DEV))
    gv.probe(gv.gnb_desc(case, precision, gnb, B_plan, tt, batch, silu, dropout, seed))
    torch.cuda.synchronize()
    rows = dx.view(B_plan, R, R, R, N * p)
    return _ncdhw(gv.unpack_rows(rows, precision, N)), rows.clone(), tt["dgamma"], tt["dbeta"], gv.guards_intact(buf)


def _gnb_ref(t, B, silu):
    """fp64 autograd of GroupNorm(32, eps 1e-6)(+SiLU) over the concatenation, driven by the transposed conv of dy."""
    x = t["x_ref"][:B].clone().requires_grad_(True)
    gamma = t["gamma"].double().clone().requires_grad_(True)
    beta = t["beta"].double().clone().requires_grad_(True)
    a = F.group_norm(x, 32, gamma, beta, eps=1e-6)
    if silu:
        a = F.silu(a)
    da = F.conv3d(t["dy_ref"][:B], t["w_ref"].transpose(0, 1).flip(2, 3, 4), padding=1)
    a.backward(da)
    return x.grad, gamma.grad, beta.grad


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("silu", [1, 0])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("case", gv.GNB_CASES, ids=lambda c: c["id"])
def test_groupnorm_backward_epilogue(case, B, silu, precision):
    gate = gv.GATES["gnb"][precision]
    t = _gnb_tensors(case, precision, 4)
    rdx, rdg, rdb = _gnb_ref(t, B, silu)
    for gnb, name in ((1, "fused"), (2, "two-pass")):
        dx, _, dg, db, ok = _gnb_run(case, precision, t, gnb, B, silu=silu)
        e = (gv.rel_err(dx, rdx), gv.rel_err(dg, rdg), gv.rel_err(db, rdb))
        print(f"gnb {case['id']} {precision} B={B} silu={silu} {name}: dx {e[0]:.3e} dgamma {e[1]:.3e} dbeta {e[2]:.3e}")
        assert ok and max(e) < gate, name
    # dropout 0.3: the fused epilogue and the two-pass path draw the same mask
    fused = _gnb_run(case, precision, t, 1, B, silu=silu, dropout=0.3, seed=99)
    two = _gnb_run(case, precision, t, 2, B, silu=silu, dropout=0.3, seed=99)
    e = (gv.rel_err(fused[0], two[0]), gv.rel_err(fused[2], two[2]), gv.rel_err(fused[3], two[3]))
    print(f"gnb {case['id']} {precision} B={B} silu={silu} dropout fused vs two-pass: dx {e[0]:.3e} dgamma {e[1]:.3e} "
          f"dbeta {e[2]:.3e}")
    assert fused[4] and max(e) < gate
    assert gv.rel_err(fused[0], rdx) > 5 * gate, "dropout 0.3 left the data gradient unchanged"
    if B == 3:
        # planned for 4, launched at 3: bitwise the op planned at 3, and no dx for sample 3
        for gnb in (1, 2):
            big = _gnb_run(case, precision, t, gnb, 4, batch=3, silu=silu, dropout=0.3, seed=99)
            small = _gnb_run(case, precision, t, gnb, 3, silu=silu, dropout=0.3, seed=99)
            assert big[4] and torch.equal(big[1][:3], small[1]), gnb
            assert torch.equal(big[2], small[2]) and torch.equal(big[3], small[3]), gnb
            assert bool((big[1][3:] == gv.SENTINEL).all()), gnb
