"""Per-kernel GPU parity through the C ABI (painter_b200.ops -> libpainter_b200.so) against plain torch fp32
restatements of the same reference op on the same seeded inputs, plus size-independent properties at the full
BASELINE geometry.  Tolerances: bf16-operand tensor-core kernels 1e-2 of max|ref|; fp32 streaming kernels 1e-5."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


def relmax(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)


# ------------------------------------------------------------------ GEMM ------------------------------------
@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_gemm_operand_majors_and_tiles(ta, tb, bn):
    from painter_b200 import _lib, ops
    M, N, K = 304, 512, 200
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.5).bfloat16()
    bias = torch.randn(N, device=DEV)
    _lib.lib().pk_gemm_force_bn(bn)
    try:
        got = ops.gemm(a.t().contiguous() if ta else a, b.t().contiguous() if tb else b, trans_a=bool(ta),
                       trans_b=bool(tb), kind=ops.EPI_F32, bias=bias)
    finally:
        _lib.lib().pk_gemm_force_bn(0)
    assert relmax(got, a.float() @ b.float().t() + bias) < 2e-5


def test_gemm_split_k_matches_single_pass():
    from painter_b200 import _lib, ops
    a = (torch.randn(3136, 256, device=DEV) * 0.5).bfloat16()   # [K, M] wgrad layout
    b = (torch.randn(3136, 384, device=DEV) * 0.5).bfloat16()   # [K, N]
    ref = a.float().t() @ b.float()
    for s in (1, 3, 7):
        _lib.lib().pk_gemm_force_splits(s)
        try:
            out = torch.zeros(256, 384, device=DEV)
            ops.gemm(a, b, trans_a=True, trans_b=True, kind=ops.EPI_F32, out=out, accumulate=2)
        finally:
            _lib.lib().pk_gemm_force_splits(0)
        assert relmax(out, ref) < 2e-5, s


@pytest.mark.parametrize("M,N,K,ta,tb", [(768, 512, 4096, True, True), (1024, 1024, 1568, True, True),
                                          (3072, 1024, 3136, True, True), (512, 256, 640, False, False),
                                          (4096, 1024, 1000, True, True)])
def test_gemm_stream_k_weight_gradient_tiling(M, N, K, ta, tb):
    """Zero-initialised fp32 outputs (accumulate=2) take the stream-K schedule of the CTA-pair kernel: every cluster
    owns an equal range of (tile, k-block) units, tiles that straddle ranges are completed with atomics."""
    from painter_b200 import ops
    a = (torch.randn((K, M) if ta else (M, K), device=DEV) * 0.5).bfloat16()
    b = (torch.randn((K, N) if tb else (N, K), device=DEV) * 0.5).bfloat16()
    ref = (a.float().t() if ta else a.float()) @ (b.float() if tb else b.float().t())
    out = torch.zeros(M, N, device=DEV)
    ops.gemm(a, b, trans_a=ta, trans_b=tb, kind=ops.EPI_F32, out=out, accumulate=2)
    assert relmax(out, ref) < 2e-5
    ops.gemm(a, b, trans_a=ta, trans_b=tb, kind=ops.EPI_F32, out=out, accumulate=2)   # second pass adds
    assert relmax(out, 2 * ref) < 2e-5


def test_gemm_epilogues():
    from painter_b200 import ops
    M, N, K = 384, 512, 256
    a = (torch.randn(M, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=DEV) * 0.5).bfloat16()
    bias = torch.randn(N, device=DEV)
    ref = a.float() @ b.float().t()
    z, hact = ops.gemm(a, b, kind=ops.EPI_GELU, bias=bias)
    assert relmax(z, ref + bias) < 1e-2 and relmax(hact, F.gelu((ref + bias).bfloat16().float())) < 1e-2
    res = torch.randn(M, N, device=DEV)
    rs = torch.tensor([1.0, 0.0, 1.1, 0.9], device=DEV)
    got = ops.gemm(a, b, kind=ops.EPI_RESID, bias=bias, aux=res, rowscale=rs, rows_per_group=M // 4)
    assert relmax(got, res + rs.repeat_interleave(M // 4)[:, None] * (ref + bias)) < 2e-5
    zz = torch.randn(M, N, device=DEV).bfloat16()
    zf = zz.float().requires_grad_(True)
    F.gelu(zf).sum().backward()
    assert relmax(ops.gemm(a, b, kind=ops.EPI_DGELU, aux=zz), ref * zf.grad) < 1e-2


def test_gemm_pixel_shuffle_epilogue_matches_reference_einsum():
    from painter_b200 import ops
    B, h, w, p, c, K = 2, 8, 4, 16, 64, 128
    a = (torch.randn(B * h * w, K, device=DEV) * 0.5).bfloat16()
    b = (torch.randn(p * p * c, K, device=DEV) * 0.5).bfloat16()
    bias = torch.randn(p * p * c, device=DEV)
    out = torch.zeros(B, h * p, w * p, c, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, b, kind=ops.EPI_PIXSHUF, bias=bias, pixshuf=(h, w, p, c, out))
    d = (a.float() @ b.float().t() + bias).reshape(B, h, w, p, p, c)
    want = torch.einsum("nhwpqc->nchpwq", d).reshape(B, c, h * p, w * p).permute(0, 2, 3, 1)  # models_painter.py:427
    assert relmax(out, want) < 1e-2


def test_gemm_linearity_at_full_size():
    """Size-independent property at the BASELINE geometry (qkv projection, M = 12544): f(a1 + a2) = f(a1) + f(a2).
    Small-integer operands make every product and partial sum exact in fp32, so the identity must hold BIT-EXACTLY
    whatever the accumulation order of the tensor cores."""
    from painter_b200 import ops
    M, N, K = 12544, 3072, 1024
    a1 = torch.randint(-4, 5, (M, K), device=DEV).bfloat16()
    a2 = torch.randint(-4, 5, (M, K), device=DEV).bfloat16()
    b = (torch.randint(-4, 5, (N, K), device=DEV).float() / 8).bfloat16()
    f = lambda x: ops.gemm(x, b, kind=ops.EPI_F32)
    lhs, rhs = f((a1.float() + a2.float()).bfloat16()), f(a1) + f(a2)
    assert torch.equal(lhs, rhs)
    assert torch.equal(f(a1)[:64], a1[:64].float() @ b.float().t())


# ------------------------------------------------------------ streaming kernels --------------------------------
def test_layernorm_fwd_bwd():
    from painter_b200 import ops
    M, C = 777, 1024
    x = torch.randn(M, C, device=DEV) * 2 + 0.5
    g = torch.randn(C, device=DEV)
    b = torch.randn(C, device=DEV)
    xr = x.clone().requires_grad_(True)
    gr, br = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = F.layer_norm(xr, (C,), gr, br, 1e-6)
    y32, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-6, out_dtype=torch.float32)
    assert relmax(y32, yr) < 1e-5
    ybf, _, _ = ops.layernorm_fwd(x, g, b, 1e-6)
    assert relmax(ybf, yr) < 1e-2
    dy = torch.randn(M, C, device=DEV)
    dres = torch.randn(M, C, device=DEV)
    yr.backward(dy)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx = ops.layernorm_bwd(dy, x, mean, rstd, g, dg, db, dres=dres)
    assert relmax(dx, xr.grad + dres) < 2e-5 and relmax(dg, gr.grad) < 1e-4 and relmax(db, br.grad) < 1e-4
    # fused form: also bf16(DropPath scale * dx) and its column sums (pk_layernorm_bwd_cast)
    rs = torch.tensor([1.25, 0.0, 0.8], device=DEV)
    dg2, db2, cs = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx2, dxb = ops.layernorm_bwd(dy, x, mean, rstd, g, dg2, db2, dres=dres, cast=(rs, M // 3, cs))
    want = (xr.grad + dres) * rs.repeat_interleave(M // 3)[:, None]
    assert relmax(dx2, xr.grad + dres) < 2e-5 and relmax(dg2, gr.grad) < 1e-4 and relmax(db2, br.grad) < 1e-4
    assert dxb.dtype == torch.bfloat16 and relmax(dxb, want) < 1e-2 and relmax(cs, want.sum(0)) < 1e-4
    # dy arriving as bf16 (the dgrad GEMM's output dtype), from a column slice of a wider buffer: exact on the
    # bf16-representable values
    wide = torch.randn(M, 2 * C, device=DEV).bfloat16()
    dyb = wide[:, C:]
    xr.grad = None
    gr.grad = None
    br.grad = None
    F.layer_norm(xr, (C,), gr, br, 1e-6).backward(dyb.float())
    dg3, db3 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx3 = ops.layernorm_bwd(dyb, x, mean, rstd, g, dg3, db3, dres=dres)
    assert relmax(dx3, xr.grad + dres) < 2e-5 and relmax(dg3, gr.grad) < 1e-4 and relmax(db3, br.grad) < 1e-4
    dg4, db4, cs4 = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dx4, _ = ops.layernorm_bwd(dyb, x, mean, rstd, g, dg4, db4, dres=dres, cast=(rs, M // 3, cs4))
    assert relmax(dx4, xr.grad + dres) < 2e-5 and relmax(dg4, gr.grad) < 1e-4


def test_patch_embed_lowering_and_token_assembly():
    from painter_b200 import ops
    B, H, W, p, C = 2, 128, 64, 16, 128
    h, w = H // p, W // p
    N = h * w
    imgs, tgts = torch.randn(B, 3, H, W, device=DEV), torch.randn(B, 3, H, W, device=DEV)
    Wp = (torch.randn(C, 3, p, p, device=DEV) * 0.02)
    bp = torch.randn(C, device=DEV) * 0.1
    cols = ops.im2col_patch(imgs, tgts, p)
    E = ops.gemm(cols, ops.cast_bf16(Wp).view(C, -1), kind=ops.EPI_F32, bias=bp)
    ref = torch.cat([F.conv2d(imgs, Wp, bp, stride=p), F.conv2d(tgts, Wp, bp, stride=p)]).permute(0, 2, 3, 1)
    assert relmax(E.view(2 * B, h, w, C), ref) < 1e-2
    mask = (torch.rand(B, N, device=DEV) < 0.5)
    mt, sx, sy = (torch.randn(C, device=DEV) for _ in range(3))
    pos = torch.randn(N, C, device=DEV)
    te = torch.randn(B, C, device=DEV)
    z = ops.assemble_tokens(E, mask.to(torch.uint8), mt, sx, sy, pos, te, B, N, C).view(2 * B, N, C)
    Ex, Ey = E.view(2 * B, N, C)[:B], E.view(2 * B, N, C)[B:]
    m = mask.float()[..., None]
    zx = Ex + sx + pos + te[:, None]
    zy = (Ey * (1 - m) + mt * m) + sy + pos + te[:, None]
    assert relmax(z, torch.cat([zx, zy])) < 1e-6
    # backward
    dZ = torch.randn(2 * B * N, C, device=DEV)
    dE, dpos, dsx, dsy, dmt = ops.assemble_tokens_bwd(dZ, mask.to(torch.uint8), B, N, C)
    d3 = dZ.view(2 * B, N, C)
    assert relmax(dpos, d3.sum(0)) < 1e-5 and relmax(dsx, d3[:B].sum((0, 1))) < 1e-5
    assert relmax(dsy, d3[B:].sum((0, 1))) < 1e-5 and relmax(dmt, (d3[B:] * m).sum((0, 1))) < 1e-5
    assert relmax(dE.view(2 * B, N, C)[B:], d3[B:] * (1 - m)) < 1e-2


@pytest.mark.parametrize("hw", [(56, 28), (8, 4), (14, 14), (112, 56)])
def test_bicubic_matches_torch_interpolate(hw):
    from painter_b200 import ops
    h, w = hw
    C = 128
    src = torch.randn(14, 14, C, device=DEV)
    ref = F.interpolate(src.permute(2, 0, 1)[None], size=(h, w), mode="bicubic", align_corners=False)[0].permute(1, 2, 0)
    assert relmax(ops.bicubic_fwd(src, h, w), ref) < 1e-5
    d = torch.randn(h, w, C, device=DEV)
    s2 = src.clone().requires_grad_(True)
    F.interpolate(s2.permute(2, 0, 1)[None], size=(h, w), mode="bicubic", align_corners=False)[0].permute(1, 2, 0) \
        .backward(d)
    assert relmax(ops.bicubic_bwd(d, 14, 14), s2.grad) < 1e-4


def test_merge_cast_colsum_ensemble():
    from painter_b200 import ops
    z = torch.randn(6, 32, 128, device=DEV)
    assert relmax(ops.merge_halves(z), (z[:3] + z[3:]) * 0.5) < 1e-6
    d = torch.randn(3, 32, 128, device=DEV)
    assert relmax(ops.merge_halves_bwd(d), torch.cat([d, d]) * 0.5) < 1e-6
    x = torch.randn(96, 384, device=DEV)
    rs = torch.tensor([1.0, 0.0, 1.25], device=DEV)
    out, cs = ops.scale_cast_colsum(x, rs, 32)
    want = x * rs.repeat_interleave(32)[:, None]
    assert relmax(out, want) < 1e-2 and relmax(cs, want.sum(0)) < 1e-5
    xb = torch.randn(1000, 384, device=DEV).bfloat16()
    assert relmax(ops.colsum_bf16(xb), xb.float().sum(0)) < 1e-5
    # SegGPT ensemble (models_seggpt.py:220-231): G=2 groups of P=3, bottom-half rows averaged inside the group
    G, P, N, C = 2, 3, 32, 128
    a, zz = torch.randn(G * P, N, C, device=DEV), torch.randn(G * P, N, C, device=DEV)
    got = ops.ensemble_resid(a, zz, G, P, N, C)
    ref = a.clone().view(G, P, N, C)
    ref[:, :, N // 2:] = ref[:, :, N // 2:].mean(1, keepdim=True)
    assert relmax(got, zz + ref.view(G * P, N, C)) < 1e-6


def test_window_partition_roundtrip_matches_reference_semantics():
    from painter_b200 import ops
    B, H, W, C, ws = 2, 8, 4, 128, 7
    x = torch.randn(B * H * W, C, device=DEV).bfloat16()
    win = ops.window_partition_bf16(x, B, H, W, ws)
    xp = F.pad(x.view(B, H, W, C), (0, 0, 0, (ws - W % ws) % ws, 0, (ws - H % ws) % ws))
    Hp, Wp = xp.shape[1], xp.shape[2]
    ref = xp.view(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, C)   # vitdet_utils.py:35-36
    assert torch.equal(win, ref)
    a = torch.randn(win.shape[0], C, device=DEV)
    res = torch.randn(B * H * W, C, device=DEV)
    rs = torch.tensor([0.0, 1.25], device=DEV)
    out = ops.window_unpartition(a, B, H, W, ws, resid=res, rowscale=rs)
    back = a.view(B, Hp // ws, Wp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, C)[:, :H, :W]
    want = res.view(B, H, W, C) + rs.view(B, 1, 1, 1) * back
    assert relmax(out.view(B, H, W, C), want) < 1e-6


# ---------------------------------------------------------------- attention -----------------------------------
def _ref_attn(qkv, th, tw, B, heads, h, w):
    N, C = h * w, heads * 64
    q, k, v = qkv.float().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q * 0.125) @ k.transpose(-1, -2)
    ih = torch.arange(h, device=DEV)[:, None] - torch.arange(h, device=DEV)[None, :] + h - 1
    iw = torch.arange(w, device=DEV)[:, None] - torch.arange(w, device=DEV)[None, :] + w - 1
    rq = q.reshape(B, heads, h, w, 64)
    rel_h = torch.einsum("bnhwc,hkc->bnhwk", rq, th.float()[ih])
    rel_w = torch.einsum("bnhwc,wkc->bnhwk", rq, tw.float()[iw])
    s = (s.reshape(B, heads, h, w, h, w) + rel_h[..., :, None] + rel_w[..., None, :]).reshape(B, heads, N, N)
    return (s.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * N, C)


@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 8, 4), (3, 1, 4, 2), (2, 2, 14, 14), (2, 1, 7, 7), (2, 2, 6, 28),
                                         (1, 2, 56, 28), (1, 1, 112, 56)])
def test_attention_fwd_bwd_vs_reference_math(B, heads, h, w):
    from painter_b200 import ops
    N, C = h * w, heads * 64
    qkv = (torch.randn(B * N, 3 * C, device=DEV) * 1.5).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=DEV) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=DEV) * 0.3)
    out, lse = ops.attn_fwd(qkv, th, tw, B, heads, h, w)
    dout = (torch.randn(B * N, C, device=DEV) * 0.5).bfloat16()
    dqkv, dTh, dTw = ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w)
    q32 = qkv.float().requires_grad_(True)
    t32, w32 = th.float().requires_grad_(True), tw.float().requires_grad_(True)
    ro = _ref_attn(q32, t32, w32, B, heads, h, w)
    assert relmax(out, ro) < 1e-2
    (ro * dout.float()).sum().backward()
    g, d = q32.grad.reshape(B * N, 3, C), dqkv.float().reshape(B * N, 3, C)
    for i in range(3):
        assert relmax(d[:, i], g[:, i]) < 2e-2, "qkv"[i]
    assert relmax(dTh, t32.grad[:2 * h - 1]) < 2e-2 and relmax(dTw, w32.grad[:2 * w - 1]) < 2e-2
    # training pair: the forward keeps the bias rows, the dQ kernel loads them instead of recomputing them
    out2, lse2, rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=True)
    assert torch.equal(out2, out) and torch.equal(lse2, lse)
    dqkv2, dTh2, dTw2 = ops.attn_bwd(qkv, out2, dout, lse2, th, tw, B, heads, h, w, rel=rel)
    # the forward stores the bias rows the recomputing pair's bias-row kernel computes with the same instructions, and
    # the dQ / dK/dV kernels read them the same way: the two pairs agree bit for bit
    assert torch.equal(dqkv2, dqkv), "saved vs recomputed"
    d2 = dqkv2.float().reshape(B * N, 3, C)
    for i in range(3):
        assert relmax(d2[:, i], g[:, i]) < 2e-2, "saved " + "qkv"[i]
    assert relmax(dTh2, t32.grad[:2 * h - 1]) < 2e-2 and relmax(dTw2, w32.grad[:2 * w - 1]) < 2e-2


@pytest.mark.parametrize("jump", [70.0, 1100.0])
def test_attention_fwd_running_max_rescale_paths(jump):
    """Scores that keep growing along the key axis: every key tile (and the second column half of every tile) outgrows
    the running reference point by more than 2^8 - resp. by more than 2^127, where exp2 of the stale reference point
    overflows - so the forward has to move the reference point and rescale O, l and the P half already written."""
    from painter_b200 import ops
    B, heads, h, w = 1, 2, 16, 28
    N, C = h * w, heads * 64
    g = torch.Generator(device="cpu").manual_seed(5)
    q = 1.0 + 0.02 * torch.randn(B * N, heads, 64, generator=g)
    u = torch.arange(N)
    c = (u // 112).float() * jump + ((u % 112) >= 64).float() * 0.8 * jump + 3.0 * torch.randn(N, generator=g)
    k = (c / 64.0)[:, None, None].expand(N, heads, 64).repeat(B, 1, 1)
    v = torch.randn(B * N, heads, 64, generator=g)
    qkv = torch.stack([q, k, v], 1).reshape(B * N, 3 * C).to(DEV).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=DEV) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=DEV) * 0.3)
    out, lse = ops.attn_fwd(qkv, th, tw, B, heads, h, w)
    ro = _ref_attn(qkv, th, tw, B, heads, h, w)
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    assert relmax(out, ro) < 1e-2


def test_attention_rows_are_convex_combinations_at_full_size():
    """Property at B=8 x 16 heads x 1568 tokens: with V = const the output equals that constant for every row,
    whatever the scores / bias (softmax rows sum to one)."""
    from painter_b200 import ops
    B, heads, h, w = 8, 16, 56, 28
    N, C = h * w, heads * 64
    qkv = (torch.randn(B * N, 3 * C, device=DEV) * 1.5).bfloat16()
    qkv[:, 2 * C:] = 0.75
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=DEV) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=DEV) * 0.3)
    out, _ = ops.attn_fwd(qkv, th, tw, B, heads, h, w)
    assert (out.float() - 0.75).abs().max().item() < 1e-2


# ---------------------------------------------------------------- decoder head --------------------------------
def _head_reference(g_nchw, c3w, c3b, lnw, lnb, c1w, c1b):
    x = F.conv2d(g_nchw, c3w, c3b, padding=1)
    x = x.bfloat16().float()  # the conv output is stored (and re-read by backward) as bf16
    mu = x.mean(1, keepdim=True)
    var = (x - mu).pow(2).mean(1, keepdim=True)
    x = (x - mu) / torch.sqrt(var + 1e-6)
    x = F.gelu(lnw[:, None, None] * x + lnb[:, None, None])
    return F.conv2d(x, c1w, c1b)


@pytest.mark.parametrize("seggpt", [False, True])
def test_decoder_head_loss_and_gradients(seggpt):
    from painter_b200 import ops
    B, H, W, p = 2, 128, 64, 16
    h, w = H // p, W // p
    g = (torch.randn(B, H, W, 64, device=DEV)).bfloat16()
    c3w = torch.randn(64, 64, 3, 3, device=DEV) * 0.05
    c3b, lnw, lnb = torch.randn(64, device=DEV) * 0.1, 1 + 0.1 * torch.randn(64, device=DEV), torch.randn(64, device=DEV) * 0.1
    c1w, c1b = torch.randn(3, 64, 1, 1, device=DEV) * 0.2, torch.randn(3, device=DEV) * 0.1
    tgts = torch.randn(B, 3, H, W, device=DEV)
    tgts[1] = (0 - torch.tensor([0.485, 0.456, 0.406], device=DEV)[:, None, None]) / \
        torch.tensor([0.229, 0.224, 0.225], device=DEV)[:, None, None]     # sample 1 triggers inds_ign (Painter)
    mask = (torch.rand(B, h * w, device=DEV) < 0.5)
    valid = torch.ones(B, 3, H, W, device=DEV)
    valid[torch.rand_like(valid) < 0.1] = 0
    valid[torch.rand_like(valid) > 0.95] = 10
    wf, wd = ops.conv3x3_pack(c3w)
    hp = torch.cat([c3b, lnw, lnb, c1w.reshape(-1), c1b, torch.zeros(5, device=DEV)])
    mu8 = mask.to(torch.uint8)
    st = ops.loss_prep(tgts, mu8, valid, p)
    c1, patch, num = ops.decoder_head_fwd(g, wf, hp, tgts, mu8, valid, p, 0)
    loss, coef = ops.loss_finalize(st, num, seggpt)
    # reference (models_painter.py:430-462 / models_seggpt.py:448-469)
    leaves = [t.clone().requires_grad_(True) for t in (g.float().permute(0, 3, 1, 2).contiguous(), c3w.bfloat16().float(),
                                                      c3b, lnw, lnb, c1w, c1b)]
    pred = _head_reference(*leaves)
    M = mask.float()[:, :, None].repeat(1, 1, p * p * 3).reshape(B, h, w, p, p, 3).permute(0, 5, 1, 3, 2, 4) \
        .reshape(B, 3, H, W)
    v = valid.clone()
    if not seggpt:
        mean = torch.tensor([0.485, 0.456, 0.406], device=DEV)[None, :, None, None]
        std = torch.tensor([0.229, 0.224, 0.225], device=DEV)[None, :, None, None]
        ign = ((tgts * std + mean) * (1 - M)).sum((1, 2, 3)) < 300
        assert ign.tolist() == [False, True]
        v[ign] = 0
    wt = M * v
    rl = (F.smooth_l1_loss(pred, tgts, reduction="none", beta=0.01) * wt).sum() / (wt.sum() + (0 if seggpt else 1e-2))
    assert abs(loss.item() - rl.item()) < 2e-3 * abs(rl.item())
    want_patch = pred.reshape(B, 3, h, p, w, p).permute(0, 2, 4, 3, 5, 1).reshape(B, h * w, p * p * 3)
    assert relmax(patch, want_patch) < 1.5e-2
    # backward
    (rl * 3.0).backward()
    gscale = torch.tensor([3.0], device=DEV)
    dc1, dhp = ops.decoder_head_bwd(c1, tgts, mu8, valid, coef, gscale, hp, p, 0)
    # the lane-pair kernel against round 1's independent warp-per-pixel implementation (same math, different
    # reduction trees): parameter gradients to fp32 summation noise, dC1 to one bf16 ulp
    from painter_b200._lib import lib
    lib().pk_head_bwd_legacy(1)
    dc1_l, dhp_l = ops.decoder_head_bwd(c1, tgts, mu8, valid, coef, gscale, hp, p, 0)
    lib().pk_head_bwd_legacy(0)
    assert relmax(dhp[64:387], dhp_l[64:387]) < 1e-4 and relmax(dc1, dc1_l) < 1e-2
    assert relmax(dhp[64:128], leaves[3].grad) < 3e-2 and relmax(dhp[128:192], leaves[4].grad) < 3e-2
    assert relmax(dhp[192:384].view(3, 64, 1, 1), leaves[5].grad) < 3e-2 and relmax(dhp[384:387], leaves[6].grad) < 3e-2
    assert relmax(ops.colsum_bf16(dc1.view(-1, 64)), leaves[2].grad) < 3e-2
    assert relmax(ops.conv3x3_wgrad(g, dc1), leaves[1].grad) < 3e-2
    dD = ops.conv3x3_dgrad_unshuffle(dc1, wd, p)     # token-major, columns (r, s, c)
    dg = leaves[0].grad.permute(0, 2, 3, 1)          # NHWC
    want = dg.reshape(B, h, p, w, p, 64).permute(0, 1, 3, 2, 4, 5).reshape(B * h * w, p * p * 64)
    assert relmax(dD, want) < 3e-2


def test_fused_adamw_and_grad_norm_match_torch():
    """SURVEY §8 f.1: the optimizer step of main_train.py:344-348 (param groups with their own lr / weight decay)
    and the gradient norm / clip of util/misc.py:252-278, against torch.optim.AdamW and clip_grad_norm_."""
    from painter_b200.optim import FusedAdamW, global_grad_norm
    torch.manual_seed(0)
    shapes = [(1024, 1024), (3,), (111, 64), (4096,), (7, 5, 3), (16384 * 3 + 5,), (64, 64, 3, 3)]
    ref = [torch.nn.Parameter(torch.randn(s, device=DEV)) for s in shapes]
    ours = [torch.nn.Parameter(p.detach().clone()) for p in ref]

    def groups(ps):
        return [{"params": ps[:3], "lr": 3e-3, "weight_decay": 0.05}, {"params": ps[3:], "lr": 1e-3, "weight_decay": 0.0}]

    o_ref = torch.optim.AdamW(groups(ref), lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    o_pk = FusedAdamW(groups(ours), lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    for step in range(4):
        gs = [torch.randn(s, device=DEV) * (10.0 if step == 2 else 1.0) for s in shapes]
        for p, q, g in zip(ref, ours, gs):
            p.grad = g.clone()
            q.grad = g.clone()
        norm_ref = torch.nn.utils.clip_grad_norm_(ref, 3.0)          # clips ref's grads in place
        norm = global_grad_norm(ours)
        assert abs(norm.item() - norm_ref.item()) < 1e-4 * norm_ref.item()
        coef = (3.0 / (norm + 1e-6)).reshape(1)
        o_ref.step()
        o_pk.step(grad_scale=coef, grad_scale_cap=1.0)
        for p, q in zip(ref, ours):
            assert relmax(q, p) < 2e-6, (step, tuple(p.shape))
    for p, q in zip(ref, ours):
        assert relmax(o_pk.state[q]["exp_avg_sq"], o_ref.state[p]["exp_avg_sq"]) < 2e-6
