"""Thin torch-tensor front end over the C ABI (include/painter_b200.h).

Every function takes CUDA tensors, passes raw device pointers + the current CUDA stream to
libpainter_b200.so and returns torch tensors.  PyTorch is only the allocator / stream provider here.
"""
import ctypes

import torch

from . import _lib
from ._lib import (EPI_BF16, EPI_DGELU, EPI_F32, EPI_GELU, EPI_PIXSHUF, EPI_RESID, PkEpilogue, check,
                   lib)

_vp = ctypes.c_void_p


def _ptr(t):
    return _vp(t.data_ptr()) if t is not None else _vp(0)


def _stream():
    return _vp(torch.cuda.current_stream().cuda_stream)


def _req(t, dtype, name):
    if not t.is_cuda:
        raise RuntimeError(f"painter_b200: {name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != dtype:
        raise RuntimeError(f"painter_b200: {name} must be {dtype}, got {t.dtype}")


def gemm(a, b, *, trans_a=False, trans_b=False, kind=EPI_BF16, out=None, out2=None, bias=None,
         aux=None, rowscale=None, rows_per_group=0, alpha=1.0, accumulate=False, pixshuf=None):
    """C[M,N] = A[M,K] . B[N,K]^T on the tensor cores (wgmma; bf16 in, fp32 accumulate).

    a: [M,K] (or [K,M] when trans_a);  b: [N,K] (or [K,N] when trans_b); last dim contiguous.
    pixshuf = (h, w, p, c, out_tensor[B, h*p, w*p, c]) for EPI_PIXSHUF.
    """
    _req(a, torch.bfloat16, "a")
    _req(b, torch.bfloat16, "b")
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    if trans_a:
        K, M = a.shape
    else:
        M, K = a.shape
    if trans_b:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, (a.shape, b.shape, trans_a, trans_b)
    e = PkEpilogue()
    e.kind = kind
    if kind == EPI_PIXSHUF:
        h, w, p, c, out = pixshuf
        e.ps_h, e.ps_w, e.ps_p, e.ps_c = h, w, p, c
        _req(out, torch.bfloat16, "out")
        assert out.is_contiguous()
        e.ldc = N
    else:
        if out is None:
            odt = torch.float32 if kind in (EPI_F32, EPI_RESID) else torch.bfloat16
            out = torch.empty((M, N), dtype=odt, device=a.device)
        assert out.stride(1) == 1 and tuple(out.shape) == (M, N)
        e.ldc = out.stride(0)
    if kind == EPI_GELU:
        if out2 is None:
            out2 = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
        assert out2.stride() == out.stride()
    e.out = out.data_ptr()
    e.out2 = out2.data_ptr() if out2 is not None else None
    if bias is not None:
        _req(bias, torch.float32, "bias")
        assert bias.numel() == N and bias.is_contiguous()
        e.bias = bias.data_ptr()
    if aux is not None:
        assert aux.stride(1) == 1 and tuple(aux.shape) == (M, N)
        _req(aux, torch.float32 if kind == EPI_RESID else torch.bfloat16, "aux")
        e.aux = aux.data_ptr()
        e.ld_aux = aux.stride(0)
    if rowscale is not None:
        _req(rowscale, torch.float32, "rowscale")
        e.rowscale = rowscale.data_ptr()
        e.rows_per_group = rows_per_group
    e.alpha = alpha
    e.accumulate = int(accumulate)  # 0 overwrite, 1 read-modify-write, 2 zero-initialised + split-K atomics
    check(lib().pk_gemm_bf16(_ptr(a), _ptr(b), M, N, K, a.stride(0), b.stride(0), int(trans_a),
                             int(trans_b), ctypes.byref(e), _stream()), "pk_gemm_bf16")
    if kind == EPI_GELU:
        return out, out2
    return out


def _pad16(n):
    return (n + 15) // 16 * 16


def relpos_table_bf16(table):
    """fp32 [L, 64] rel-pos table -> zero-padded bf16 [pad16(L), 64] (attention kernel operand)."""
    _req(table, torch.float32, "table")
    assert table.dim() == 2 and table.shape[1] == 64 and table.is_contiguous()
    L = table.shape[0]
    out = torch.empty((_pad16(L), 64), dtype=torch.bfloat16, device=table.device)
    check(lib().pk_relpos_table_bf16(_ptr(table), _ptr(out), L, out.shape[0], _stream()), "pk_relpos_table_bf16")
    return out


def attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=False):
    """Fused attention forward. qkv: bf16 [B*h*w, 3*heads*64]; th/tw: padded bf16 tables for an (h, w) grid.
    Returns (out bf16 [B*h*w, heads*64], lse fp32 [B*heads, h*w] in the log2 domain); with save_rel=True a third
    value: the (relh, relw) bias-row buffers the forward keeps for `attn_bwd(..., rel=...)`.  The module does not use
    that pair (72 MB of extra saved activations per block application at batch 8, to save one small kernel); the
    tests compare the recomputing backward against it."""
    _req(qkv, torch.bfloat16, "qkv")
    N, C = h * w, heads * 64
    assert qkv.is_contiguous() and tuple(qkv.shape) == (B * N, 3 * C)
    assert th.shape[0] >= 2 * h - 1 and tw.shape[0] >= 2 * w - 1
    out = torch.empty((B * N, C), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((B * heads, N), dtype=torch.float32, device=qkv.device)
    if save_rel:
        Np = (N + 127) // 128 * 128     # whole 128-query tiles, query row innermost
        relh = torch.empty((B * heads * Np * h,), dtype=torch.float32, device=qkv.device)
        relw = torch.empty((B * heads * Np * w,), dtype=torch.float32, device=qkv.device)
        check(lib().pk_attn_fwd_save(_ptr(qkv), _ptr(th), _ptr(tw), _ptr(out), _ptr(lse), _ptr(relh), _ptr(relw),
                                     B, heads, h, w, th.shape[0], tw.shape[0], _stream()), "pk_attn_fwd_save")
        return out, lse, (relh, relw)
    check(lib().pk_attn_fwd(_ptr(qkv), _ptr(th), _ptr(tw), _ptr(out), _ptr(lse), B, heads, h, w,
                            th.shape[0], tw.shape[0], _stream()), "pk_attn_fwd")
    return out, lse


def attn_fwd_split3(qkv, th, tw, B, heads, h, w):
    """fp32-accurate fused attention forward (split-bf16 products, accumulated in fp32).  qkv: fp32 [B*h*w, 3*heads*64];
    th / tw: fp32 rel-pos tables [2h-1, 64] / [2w-1, 64].  Returns out fp32 [B*h*w, heads*64]."""
    _req(qkv, torch.float32, "qkv")
    _req(th, torch.float32, "th")
    _req(tw, torch.float32, "tw")
    N, C = h * w, heads * 64
    assert qkv.is_contiguous() and tuple(qkv.shape) == (B * N, 3 * C)
    assert th.is_contiguous() and tw.is_contiguous()
    assert tuple(th.shape) == (2 * h - 1, 64) and tuple(tw.shape) == (2 * w - 1, 64)
    out = torch.empty((B * N, C), dtype=torch.float32, device=qkv.device)
    check(lib().pk_attn_fwd_split3(_ptr(qkv), _ptr(th), _ptr(tw), _ptr(out), B, heads, h, w, _stream()),
          "pk_attn_fwd_split3")
    return out


def attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, dT_out=None, rel=None, table_grads=True):
    """Fused attention backward.  Returns (dqkv bf16 [B*N, 3C], dTh fp32 [2h-1, 64], dTw fp32 [2w-1, 64]).
    rel: the (relh, relw) buffers of `attn_fwd(..., save_rel=True)` on the same operands (the dQ kernel then loads its
    bias rows instead of recomputing them).  table_grads=False (frozen tables): dTh = dTw = None, the table-gradient
    work is skipped and dqkv is bit-identical."""
    N, C = h * w, heads * 64
    _req(dout, torch.bfloat16, "dout")
    assert dout.is_contiguous() and out.is_contiguous() and qkv.is_contiguous()
    dev = qkv.device
    dqkv = torch.empty_like(qkv)
    if not table_grads:
        dTh = dTw = None
    elif dT_out is not None:       # caller-provided, zero-initialised (or running) fp32 accumulators
        dTh, dTw = dT_out
        assert tuple(dTh.shape) == (2 * h - 1, 64) and tuple(dTw.shape) == (2 * w - 1, 64)
        assert dTh.is_contiguous() and dTw.is_contiguous() and dTh.dtype == torch.float32
    else:
        dTh = torch.zeros((2 * h - 1, 64), dtype=torch.float32, device=dev)
        dTw = torch.zeros((2 * w - 1, 64), dtype=torch.float32, device=dev)
    delta = torch.empty((B * heads * N,), dtype=torch.float32, device=dev)
    Np = (N + 127) // 128 * 128     # the bias-row scratch is laid out in whole 128-query tiles
    L = lib()
    L.pk_attn_bwd_ws_floats.restype = ctypes.c_longlong
    dt_ws = (torch.empty((int(L.pk_attn_bwd_ws_floats(B, heads, h, w)),), dtype=torch.float32, device=dev)
             if table_grads else None)
    if rel is not None:
        relh_g, relw_g = rel
        assert relh_g.numel() == B * heads * Np * h and relw_g.numel() == B * heads * Np * w
        _req(relh_g, torch.float32, "relh")
        _req(relw_g, torch.float32, "relw")
        check(L.pk_attn_bwd_saved(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse), _ptr(th), _ptr(tw), _ptr(dqkv),
                                  _ptr(dTh), _ptr(dTw), _ptr(delta), _ptr(relh_g), _ptr(relw_g), _ptr(dt_ws), B, heads,
                                  h, w, th.shape[0], tw.shape[0], _stream()), "pk_attn_bwd_saved")
        return dqkv, dTh, dTw
    relh_g = torch.empty((B * heads * Np * h,), dtype=torch.float32, device=dev)
    relw_g = torch.empty((B * heads * Np * w,), dtype=torch.float32, device=dev)
    check(L.pk_attn_bwd(_ptr(qkv), _ptr(out), _ptr(dout), _ptr(lse), _ptr(th), _ptr(tw), _ptr(dqkv),
                        _ptr(dTh), _ptr(dTw), _ptr(delta), _ptr(relh_g), _ptr(relw_g), _ptr(dt_ws), B, heads, h, w,
                        th.shape[0], tw.shape[0], _stream()), "pk_attn_bwd")
    return dqkv, dTh, dTw


# --------------------------------------------------------------------------------------------------
# bandwidth kernels
# --------------------------------------------------------------------------------------------------
def layernorm_fwd(x, gamma, beta, eps, out=None, out_dtype=torch.bfloat16, want_stats=True):
    """x fp32 [M, C] (row stride free) -> LN(x) (bf16 or fp32, may be a column slice of a wider buffer)."""
    _req(x, torch.float32, "x")
    M, C = x.shape
    assert x.stride(1) == 1
    if out is None:
        out = torch.empty((M, C), dtype=out_dtype, device=x.device)
    assert out.stride(1) == 1 and tuple(out.shape) == (M, C)
    mean = torch.empty((M,), dtype=torch.float32, device=x.device) if want_stats else None
    rstd = torch.empty((M,), dtype=torch.float32, device=x.device) if want_stats else None
    check(lib().pk_layernorm_fwd(_ptr(x), x.stride(0), _ptr(gamma), _ptr(beta), ctypes.c_float(eps), _ptr(out),
                                 out.stride(0), int(out.dtype == torch.bfloat16), _ptr(mean), _ptr(rstd), M, C,
                                 _stream()), "pk_layernorm_fwd")
    return out, mean, rstd


def layernorm_bwd(dy, x, mean, rstd, gamma, dgamma, dbeta, dres=None, cast=None):
    """Returns dx fp32 [M, C] (+ dres); accumulates into dgamma / dbeta (fp32, caller-initialised).
    cast = (rowscale or None, rows_per_group, colsum_out[C]): also returns bf16(rowscale * dx) and adds its column
    sums to colsum_out (the fused form of `scale_cast_colsum(layernorm_bwd(...))`).
    dgamma = dbeta = None (frozen LayerNorm) / colsum_out = None: that reduction is skipped; dx is unchanged."""
    if dy.dtype != torch.bfloat16:
        _req(dy, torch.float32, "dy")
    dyb = int(dy.dtype == torch.bfloat16)
    _req(x, torch.float32, "x")
    M, C = x.shape
    assert dy.stride(1) == 1 and x.stride(1) == 1
    dx = torch.empty((M, C), dtype=torch.float32, device=x.device)
    if dres is not None:
        assert dres.is_contiguous()
    L = lib()
    L.pk_layernorm_bwd_ws_floats.restype = ctypes.c_longlong
    sums = dgamma is not None or dbeta is not None or (cast is not None and cast[2] is not None)
    ws = torch.empty((int(L.pk_layernorm_bwd_ws_floats(M, C)),), dtype=torch.float32, device=x.device) if sums else None
    if cast is not None:
        rowscale, rpg, cs = cast
        dxb = torch.empty((M, C), dtype=torch.bfloat16, device=x.device)
        check(L.pk_layernorm_bwd_cast(_ptr(dy), dyb, dy.stride(0), _ptr(x), x.stride(0), _ptr(mean), _ptr(rstd),
                                      _ptr(gamma), _ptr(dres), _ptr(dx), _ptr(dgamma), _ptr(dbeta), _ptr(ws),
                                      _ptr(rowscale), rpg, _ptr(dxb), _ptr(cs), M, C, _stream()),
              "pk_layernorm_bwd_cast")
        return dx, dxb
    check(L.pk_layernorm_bwd(_ptr(dy), dyb, dy.stride(0), _ptr(x), x.stride(0), _ptr(mean), _ptr(rstd), _ptr(gamma),
                             _ptr(dres), _ptr(dx), _ptr(dgamma), _ptr(dbeta), _ptr(ws), M, C, _stream()),
          "pk_layernorm_bwd")
    return dx


def im2col_patch(imgs, tgts, p):
    _req(imgs, torch.float32, "imgs")
    _req(tgts, torch.float32, "tgts")
    assert imgs.is_contiguous() and tgts.is_contiguous() and imgs.shape == tgts.shape
    B, Cin, H, W = imgs.shape
    out = torch.empty((2 * B * (H // p) * (W // p), Cin * p * p), dtype=torch.bfloat16, device=imgs.device)
    check(lib().pk_im2col_patch(_ptr(imgs), _ptr(tgts), _ptr(out), B, Cin, H, W, p, _stream()), "pk_im2col_patch")
    return out


def col2im_patch(dcols_x, dcols_y, B, Cin, H, W, p):
    """Input gradient of `im2col_patch`: the patch-embed dgrad of the x rows / y rows, fp32 [B*(H/p)*(W/p), Cin*p*p]
    each (None: that half is not wanted) -> (dimgs, dtgts) fp32 NCHW, None where not wanted."""
    out = []
    for d in (dcols_x, dcols_y):
        if d is not None:
            _req(d, torch.float32, "dcols")
            assert d.is_contiguous() and tuple(d.shape) == (B * (H // p) * (W // p), Cin * p * p)
        out.append(torch.empty((B, Cin, H, W), dtype=torch.float32, device=d.device) if d is not None else None)
    dimgs, dtgts = out
    check(lib().pk_col2im_patch(_ptr(dcols_x), _ptr(dcols_y), _ptr(dimgs), _ptr(dtgts), B, Cin, H, W, p, _stream()),
          "pk_col2im_patch")
    return dimgs, dtgts


def assemble_tokens(E, mask_u8, mask_token, seg_x, seg_y, pos, type_emb, B, N, C):
    out = torch.empty_like(E)
    check(lib().pk_assemble_tokens(_ptr(E), _ptr(mask_u8), mask_u8.shape[0], _ptr(mask_token), _ptr(seg_x),
                                   _ptr(seg_y), _ptr(pos), _ptr(type_emb), _ptr(out), B, N, C, _stream()),
          "pk_assemble_tokens")
    return out


def assemble_tokens_bwd(dZ, mask_u8, B, N, C, token_grads=None, want_tokens=True, want_pos=True, type_grads=None):
    """token_grads: optional (dseg_x, dseg_y, dmask_token) zero-initialised fp32 [C] accumulators (arena views).
    want_tokens=False / want_pos=False (frozen parameters): those gradients are skipped and returned as None.
    type_grads: optional (seg_type fp32 [B], dtype_cls, dtype_ins) - SegGPT's type-token gradients are accumulated
    into the two zero-initialised fp32 [C] buffers in the same pass."""
    dev = dZ.device
    dE = torch.empty((2 * B * N, C), dtype=torch.bfloat16, device=dev)
    dpos = torch.empty((N, C), dtype=torch.float32, device=dev) if want_pos else None
    if not want_tokens:
        token_grads = (None, None, None)
    elif token_grads is None:
        small = torch.zeros((3, C), dtype=torch.float32, device=dev)
        token_grads = (small[0], small[1], small[2])
    sx, sy, mt = token_grads
    st, tc, ti = type_grads if type_grads is not None else (None, None, None)
    if st is not None:
        _req(st, torch.float32, "seg_type")
        assert st.is_contiguous() and st.numel() == B
    check(lib().pk_assemble_tokens_bwd_typed(_ptr(dZ), _ptr(mask_u8), mask_u8.shape[0], _ptr(dE), _ptr(dpos),
                                             _ptr(sx), _ptr(sy), _ptr(mt), _ptr(st), _ptr(tc), _ptr(ti), B, N, C,
                                             _stream()),
          "pk_assemble_tokens_bwd_typed")
    return dE, dpos, sx, sy, mt


def bicubic_fwd(src, h, w):
    """src fp32 [s, s, C] -> [h, w, C]  (F.interpolate bicubic, align_corners=False)."""
    sh, sw, C = src.shape
    out = torch.empty((h, w, C), dtype=torch.float32, device=src.device)
    check(lib().pk_bicubic_fwd(_ptr(src), _ptr(out), sh, sw, h, w, C, _stream()), "pk_bicubic_fwd")
    return out


def bicubic_bwd(dout, sh, sw, out=None):
    """out: optional zero-initialised (or running) fp32 [sh, sw, C] accumulator."""
    h, w, C = dout.shape
    dsrc = out if out is not None else torch.zeros((sh, sw, C), dtype=torch.float32, device=dout.device)
    check(lib().pk_bicubic_bwd(_ptr(dout), _ptr(dsrc), sh, sw, h, w, C, _stream()), "pk_bicubic_bwd")
    return dsrc


def merge_halves(z):
    half = z.shape[0] // 2
    out = torch.empty((half,) + tuple(z.shape[1:]), dtype=torch.float32, device=z.device)
    check(lib().pk_merge_halves(_ptr(z), _ptr(out), ctypes.c_longlong(out.numel()), _stream()), "pk_merge_halves")
    return out


def merge_halves_bwd(d):
    out = torch.empty((2 * d.shape[0],) + tuple(d.shape[1:]), dtype=torch.float32, device=d.device)
    check(lib().pk_merge_halves_bwd(_ptr(d), _ptr(out), ctypes.c_longlong(d.numel()), _stream()),
          "pk_merge_halves_bwd")
    return out


def cast_bf16(x):
    _req(x, torch.float32, "x")
    assert x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    check(lib().pk_cast_bf16(_ptr(x), _ptr(out), ctypes.c_longlong(x.numel()), _stream()), "pk_cast_bf16")
    return out


def scale_cast_colsum(x, rowscale=None, rows_per_group=0, want_colsum=True, colsum_out=None):
    """fp32 [M, C] -> (bf16 [M, C] scaled per row group, column sums fp32 [C]).  colsum_out: pre-zeroed [C] buffer."""
    _req(x, torch.float32, "x")
    M, C = x.shape
    out = torch.empty((M, C), dtype=torch.bfloat16, device=x.device)
    if colsum_out is not None:
        cs = colsum_out
    else:
        cs = torch.zeros((C,), dtype=torch.float32, device=x.device) if want_colsum else None
    check(lib().pk_scale_cast_colsum(_ptr(x), x.stride(0), _ptr(rowscale), rows_per_group, _ptr(out), _ptr(cs), M, C,
                                     _stream()), "pk_scale_cast_colsum")
    return out, cs


def colsum_bf16(x, out=None):
    """Column sums of a bf16 [M, C] matrix, accumulated into `out` (pre-zeroed fp32 [C]) if given."""
    _req(x, torch.bfloat16, "x")
    M, C = x.shape
    cs = out if out is not None else torch.zeros((C,), dtype=torch.float32, device=x.device)
    check(lib().pk_colsum_bf16(_ptr(x), x.stride(0), _ptr(cs), M, C, _stream()), "pk_colsum_bf16")
    return cs


def ensemble_resid(a, z, G, P, N, C):
    out = torch.empty_like(z)
    check(lib().pk_ensemble_resid(_ptr(a), _ptr(z), _ptr(out), G, P, N, C, _stream()), "pk_ensemble_resid")
    return out


# --------------------------------------------------------------------------------------------------
# decoder head
# --------------------------------------------------------------------------------------------------
def conv3x3_pack(w):
    _req(w, torch.float32, "w")
    assert tuple(w.shape) == (64, 64, 3, 3) and w.is_contiguous()
    wf = torch.empty((64, 576), dtype=torch.bfloat16, device=w.device)
    wd = torch.empty((64, 576), dtype=torch.bfloat16, device=w.device)
    check(lib().pk_conv3x3_pack(_ptr(w), _ptr(wf), _ptr(wd), _stream()), "pk_conv3x3_pack")
    return wf, wd


def loss_prep(tgts, mask_u8, valid, p):
    B, _, H, W = tgts.shape
    stats = torch.zeros((B, 2), dtype=torch.float32, device=tgts.device)
    check(lib().pk_loss_prep(_ptr(tgts), _ptr(mask_u8), mask_u8.shape[0], _ptr(valid), _ptr(stats), B, H, W, p,
                             _stream()), "pk_loss_prep")
    return stats


# The decoder head's packed parameter vector (pk_decoder_head_fwd / pk_decoder_head_bwd / pk_head_f32), fp32 [392]:
# conv3x3 bias [64] | LayerNorm2D weight [64] | bias [64] | conv1x1 weight [3*64] | conv1x1 bias [3] | 5 zeros.  The
# head backward returns the gradients of the last four in the same slices (the conv3x3 bias gradient is a column sum
# of dc1 instead).
HEAD_SLICES = {"ln_w": slice(64, 128), "ln_b": slice(128, 192), "c1_w": slice(192, 384), "c1_b": slice(384, 387)}


def pack_head_params(c3_b, ln_w, ln_b, c1_w, c1_b):
    return torch.cat([c3_b, ln_w, ln_b, c1_w.reshape(-1), c1_b, c1_b.new_zeros(5)]).contiguous()


def decoder_head_fwd(g_nhwc, wf, head_params, tgts, mask_u8, valid, p, loss_kind):
    B, H, W, c = g_nhwc.shape
    assert c == 64 and g_nhwc.is_contiguous()
    dev = g_nhwc.device
    c1 = torch.empty((B, H, W, 64), dtype=torch.bfloat16, device=dev)
    patch = torch.empty((B, (H // p) * (W // p), p * p * 3), dtype=torch.float32, device=dev)
    num = torch.zeros((B,), dtype=torch.float32, device=dev)
    check(lib().pk_decoder_head_fwd(_ptr(g_nhwc), _ptr(wf), _ptr(head_params), _ptr(tgts), _ptr(mask_u8),
                                    mask_u8.shape[0], _ptr(valid), _ptr(c1), _ptr(patch), _ptr(num), B, H, W, p,
                                    loss_kind, _stream()), "pk_decoder_head_fwd")
    return c1, patch, num


def loss_finalize(stats, num, seggpt):
    B = num.shape[0]
    loss = torch.empty((1,), dtype=torch.float32, device=num.device)
    coef = torch.empty((B,), dtype=torch.float32, device=num.device)
    check(lib().pk_loss_finalize(_ptr(stats), _ptr(num), _ptr(loss), _ptr(coef), B, int(seggpt), _stream()),
          "pk_loss_finalize")
    return loss, coef


def decoder_head_bwd(c1, tgts, mask_u8, valid, coef, gscale, head_params, p, loss_kind, params=True):
    """Returns (dc1 bf16 NHWC, dhp fp32 [392]); params=False (frozen head): no parameter reductions, dhp is None."""
    B, H, W, _ = c1.shape
    dc1 = torch.empty_like(c1)
    dhp = torch.zeros((392,), dtype=torch.float32, device=c1.device) if params else None
    check(lib().pk_decoder_head_bwd(_ptr(c1), _ptr(tgts), _ptr(mask_u8), mask_u8.shape[0], _ptr(valid), _ptr(coef),
                                    _ptr(gscale), _ptr(head_params), _ptr(dc1), _ptr(dhp), B, H, W, p, loss_kind,
                                    _stream()), "pk_decoder_head_bwd")
    return dc1, dhp


def decoder_head_bwd_dtgt(c1, tgts, mask_u8, valid, coef, gscale, head_params, p, loss_kind, params=True):
    """decoder_head_bwd that also returns the loss's gradient with respect to the targets, dtgts fp32 NCHW = -dpred
    (not including the targets' path through the encoder): (dc1, dhp or None, dtgts)."""
    B, H, W, _ = c1.shape
    dc1 = torch.empty_like(c1)
    dhp = torch.zeros((392,), dtype=torch.float32, device=c1.device) if params else None
    dt = torch.empty(tgts.shape, dtype=torch.float32, device=c1.device)
    check(lib().pk_decoder_head_bwd_dtgt(_ptr(c1), _ptr(tgts), _ptr(mask_u8), mask_u8.shape[0], _ptr(valid),
                                         _ptr(coef), _ptr(gscale), _ptr(head_params), _ptr(dc1), _ptr(dhp), _ptr(dt),
                                         B, H, W, p, loss_kind, _stream()), "pk_decoder_head_bwd_dtgt")
    return dc1, dhp, dt


def conv3x3_dgrad_unshuffle(dc1, wd, p):
    B, H, W, _ = dc1.shape
    out = torch.empty((B * (H // p) * (W // p), p * p * 64), dtype=torch.bfloat16, device=dc1.device)
    check(lib().pk_conv3x3_dgrad_unshuffle(_ptr(dc1), _ptr(wd), _ptr(out), B, H, W, p, _stream()),
          "pk_conv3x3_dgrad_unshuffle")
    return out


def conv3x3_wgrad(g_nhwc, dc1, out=None):
    B, H, W, _ = dc1.shape
    acc = torch.zeros((640, 64), dtype=torch.float32, device=dc1.device)
    check(lib().pk_conv3x3_wgrad(_ptr(g_nhwc), _ptr(dc1), _ptr(acc), B, H, W, _stream()), "pk_conv3x3_wgrad")
    dw = out if out is not None else torch.empty((64, 64, 3, 3), dtype=torch.float32, device=dc1.device)
    assert dw.is_contiguous() and tuple(dw.shape) == (64, 64, 3, 3)
    check(lib().pk_conv3x3_wgrad_unpack(_ptr(acc), _ptr(dw), _stream()), "pk_conv3x3_wgrad_unpack")
    return dw


def window_partition_bf16(x, B, H, W, ws):
    """bf16 [B*H*W, C] -> zero-padded windows [B*nWh*nWw*ws*ws, C]."""
    _req(x, torch.bfloat16, "x")
    C = x.shape[1]
    nWh, nWw = (H + ws - 1) // ws, (W + ws - 1) // ws
    out = torch.empty((B * nWh * nWw * ws * ws, C), dtype=torch.bfloat16, device=x.device)
    check(lib().pk_window_partition_bf16(_ptr(x), _ptr(out), B, H, W, C, ws, _stream()), "pk_window_partition_bf16")
    return out


def window_unpartition(win, B, H, W, ws, resid=None, rowscale=None):
    """fp32 windows -> fp32 [B*H*W, C] (+ resid, per-sample scale)."""
    _req(win, torch.float32, "win")
    C = win.shape[1]
    out = torch.empty((B * H * W, C), dtype=torch.float32, device=win.device)
    check(lib().pk_window_unpartition(_ptr(win), _ptr(resid), _ptr(rowscale), _ptr(out), B, H, W, C, ws, _stream()),
          "pk_window_unpartition")
    return out


def droppath_scales(r, keep):
    """timm DropPath scales for a whole step: r = concatenated torch.rand draws (fp32 / bf16 / fp16, the dtype the
    reference draws in), keep = per-element keep probability (fp32).  Returns floor(round_dtype(keep + r)) / keep."""
    code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[r.dtype]
    assert r.is_contiguous() and keep.is_contiguous() and keep.dtype == torch.float32 and keep.numel() == r.numel()
    out = torch.empty(r.numel(), dtype=torch.float32, device=r.device)
    check(lib().pk_droppath_scales(_ptr(r), code, _ptr(keep), _ptr(out), r.numel(), _stream()), "pk_droppath_scales")
    return out


def set_sm_budget(n):
    """Cap the SM count the persistent kernels size their grids for (0 = all SMs); returns the previous cap."""
    return int(lib().pk_set_sm_budget(int(n)))


def set_pdl(on):
    """Programmatic dependent launch of the hot kernels (include/painter_b200.h: pk_set_pdl); returns the previous
    setting.  Default on (PK_PDL=0 in the environment disables it)."""
    return int(lib().pk_set_pdl(int(bool(on))))
