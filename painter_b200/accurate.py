"""fp32-ACCURATE forward of the painter_b200 modules (north star: within 1e-5 of the reference's fp32 forward; the
reference runs inference exactly so - `model(x.float(), ...)` with no autocast, seggpt_engine.py:47,
painter_inference_segm.py:83).

Selected by `model.precision`:  "bf16" = the training arithmetic (bf16 tensor-core operands, fp32 accumulate);
"fp32" = this path; "auto" (default) = this path when the module is called outside autocast with gradients disabled
(i.e. the reference's fp32 inference calls), bf16 otherwise.  Forward only - the reference never trains in fp32.

Still tensor-core code: every GEMM operand is split into three bf16 terms and the six significant cross products run as
ONE pk_gemm_bf16 call over K-concatenated operands (csrc/accurate.cu has the derivation); softmax, LayerNorm, GELU
(exact erf), the residual stream and the loss stay fp32 (the loss numerator accumulates in fp64).  Global blocks
materialise the score matrix per (sample, head) like the reference does (`attention`); windowed blocks run all their
windows through one fused kernel in the same split arithmetic (ops.attn_fwd_split3) - this mode is about digits,
not speed: 6x the tensor-core work of the bf16 path plus the split passes.

Stage map = engine.py's (same reference lines): embed, 24 blocks (+ early merge, SegGPT ensemble), decoder, loss.
"""
import ctypes

import torch

from . import ops
from ._lib import check, lib
from .ops import EPI_F32, EPI_RESID, _ptr, _stream


def _pad64(n):
    return (n + 63) // 64 * 64


def selected(model):
    """Whether a forward of `model` called now runs this path (model.precision, see the module docstring)."""
    prec = model.precision
    return prec == "fp32" or (prec == "auto" and not torch.is_autocast_enabled("cuda") and
                              not torch.is_grad_enabled())


def workspace_bytes(model, B, H, W):
    """Device memory a forward of B canvases [3, H, W] in this mode allocates at its peak, from the shapes: the global
    blocks before the early merge (2B token grids) hold the per-(sample, head) score matrix and split operands of
    `attention`, the rel-pos projections, the block's fp32 activations and the split qkv operand; the decoder (one
    image's im2col at a time) needs less for the stock geometry but is counted in case it does not.  Includes the
    weights' split copies when they are not cached yet."""
    p, C, heads = model.patch_size, model.embed_dim, model.num_heads
    h, w = H // p, W // p
    N, Bp = h * w, 2 * B
    Np = _pad64(N)
    attn = Bp * heads * (N * 384 * 2 + Np * 384 * 2 + 6 * Np * 64 * 2 + N * Np * 4 + N * 6 * Np * 2 +
                         N * (_pad64(2 * h - 1) + _pad64(2 * w - 1)) * 4)
    blocks = attn + Bp * N * C * (4 + 4 + 12 + 12 + 4)          # z, u, split3(u), qkv, attention output
    dd = model.decoder_embed_dim
    dec = B * N * C * 4 * 8 + B * N * p * p * dd * 4 + B * H * W * 64 * 4 + H * W * 6 * 9 * dd * 2
    need = max(blocks, dec)
    if getattr(model.blocks[0].attn.qkv.weight, "_pk_split3", None) is None:
        need += 12 * sum(q.numel() for q in model.parameters() if q.dim() >= 2)
    return need


def split3(x, side_b=False, gelu=False):
    """fp32 [M, K] (row stride free) -> bf16 [M, 6K] split operand (A-side or B-side term order)."""
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    out = torch.empty((M, 6 * K), dtype=torch.bfloat16, device=x.device)
    check(lib().pk_split3(_ptr(x), x.stride(0), _ptr(out), M, K, int(side_b), int(gelu), _stream()), "pk_split3")
    return out


def split_weight(p, shape2d=None, pad_rows=0):
    """B-side split copy [N(+pad), 6K] of an fp32 parameter, cached on the parameter like engine.bf16_weight."""
    ent = getattr(p, "_pk_split3", None)
    if ent is not None and ent[0] == p._version and ent[1] == p.data_ptr() and ent[2].device == p.device and \
            ent[3] == pad_rows:
        return ent[2]
    src = p.detach().contiguous()
    if shape2d is not None:
        src = src.view(shape2d)
    w = split3(src, side_b=True)
    if pad_rows > w.shape[0]:
        wp = torch.zeros((pad_rows, w.shape[1]), dtype=torch.bfloat16, device=w.device)
        wp[:w.shape[0]] = w
        w = wp
    p._pk_split3 = (p._version, p.data_ptr(), w, pad_rows)
    return w


def _gemm(a6, b6, **kw):
    return ops.gemm(a6, b6, **kw)


class _AttnWorkspace:
    """Zero-initialised split operands whose padding must stay zero (keys / probabilities beyond N)."""

    def __init__(self, BH, N, dev):
        Np = _pad64(N)
        self.BH, self.N, self.Np = BH, N, Np
        self.q = torch.empty((BH, N, 384), dtype=torch.bfloat16, device=dev)
        self.k = torch.zeros((BH, Np, 384), dtype=torch.bfloat16, device=dev)
        self.v = torch.zeros((BH, 6 * Np, 64), dtype=torch.bfloat16, device=dev)
        self.S = torch.empty((BH, N, Np), dtype=torch.float32, device=dev)
        self.P = torch.zeros((BH, N, 6 * Np), dtype=torch.bfloat16, device=dev)


def attention(u, blk, Bp, h, w, heads, ws_cache, rel_h, rel_w):
    """u fp32 [Bp*N, C] (LayerNorm output) -> attention output before proj, fp32 [Bp*N, C]
    (models_painter.py:73-86 + vitdet_utils.py:96-125)."""
    N, C = h * w, heads * 64
    dev = u.device
    a = blk.attn
    qkv = _gemm(split3(u), split_weight(a.qkv.weight), kind=EPI_F32, bias=a.qkv.bias)          # [M, 3C] fp32
    BH = Bp * heads
    ws = ws_cache.get((BH, N))
    if ws is None:
        ws = _AttnWorkspace(BH, N, dev)
        ws_cache[(BH, N)] = ws
    L = lib()
    for which, dst in ((0, ws.q), (1, ws.k), (2, ws.v)):
        check(L.pk_split3_heads(_ptr(qkv), _ptr(dst), Bp, heads, N, ws.Np, which, _stream()), "pk_split3_heads")
    # decomposed rel-pos projections for every (b, head, query) at once: G = q . T^T  (bias uses the UNSCALED q)
    Lh, Lw = 2 * h - 1, 2 * w - 1
    th = split_weight(rel_h, pad_rows=_pad64(Lh)) if isinstance(rel_h, torch.nn.Parameter) else _split_table(rel_h, Lh)
    tw = split_weight(rel_w, pad_rows=_pad64(Lw)) if isinstance(rel_w, torch.nn.Parameter) else _split_table(rel_w, Lw)
    qall = ws.q.view(BH * N, 384)
    Gh = _gemm(qall, th, kind=EPI_F32)
    Gw = _gemm(qall, tw, kind=EPI_F32)
    for bh in range(BH):
        _gemm(ws.q[bh], ws.k[bh], kind=EPI_F32, out=ws.S[bh])
    check(L.pk_softmax_relpos_split3(_ptr(ws.S), _ptr(Gh), Gh.shape[1], _ptr(Gw), Gw.shape[1], _ptr(ws.P), BH, N, ws.Np,
                                     h, w, ctypes.c_float(0.125), _stream()), "pk_softmax_relpos_split3")
    ao = torch.empty((Bp * N, C), dtype=torch.float32, device=dev)
    for bh in range(BH):
        b, hd = divmod(bh, heads)
        _gemm(ws.P[bh], ws.v[bh], trans_b=True, kind=EPI_F32, out=ao[b * N:(b + 1) * N, hd * 64:(hd + 1) * 64])
    return ao


def _split_table(t, L):
    w = split3(t.detach().float().contiguous(), side_b=True)
    wp = torch.zeros((_pad64(L), w.shape[1]), dtype=torch.bfloat16, device=w.device)
    wp[:w.shape[0]] = w
    return wp


def block(z, blk, Bp, h, w, heads, eps, ens, ws_cache, rel_h, rel_w):
    """models_painter.py:216-235 (+ SegGPT ensemble models_seggpt.py:220-231); eval mode (DropPath = identity).
    rel_h / rel_w: the block's tables for its attention grid (the window for a windowed block)."""
    N = h * w
    C = z.shape[1]
    ws = blk.window_size
    u, _, _ = ops.layernorm_fwd(z, blk.norm1.weight, blk.norm1.bias, eps, out_dtype=torch.float32, want_stats=False)
    a = blk.attn
    if ws > 0:
        # vitdet_utils.py:16-60: LN1's output is zero-padded to whole windows BEFORE qkv, so padded tokens carry the qkv
        # bias and take part as keys.  Partitioning the split operand is exact: zero rows split to zero.
        us = ops.window_partition_bf16(split3(u), Bp, h, w, ws)
        Bw = us.shape[0] // (ws * ws)
        qkv = _gemm(us, split_weight(a.qkv.weight), kind=EPI_F32, bias=a.qkv.bias)
        ao = ops.attn_fwd_split3(qkv, rel_h.detach().contiguous(), rel_w.detach().contiguous(), Bw, heads, ws, ws)
        pa = _gemm(split3(ao), split_weight(a.proj.weight), kind=EPI_F32, bias=a.proj.bias)
        if ens[0] > 0:   # the ensemble merges on the full token grid, after window_unpartition (models_seggpt.py:214-231)
            x1 = ops.ensemble_resid(ops.window_unpartition(pa, Bp, h, w, ws), z, ens[0], ens[1], N, C)
        else:
            x1 = ops.window_unpartition(pa, Bp, h, w, ws, resid=z)
    else:
        ao = attention(u, blk, Bp, h, w, heads, ws_cache, rel_h, rel_w)
        if ens[0] > 0:
            pa = _gemm(split3(ao), split_weight(a.proj.weight), kind=EPI_F32, bias=a.proj.bias)
            x1 = ops.ensemble_resid(pa, z, ens[0], ens[1], N, C)
        else:
            x1 = _gemm(split3(ao), split_weight(a.proj.weight), kind=EPI_RESID, bias=a.proj.bias, aux=z)
    v, _, _ = ops.layernorm_fwd(x1, blk.norm2.weight, blk.norm2.bias, eps, out_dtype=torch.float32, want_stats=False)
    hid = _gemm(split3(v), split_weight(blk.mlp.fc1.weight), kind=EPI_F32, bias=blk.mlp.fc1.bias)
    return _gemm(split3(hid, gelu=True), split_weight(blk.mlp.fc2.weight), kind=EPI_RESID, bias=blk.mlp.fc2.bias, aux=x1)


@torch.no_grad()
def forward(model, imgs, tgts, mask_u8, valid, type_emb, merge_between_batch, prompts_per_query=None):
    """(loss [()], patchify(pred) [B, N, p*p*3]) - Painter._run in fp32-accurate arithmetic."""
    from . import engine
    p = model.patch_size
    B, Cin, H, W = imgs.shape
    h, w = H // p, W // p
    N, C = h * w, model.embed_dim
    dev = imgs.device
    L = lib()
    # ---- embed (vitdet_utils.py:178-186, models_painter.py:392-409)
    pe = model.patch_embed.proj
    cols = torch.empty((2 * B * N, 6 * Cin * p * p), dtype=torch.bfloat16, device=dev)
    check(L.pk_im2col_patch_split3(_ptr(imgs), _ptr(tgts), _ptr(cols), B, Cin, H, W, p, _stream()),
          "pk_im2col_patch_split3")
    E = _gemm(cols, split_weight(pe.weight, (C, Cin * p * p)), kind=EPI_F32, bias=pe.bias)
    pos = model.pos_embed[0, 1:] if model.pretrain_use_cls_token else model.pos_embed[0]
    s = int(round(pos.shape[0] ** 0.5))
    pos = pos.detach().contiguous()
    if not (s == h and s == w):
        pos = ops.bicubic_fwd(pos.view(s, s, C), h, w).view(N, C)
    z = ops.assemble_tokens(E, mask_u8, model.mask_token.detach().reshape(C).contiguous(),
                            model.segment_token_x.detach().reshape(C).contiguous(),
                            model.segment_token_y.detach().reshape(C).contiguous(), pos, type_emb, B, N, C)
    # ---- blocks
    ws_cache = {}
    Bp, merge_idx, taps = 2 * B, 2, []
    for i, blk in enumerate(model.blocks):
        ens = model._ensemble(i, B, merge_between_batch, prompts_per_query, merge_idx)
        ws = blk.window_size
        rel_h = engine.resize_rel_table(blk.attn.rel_pos_h, ws if ws > 0 else h)
        rel_w = engine.resize_rel_table(blk.attn.rel_pos_w, ws if ws > 0 else w)
        z = block(z, blk, Bp, h, w, model.num_heads, blk.norm1.eps, ens, ws_cache, rel_h, rel_w)
        if i == merge_idx:
            z = ops.merge_halves(z)
            Bp = B
            ws_cache.clear()
        if i in (5, 11, 17, 23):
            taps.append(z)
    del ws_cache
    # ---- decoder (models_painter.py:417-431) + loss (:433-462)
    M = B * N
    cat = torch.empty((M, 4 * C), dtype=torch.float32, device=dev)
    for k, t in enumerate(taps):
        ops.layernorm_fwd(t, model.norm.weight, model.norm.bias, model.norm.eps, out=cat[:, k * C:(k + 1) * C],
                          want_stats=False)
    D = _gemm(split3(cat), split_weight(model.decoder_embed.weight), kind=EPI_F32, bias=model.decoder_embed.bias)
    dp = model.decoder_pred
    dd = model.decoder_embed_dim
    if dd != 64:
        raise NotImplementedError("painter_b200: decoder_embed_dim must be 64 (the stock configuration)")
    Hh, Ww = h * p, w * p
    c1 = torch.empty((B * Hh * Ww, 64), dtype=torch.float32, device=dev)
    wconv = split_weight(dp[0].weight, None) if False else _conv_weight(dp[0].weight)
    # the im2col operand is 6 * 576 bf16 per pixel (2.8 GB per 896x448 image): one image at a time
    for b in range(B):
        icol = torch.empty((Hh * Ww, 6 * 9 * dd), dtype=torch.bfloat16, device=dev)
        check(L.pk_dec_im2col_split3(_ptr(D[b * N:(b + 1) * N]), _ptr(icol), 1, h, w, p, dd, _stream()),
              "pk_dec_im2col_split3")
        _gemm(icol, wconv, kind=EPI_F32, bias=dp[0].bias, out=c1[b * Hh * Ww:(b + 1) * Hh * Ww])
        del icol
    hp = ops.pack_head_params(dp[0].bias, dp[1].weight, dp[1].bias, dp[3].weight, dp[3].bias)
    st = ops.loss_prep(tgts, mask_u8, valid, p)
    patch = torch.empty((B, N, p * p * 3), dtype=torch.float32, device=dev)
    numd = torch.zeros((B,), dtype=torch.float64, device=dev)
    num = torch.empty((B,), dtype=torch.float32, device=dev)
    check(L.pk_head_f32(_ptr(c1), _ptr(hp), _ptr(tgts), _ptr(mask_u8), mask_u8.shape[0], _ptr(valid), _ptr(patch),
                        _ptr(numd), _ptr(num), B, Hh, Ww, p, engine.LOSS_KINDS[model.loss_func], _stream()),
          "pk_head_f32")
    loss, _ = ops.loss_finalize(st, num, model.seggpt)
    return loss.reshape(()), patch


def _conv_weight(w):
    """conv3x3 weight [o, c, ky, kx] -> B-side split of the im2col matrix [o, (ky*3 + kx)*64 + c]; cached."""
    ent = getattr(w, "_pk_split3", None)
    if ent is not None and ent[0] == w._version and ent[1] == w.data_ptr() and ent[2].device == w.device:
        return ent[2]
    m = w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()
    s = split3(m, side_b=True)
    w._pk_split3 = (w._version, w.data_ptr(), s, 0)
    return s
