"""Host-side orchestration of the hot path: one torch.autograd.Function per stage (embed, block, merge,
decoder+loss) so that autograd / DDP hooks fire block by block.  Every arithmetic step is a call into
libpainter_b200.so (painter_b200/ops.py); torch is used for memory, streams and the autograd tape only.

Stage map (reference file:line -> Function):
  EmbedFn     Painter/models_painter.py:385-409 (PatchEmbed x2, mask-token blend, segment/pos/type tokens)
  BlockFn     Painter/models_painter.py:216-235 + Attention :73-89 (+ SegGPT ensemble models_seggpt.py:220-231)
  MergeFn     Painter/models_painter.py:414-415
  DecoderFn   Painter/models_painter.py:417 (final LN taps), :420-431 (decoder), :433-462 (loss), :355-368 (patchify)
"""
import torch
import torch.nn.functional as F

from . import ops
from .ops import EPI_BF16, EPI_DGELU, EPI_F32, EPI_GELU, EPI_PIXSHUF, EPI_RESID

LOSS_KINDS = {"smoothl1": 0, "l1": 1, "l2": 2, "l1l2": 3}


class StageEnv:
    """Per-forward bookkeeping handed to every stage (non-tensor argument): the module's gradient arena, a token that
    identifies the step, the stage's arena group name and its parameters by role, and - for a block - the hand-off to
    the block below it in the stack (whose MLP branch consumes this block's dx)."""
    __slots__ = ("arena", "token", "name", "prm", "below")

    def __init__(self, arena, token, name, prm, below=None):
        self.arena, self.token, self.name, self.prm, self.below = arena, token, name, prm, below

    def begin(self):
        """True if this backward writes parameter gradients into the arena."""
        return self.arena is not None and self.arena.begin_backward(self.token)

    def grad(self, active, role, fallback_shape=None, device=None):
        """Zero-initialised fp32 accumulator for the gradient of parameter `role`: its arena slot, or a fresh buffer."""
        p = self.prm[role]
        if active:
            return self.arena.view(p)
        return torch.zeros(p.shape if fallback_shape is None else fallback_shape, dtype=torch.float32,
                           device=p.device if device is None else device)


def bf16_weight(p, shape2d=None):
    """bf16 copy of an fp32 parameter, cached ON the parameter object and keyed by (version, storage): the cast is
    redone only after an optimizer step / load_state_dict changed the values."""
    ent = getattr(p, "_pk_bf16", None)
    ver = p._version
    if ent is not None and ent[0] == ver and ent[1] == p.data_ptr() and ent[2].device == p.device:
        return ent[2]
    src = p.detach()
    if not src.is_contiguous():
        src = src.contiguous()
    w = ops.cast_bf16(src)
    if shape2d is not None:
        w = w.view(shape2d)
    p._pk_bf16 = (ver, p.data_ptr(), w)
    return w


def bf16_table(t):
    """Zero-padded bf16 copy [pad16(L), 64] of a rel-pos table (the attention kernels' operand).  For a parameter the
    copy is cached like bf16_weight (and refreshed by optim.FusedAdamW itself); a resized (non-leaf) table is cast
    on every call."""
    if not isinstance(t, torch.nn.Parameter):
        return ops.relpos_table_bf16(t.contiguous())
    ent = getattr(t, "_pk_bf16", None)
    if ent is not None and ent[0] == t._version and ent[1] == t.data_ptr() and ent[2].device == t.device:
        return ent[2]
    w = ops.relpos_table_bf16(t.detach().contiguous())
    t._pk_bf16 = (t._version, t.data_ptr(), w)
    return w


def invalidate_weight_cache(module):
    """Drop every cached bf16 operand copy (call after writing parameters through `.data`, which autograd's version
    counter does not see)."""
    for p in module.parameters():
        if hasattr(p, "_pk_bf16"):
            del p._pk_bf16


def _wgrad(dy_bf16, x_bf16, out=None):
    """dW[out, in] = dY^T . X  (both operands read MN-major; stream-K over the zero-initialised fp32 output)."""
    if out is None:
        out = torch.zeros((dy_bf16.shape[1], x_bf16.shape[1]), dtype=torch.float32, device=dy_bf16.device)
    return ops.gemm(dy_bf16, x_bf16, trans_a=True, trans_b=True, kind=EPI_F32, out=out, accumulate=2)


def th_rows(size):
    """Rows of a decomposed rel-pos table for a grid side `size` (vitdet_utils.get_rel_pos: 2 * size - 1)."""
    return 2 * size - 1


def resize_rel_table(table, size):
    """vitdet_utils.get_rel_pos (:75-86): linear resize of the table when its length != 2*size-1.
    Tiny host-side parameter preprocessing; autograd carries the transpose for the backward."""
    L = 2 * size - 1
    if table.shape[0] == L:
        return table
    return F.interpolate(table.t().unsqueeze(0), size=L, mode="linear")[0].t().contiguous()


class EmbedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, imgs, tgts, mask_u8, type_emb, Wp, bp, mask_token, seg_x, seg_y, pos_embed, p, has_cls, env):
        B, Cin, H, W = imgs.shape
        h, w = H // p, W // p
        N, C = h * w, Wp.shape[0]
        cols = ops.im2col_patch(imgs, tgts, p)
        E = ops.gemm(cols, bf16_weight(Wp, (C, Cin * p * p)), kind=EPI_F32, bias=bp)
        pe = pos_embed[0, 1:] if has_cls else pos_embed[0]
        s = int(round(pe.shape[0] ** 0.5))
        assert s * s == pe.shape[0]
        pe = pe.contiguous()
        pos = pe if (s == h and s == w) else ops.bicubic_fwd(pe.view(s, s, C), h, w).view(N, C)
        z = ops.assemble_tokens(E, mask_u8, mask_token.reshape(C).contiguous(), seg_x.reshape(C).contiguous(),
                                seg_y.reshape(C).contiguous(), pos, type_emb, B, N, C)
        ctx.save_for_backward(cols, mask_u8)
        ctx.meta = (B, N, C, h, w, s, has_cls, Wp.shape, pos_embed.shape, mask_token.shape, type_emb is not None)
        ctx.env = env
        return z

    @staticmethod
    def backward(ctx, dz):
        cols, mask_u8 = ctx.saved_tensors
        B, N, C, h, w, s, has_cls, wshape, pshape, tshape, has_type = ctx.meta
        if has_type and ctx.needs_input_grad[3]:
            raise NotImplementedError("painter_b200: gradients of the SegGPT type tokens are not implemented "
                                      "(SegGPT is an inference path, seggpt_engine.py:26)")
        env = ctx.env
        act = env is not None and env.begin()
        dz = dz.contiguous()
        if act:
            g = {k: env.grad(True, k) for k in ("w", "b", "mt", "sx", "sy", "pe")}
            tok = (g["sx"].view(C), g["sy"].view(C), g["mt"].view(C))
        else:
            g, tok = None, None
        dE, dpos, dsx, dsy, dmt = ops.assemble_tokens_bwd(dz, mask_u8, B, N, C, token_grads=tok)
        dW = _wgrad(dE, cols, out=g["w"].view(wshape[0], -1) if act else None).view(wshape)
        db = ops.colsum_bf16(dE, out=g["b"] if act else None)
        dpe = g["pe"] if act else torch.zeros(pshape, dtype=torch.float32, device=dz.device)
        off = 1 if has_cls else 0
        if s == h and s == w:
            dpe[0, off:] = dpos
        else:
            ops.bicubic_bwd(dpos.view(h, w, C), s, s, out=dpe[0, off:].view(s, s, C))
        if act:
            env.arena.stage_done(env.name)
            env.arena.end_backward()
            return (None, None, None, None, dW, db, g["mt"], g["sx"], g["sy"], dpe, None, None, None)
        return (None, None, None, None, dW, db, dmt.view(tshape), dsx.view(tshape), dsy.view(tshape), dpe, None,
                None, None)


class BlockFn(torch.autograd.Function):
    """x [B'*N, C] fp32 -> same.  meta = (Bp, h, w, heads, eps, ens_groups, ens_P, ws); ws > 0 = windowed block
    (vitdet_utils.window_partition / window_unpartition around the attention, models_painter.py:220-227)."""

    @staticmethod
    def forward(ctx, x, drop_a, drop_m, n1w, n1b, rel_h, rel_w, qkv_w, qkv_b, proj_w, proj_b, n2w, n2b, fc1_w,
                fc1_b, fc2_w, fc2_b, meta, env=None):
        Bp, h, w, heads, eps, ens_groups, ens_P, ws = meta
        ctx.env = env
        N = h * w
        M, C = x.shape
        u, mean1, rstd1 = ops.layernorm_fwd(x, n1w, n1b, eps)
        wqkv, wproj = bf16_weight(qkv_w), bf16_weight(proj_w)
        wfc1, wfc2 = bf16_weight(fc1_w), bf16_weight(fc2_w)
        th, tw = bf16_table(rel_h), bf16_table(rel_w)
        # ops.attn_fwd(save_rel=True) / attn_bwd(rel=...) can keep every query's bias rows for the backward (the dQ
        # kernel then loads them instead of recomputing them).  That costs 72 MB of extra saved activations per block
        # application at batch 8 and saves one small kernel, so the module does not use it.
        save_rel = False
        relh = relw = x.new_empty(0)
        if ws > 0:
            u = ops.window_partition_bf16(u, Bp, h, w, ws)   # zero-padded windows [Bp*nW*ws*ws, C]
            Bw = u.shape[0] // (ws * ws)
            qkv = ops.gemm(u, wqkv, kind=EPI_BF16, bias=qkv_b)
            if save_rel:
                ao, lse, (relh, relw) = ops.attn_fwd(qkv, th, tw, Bw, heads, ws, ws, save_rel=True)
            else:
                ao, lse = ops.attn_fwd(qkv, th, tw, Bw, heads, ws, ws)
            a = ops.gemm(ao, wproj, kind=EPI_F32, bias=proj_b)
            if ens_groups > 0:   # the ensemble merges on the full token grid, after window_unpartition
                x1 = ops.ensemble_resid(ops.window_unpartition(a, Bp, h, w, ws), x, ens_groups, ens_P, N, C)
            else:
                x1 = ops.window_unpartition(a, Bp, h, w, ws, resid=x, rowscale=drop_a)
        else:
            qkv = ops.gemm(u, wqkv, kind=EPI_BF16, bias=qkv_b)
            if save_rel:
                ao, lse, (relh, relw) = ops.attn_fwd(qkv, th, tw, Bp, heads, h, w, save_rel=True)
            else:
                ao, lse = ops.attn_fwd(qkv, th, tw, Bp, heads, h, w)
        if ws > 0:
            pass
        elif ens_groups > 0:
            a = ops.gemm(ao, wproj, kind=EPI_F32, bias=proj_b)
            x1 = ops.ensemble_resid(a, x, ens_groups, ens_P, N, C)
        else:
            x1 = ops.gemm(ao, wproj, kind=EPI_RESID, bias=proj_b, aux=x, rowscale=drop_a, rows_per_group=N)
        v, mean2, rstd2 = ops.layernorm_fwd(x1, n2w, n2b, eps)
        z, hact = ops.gemm(v, wfc1, kind=EPI_GELU, bias=fc1_b)
        x2 = ops.gemm(hact, wfc2, kind=EPI_RESID, bias=fc2_b, aux=x1, rowscale=drop_m, rows_per_group=N)
        ctx.save_for_backward(x, mean1, rstd1, u, qkv, ao, lse, th, tw, x1, mean2, rstd2, v, z, hact, wqkv, wproj,
                              wfc1, wfc2, n1w, n2w, drop_a, drop_m, relh, relw)
        ctx.meta = meta
        return x2

    @staticmethod
    def backward(ctx, dx2):
        (x, mean1, rstd1, u, qkv, ao, lse, th, tw, x1, mean2, rstd2, v, z, hact, wqkv, wproj, wfc1, wfc2, n1w, n2w,
         drop_a, drop_m, relh, relw) = ctx.saved_tensors
        rel = (relh, relw) if relh.numel() > 0 else None
        Bp, h, w, heads, eps, ens_groups, ens_P, ws = ctx.meta
        if ens_groups > 0:
            raise NotImplementedError("painter_b200: backward through the SegGPT prompt ensemble is not implemented")
        N = h * w
        M, C = x.shape
        dev = x.device
        dx2 = dx2.contiguous()
        H4 = wfc1.shape[0]
        # Accumulation targets of the block (LN affine grads, bias grads, the four weight gradients the stream-K
        # GEMMs add into, the rel-pos table gradients): the parameters' slots in the module's zero-initialised
        # gradient arena, or - gradient accumulation / no arena - ONE zero-filled slab for the block.
        env = ctx.env
        act = env is not None and env.begin()
        Lh, Lw = th_rows(h if ws == 0 else ws), th_rows(w if ws == 0 else ws)
        rel_native = act and env.prm["rel_h"].shape[0] == Lh and env.prm["rel_w"].shape[0] == Lw
        if act:
            gv = env.arena.view
            P = env.prm
            dn1w, dn1b, dn2w, dn2b = gv(P["n1w"]), gv(P["n1b"]), gv(P["n2w"]), gv(P["n2b"])
            dfc2_b, dproj_b, dfc1_b, dqkv_b = gv(P["fc2_b"]), gv(P["proj_b"]), gv(P["fc1_b"]), gv(P["qkv_b"])
            g_qkv, g_proj, g_fc1, g_fc2 = gv(P["qkv_w"]), gv(P["proj_w"]), gv(P["fc1_w"]), gv(P["fc2_w"])
            if rel_native:
                g_th, g_tw = gv(P["rel_h"]), gv(P["rel_w"])
            else:   # resized tables: the gradient flows on through autograd's transpose of the linear resize
                g_th = torch.zeros((Lh, 64), dtype=torch.float32, device=dev)
                g_tw = torch.zeros((Lw, 64), dtype=torch.float32, device=dev)
        else:
            n_small = 4 * C + 2 * C + H4 + 3 * C
            sizes = [n_small, 3 * C * C, C * C, H4 * C, C * H4, Lh * 64, Lw * 64]
            slab = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
            small, g_qkv, g_proj, g_fc1, g_fc2, g_th, g_tw = torch.split(slab, sizes)
            g_qkv, g_proj = g_qkv.view(3 * C, C), g_proj.view(C, C)
            g_fc1, g_fc2 = g_fc1.view(H4, C), g_fc2.view(C, H4)
            g_th, g_tw = g_th.view(Lh, 64), g_tw.view(Lw, 64)
            dn1w, dn1b, dn2w, dn2b = small[0:C], small[C:2 * C], small[2 * C:3 * C], small[3 * C:4 * C]
            dfc2_b, dproj_b = small[4 * C:5 * C], small[5 * C:6 * C]
            dfc1_b, dqkv_b = small[6 * C:6 * C + H4], small[6 * C + H4:]
        # ---- MLP branch ----
        # bf16(DropPath scale * dx2) and its column sums (fc2 bias gradient) normally arrive from the LN1 backward of
        # the block above, which produced dx2 (hand-off through the arena); otherwise one pass over dx2 here
        ho = env.arena.handoff if act else None
        if ho is not None:
            env.arena.handoff = None
            if ho[0].data_ptr() != dx2.data_ptr() or ho[0].shape != dx2.shape:
                raise RuntimeError("painter_b200: gradient hand-off between blocks does not match the incoming grad")
            dy = ho[1]
        else:
            dy, _ = ops.scale_cast_colsum(dx2, drop_m, N, colsum_out=dfc2_b)
        dfc2_w = _wgrad(dy, hact, out=g_fc2)
        dz = ops.gemm(dy, wfc2, trans_b=True, kind=EPI_DGELU, aux=z)
        ops.colsum_bf16(dz, out=dfc1_b)
        dfc1_w = _wgrad(dz, v, out=g_fc1)
        # dgrad outputs that feed a LayerNorm backward are written as bf16 (the reference's autocast Linear backward
        # rounds there too): half the store traffic of the GEMM epilogue and of the LN-backward's dy stream
        dv = ops.gemm(dz, wfc1, trans_b=True, kind=EPI_BF16)
        # LN2 backward also emits the attention branch's incoming gradient: bf16(DropPath scale * dx1) + its column sums
        dx1, da = ops.layernorm_bwd(dv, x1, mean2, rstd2, n2w, dn2w, dn2b, dres=dx2, cast=(drop_a, N, dproj_b))
        # ---- attention branch ----
        if ws > 0:
            da = ops.window_partition_bf16(da, Bp, h, w, ws)
            Bw = da.shape[0] // (ws * ws)
        dproj_w = _wgrad(da, ao, out=g_proj)
        dao = ops.gemm(da, wproj, trans_b=True, kind=EPI_BF16)
        if ws > 0:
            dqkv, dTh, dTw = ops.attn_bwd(qkv, ao, dao, lse, th, tw, Bw, heads, ws, ws, dT_out=(g_th, g_tw), rel=rel)
        else:
            dqkv, dTh, dTw = ops.attn_bwd(qkv, ao, dao, lse, th, tw, Bp, heads, h, w, dT_out=(g_th, g_tw), rel=rel)
        ops.colsum_bf16(dqkv, out=dqkv_b)
        dqkv_w = _wgrad(dqkv, u, out=g_qkv)
        if ws > 0:
            du = ops.gemm(dqkv, wqkv, trans_b=True, kind=EPI_F32)
            du = ops.window_unpartition(du, Bp, h, w, ws)   # gradients at padded tokens are dropped
        else:
            du = ops.gemm(dqkv, wqkv, trans_b=True, kind=EPI_BF16)
        below = env.below if act else None
        if below is not None:
            # the block below consumes dx only through bf16(its DropPath scale * dx): emit that (and the fc2 bias
            # gradient it implies) in the same pass
            b_fc2_b, b_drop_m, b_N = below
            dx, dxb = ops.layernorm_bwd(du, x, mean1, rstd1, n1w, dn1w, dn1b, dres=dx1,
                                        cast=(b_drop_m, b_N, env.arena.view(b_fc2_b)))
            env.arena.handoff = (dx, dxb)
        else:
            dx = ops.layernorm_bwd(du, x, mean1, rstd1, n1w, dn1w, dn1b, dres=dx1)
        if act:
            env.arena.stage_done(env.name)
        return (dx, None, None, dn1w, dn1b, dTh, dTw, dqkv_w, dqkv_b, dproj_w, dproj_b, dn2w, dn2b, dfc1_w, dfc1_b,
                dfc2_w, dfc2_b, None, None)


class MergeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        return ops.merge_halves(z)

    @staticmethod
    def backward(ctx, d):
        return ops.merge_halves_bwd(d.contiguous())


class DecoderFn(torch.autograd.Function):
    """(4 tap activations) -> (loss[1], patchified prediction [B, N, p*p*3])."""

    @staticmethod
    def forward(ctx, t0, t1, t2, t3, norm_w, norm_b, dec_w, dec_b, c3_w, c3_b, ln_w, ln_b, c1_w, c1_b, tgts, mask_u8,
                valid, meta, env=None):
        B, h, w, p, eps, loss_kind, seggpt = meta
        ctx.env = env
        M, C = t0.shape
        dev = t0.device
        dd = ln_w.shape[0]
        if dd != 64:
            raise NotImplementedError("painter_b200: decoder_embed_dim must be 64 (the stock configuration)")
        taps = (t0, t1, t2, t3)
        cat = torch.empty((M, 4 * C), dtype=torch.bfloat16, device=dev)
        stats = []
        for k, t in enumerate(taps):
            _, mean, rstd = ops.layernorm_fwd(t, norm_w, norm_b, eps, out=cat[:, k * C:(k + 1) * C])
            stats.append((mean, rstd))
        wdec = bf16_weight(dec_w)
        g = torch.empty((B, h * p, w * p, dd), dtype=torch.bfloat16, device=dev)
        ops.gemm(cat, wdec, kind=EPI_PIXSHUF, bias=dec_b, pixshuf=(h, w, p, dd, g))
        wf, wd = ops.conv3x3_pack(c3_w.contiguous())
        hp = torch.cat([c3_b, ln_w, ln_b, c1_w.reshape(-1), c1_b, c1_b.new_zeros(5)]).contiguous()
        st = ops.loss_prep(tgts, mask_u8, valid, p)
        c1, patch, num = ops.decoder_head_fwd(g, wf, hp, tgts, mask_u8, valid, p, loss_kind)
        loss, coef = ops.loss_finalize(st, num, seggpt)
        ctx.save_for_backward(t0, t1, t2, t3, norm_w, cat, wdec, g, wd, hp, c1, tgts, mask_u8, valid, coef,
                              *[s for pair in stats for s in pair])
        ctx.meta = meta
        ctx.shapes = (c3_w.shape, c1_w.shape)
        ctx.mark_non_differentiable(patch)
        return loss, patch

    @staticmethod
    def backward(ctx, dloss, _dpatch):
        sv = ctx.saved_tensors
        t = sv[0:4]
        norm_w, cat, wdec, g, wd, hp, c1, tgts, mask_u8, valid, coef = sv[4:15]
        stats = sv[15:]
        B, h, w, p, eps, loss_kind, seggpt = ctx.meta
        M, C = t[0].shape
        dev = c1.device
        env = ctx.env
        act = env is not None and env.begin()
        G = (lambda k: env.grad(True, k)) if act else (lambda k: None)
        gscale = dloss.reshape(1).to(torch.float32).contiguous()
        dc1, dhp = ops.decoder_head_bwd(c1, tgts, mask_u8, valid, coef, gscale, hp, p, loss_kind)
        dc3_b = ops.colsum_bf16(dc1.view(-1, 64), out=G("c3_b"))
        dc3_w = ops.conv3x3_wgrad(g, dc1, out=G("c3_w"))
        dD = ops.conv3x3_dgrad_unshuffle(dc1, wd, p)          # [M, p*p*64] bf16, token-major
        ddec_b = ops.colsum_bf16(dD, out=G("dec_b"))
        ddec_w = _wgrad(dD, cat, out=G("dec_w"))
        dcat = ops.gemm(dD, wdec, trans_b=True, kind=EPI_BF16)  # [M, 4C] bf16, read by the 4 LayerNorm backwards
        dnw = G("norm_w") if act else torch.zeros(C, dtype=torch.float32, device=dev)
        dnb = G("norm_b") if act else torch.zeros(C, dtype=torch.float32, device=dev)
        dts = []
        for k in range(4):
            dts.append(ops.layernorm_bwd(dcat[:, k * C:(k + 1) * C], t[k], stats[2 * k], stats[2 * k + 1], norm_w,
                                         dnw, dnb))
        c3shape, c1shape = ctx.shapes
        if act:
            dlw, dlb, dc1w, dc1b = G("ln_w"), G("ln_b"), G("c1_w"), G("c1_b")
            dlw.copy_(dhp[64:128])
            dlb.copy_(dhp[128:192])
            dc1w.view(-1).copy_(dhp[192:384])
            dc1b.copy_(dhp[384:387])
            env.arena.stage_done(env.name)
        else:
            dlw, dlb = dhp[64:128].clone(), dhp[128:192].clone()
            dc1w, dc1b = dhp[192:384].reshape(c1shape).clone(), dhp[384:387].clone()
        return (dts[0], dts[1], dts[2], dts[3], dnw, dnb, ddec_w, ddec_b, dc3_w, dc3_b, dlw, dlb, dc1w, dc1b, None,
                None, None, None, None)
