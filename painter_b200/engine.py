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


class StepLink:
    """State the block backwards of one forward share: the hand-off (dx fp32, bf16(scale * dx)) that block i+1's LN1
    backward passes to block i's MLP branch."""
    __slots__ = ("handoff",)

    def __init__(self):
        self.handoff = None


class StageEnv:
    """Per-forward bookkeeping handed to every stage (non-tensor argument): the module's gradient arena (None: no
    parameter requires grad), a token that identifies the step, the stage's arena group name and its parameters by
    role, and - for a block - the block below it in the stack (whose MLP branch consumes this block's dx) and the
    forward's StepLink that carries the hand-off."""
    __slots__ = ("arena", "token", "name", "prm", "below", "link")

    def __init__(self, arena, token, name, prm, below=None, link=None):
        self.arena, self.token, self.name, self.prm, self.below, self.link = arena, token, name, prm, below, link

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


def type_embedding(seg_type, type_cls, type_ins):
    """SegGPT's per-sample type embedding [B, C] fp32 (models_seggpt.py:415-417): type_token_cls where seg_type is 0,
    type_token_ins where it is 1, zero otherwise.  Mask arithmetic instead of boolean indexing: no host
    synchronisation, so the step stays CUDA-graph capturable.  seg_type: fp32 [B, 1] on the device."""
    C = type_cls.shape[-1]
    return ((seg_type == 0).to(torch.float32) * type_cls.reshape(1, C).float() +
            (seg_type == 1).to(torch.float32) * type_ins.reshape(1, C).float()).contiguous()


class EmbedFn(torch.autograd.Function):
    """imgs, tgts fp32 NCHW -> tokens [2B*N, C].  Gradients flow to imgs / tgts (prompt tuning, saliency) through the
    patch-embed dgrad and pk_col2im_patch; every parameter gradient is computed only if that parameter requires grad
    (the weight gradient's operand `cols` is not even saved when the weight is frozen).  SegGPT passes seg_type (fp32
    [B, 1] on the device) and its two type tokens; Painter passes None for all three."""

    @staticmethod
    def forward(ctx, imgs, tgts, mask_u8, seg_type, Wp, bp, mask_token, seg_x, seg_y, pos_embed, type_cls, type_ins,
                p, has_cls, env):
        B, Cin, H, W = imgs.shape
        h, w = H // p, W // p
        N, C = h * w, Wp.shape[0]
        cols = ops.im2col_patch(imgs, tgts, p)
        wp = bf16_weight(Wp, (C, Cin * p * p))
        E = ops.gemm(cols, wp, kind=EPI_F32, bias=bp)
        pe = pos_embed[0, 1:] if has_cls else pos_embed[0]
        s = int(round(pe.shape[0] ** 0.5))
        assert s * s == pe.shape[0]
        pe = pe.contiguous()
        pos = pe if (s == h and s == w) else ops.bicubic_fwd(pe.view(s, s, C), h, w).view(N, C)
        type_emb = None if seg_type is None else type_embedding(seg_type, type_cls, type_ins)
        z = ops.assemble_tokens(E, mask_u8, mask_token.reshape(C).contiguous(), seg_x.reshape(C).contiguous(),
                                seg_y.reshape(C).contiguous(), pos, type_emb, B, N, C)
        need = ctx.needs_input_grad
        need_type = seg_type is not None and (need[10] or need[11])
        ctx.save_for_backward(cols if need[4] else None, mask_u8, wp if (need[0] or need[1]) else None,
                              seg_type.reshape(B).contiguous() if need_type else None)
        ctx.meta = (B, N, C, h, w, s, has_cls, Wp.shape, pos_embed.shape, mask_token.shape, need_type,
                    (Cin, H, W, p))
        ctx.env = env
        return z

    @staticmethod
    def backward(ctx, dz):
        cols, mask_u8, wp, seg_type = ctx.saved_tensors
        B, N, C, h, w, s, has_cls, wshape, pshape, tshape, need_type, (Cin, H, W, p) = ctx.meta
        need = ctx.needs_input_grad
        env = ctx.env
        act = env is not None and env.begin()
        dz = dz.contiguous()
        need_tok = need[6] or need[7] or need[8]
        tok = tuple(env.grad(True, k).view(C) for k in ("sx", "sy", "mt")) if act and need_tok else None
        typ = None
        if need_type:   # both type tokens are reduced in one pass, even when only one of them requires grad
            dtt = tuple(env.grad(True, k).view(C) for k in ("tc", "ti")) if act else \
                torch.zeros((2, C), dtype=torch.float32, device=dz.device).unbind(0)
            typ = (seg_type, *dtt)
        dE, dpos, dsx, dsy, dmt = ops.assemble_tokens_bwd(dz, mask_u8, B, N, C, token_grads=tok, want_tokens=need_tok,
                                                          want_pos=need[9], type_grads=typ)
        dW = _wgrad(dE, cols, out=env.grad(True, "w").view(wshape[0], -1) if act else None).view(wshape) \
            if need[4] else None
        db = ops.colsum_bf16(dE, out=env.grad(True, "b") if act else None) if need[5] else None
        dpe = None
        if need[9]:
            dpe = env.grad(True, "pe") if act else torch.zeros(pshape, dtype=torch.float32, device=dz.device)
            off = 1 if has_cls else 0
            if s == h and s == w:
                dpe[0, off:] = dpos
            else:
                ops.bicubic_bwd(dpos.view(h, w, C), s, s, out=dpe[0, off:].view(s, s, C))
        dimgs = dtgts = None
        if need[0] or need[1]:
            # patch-embed dgrad dE . Wp of the wanted halves only (x rows -> imgs, y rows -> tgts), one GEMM over the
            # rows of both when both are wanted, then the inverse of the im2col layout
            lo, hi = (0 if need[0] else B * N), (2 * B * N if need[1] else B * N)
            dcols = ops.gemm(dE[lo:hi], wp, trans_b=True, kind=EPI_F32)
            dimgs, dtgts = ops.col2im_patch(dcols[:B * N] if need[0] else None,
                                            dcols[hi - lo - B * N:] if need[1] else None, B, Cin, H, W, p)
        if act:
            env.arena.stage_done(env.name)
            env.arena.end_backward()
            return (dimgs, dtgts, None, None, dW, db, env.grad(True, "mt") if need[6] else None,
                    env.grad(True, "sx") if need[7] else None, env.grad(True, "sy") if need[8] else None, dpe,
                    env.grad(True, "tc") if need[10] else None, env.grad(True, "ti") if need[11] else None, None,
                    None, None)
        return (dimgs, dtgts, None, None, dW, db, dmt.view(tshape) if need[6] else None,
                dsx.view(tshape) if need[7] else None, dsy.view(tshape) if need[8] else None, dpe,
                typ[1].view(tshape) if need[10] else None, typ[2].view(tshape) if need[11] else None, None, None, None)


# BlockFn's parameter inputs (positions 3 .. 16 of its forward) in the order of models_painter.Block.ROLES
BLOCK_ROLES = ("n1w", "n1b", "rel_h", "rel_w", "qkv_w", "qkv_b", "proj_w", "proj_b", "n2w", "n2b", "fc1_w", "fc1_b",
               "fc2_w", "fc2_b")


class BlockFn(torch.autograd.Function):
    """x [B'*N, C] fp32 -> same.  meta = (Bp, h, w, heads, eps, ens_groups, ens_P, ws); ws > 0 = windowed block
    (vitdet_utils.window_partition / window_unpartition around the attention, models_painter.py:220-227).
    Every parameter gradient (weight-gradient GEMM, bias column sums, LayerNorm affine reductions, rel-pos table
    gradients) is computed only if that parameter requires grad, and the activations only the weight gradients read
    (u, v, hact) are saved only if qkv / fc1 / fc2 weight requires grad; the dx chain is the same either way."""

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
        need = ctx.needs_input_grad
        ctx.save_for_backward(x, mean1, rstd1, u if need[7] else None, qkv, ao, lse, th, tw, x1, mean2, rstd2,
                              v if need[13] else None, z, hact if need[15] else None, wqkv, wproj, wfc1, wfc2, n1w,
                              n2w, drop_a, drop_m, relh, relw)
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
        need = dict(zip(BLOCK_ROLES, ctx.needs_input_grad[3:17]))
        tables = need["rel_h"] or need["rel_w"]
        # Accumulation targets of the parameters that require grad (LN affine grads, bias grads, the four weight
        # gradients the stream-K GEMMs add into, the rel-pos table gradients): their slots in the module's
        # zero-initialised gradient arena, or - gradient accumulation / no arena - ONE zero-filled slab for the block.
        # None for a frozen parameter: its reduction is skipped.
        env = ctx.env
        act = env is not None and env.begin()
        Lh, Lw = th_rows(h if ws == 0 else ws), th_rows(w if ws == 0 else ws)
        shapes = {"n1w": (C,), "n1b": (C,), "rel_h": (Lh, 64), "rel_w": (Lw, 64), "qkv_w": (3 * C, C),
                  "qkv_b": (3 * C,), "proj_w": (C, C), "proj_b": (C,), "n2w": (C,), "n2b": (C,), "fc1_w": (H4, C),
                  "fc1_b": (H4,), "fc2_w": (C, H4), "fc2_b": (C,)}
        if tables:      # the attention kernel produces both table gradients together
            need_t = dict(need, rel_h=True, rel_w=True)
        else:
            need_t = need
        g = dict.fromkeys(BLOCK_ROLES)
        rel_native = act and env.prm["rel_h"].shape[0] == Lh and env.prm["rel_w"].shape[0] == Lw
        if act:
            # resized tables get slab buffers: their gradient flows on through autograd's transpose of the resize
            for r in BLOCK_ROLES:
                if need_t[r] and (rel_native or r not in ("rel_h", "rel_w")):
                    g[r] = env.arena.view(env.prm[r])
        pending = [r for r in BLOCK_ROLES if need_t[r] and g[r] is None]
        if pending:
            sizes = [int(torch.Size(shapes[r]).numel()) for r in pending]
            slab = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
            for r, t in zip(pending, torch.split(slab, sizes)):
                g[r] = t.view(shapes[r])
        # ---- MLP branch ----
        # bf16(DropPath scale * dx2) and its column sums (fc2 bias gradient) normally arrive from the LN1 backward of
        # the block above, which produced dx2 (hand-off through the step's StepLink); otherwise one pass over dx2 here
        link = env.link if env is not None else None
        ho = link.handoff if link is not None else None
        if ho is not None:
            link.handoff = None
            if ho[0].data_ptr() != dx2.data_ptr() or ho[0].shape != dx2.shape:
                raise RuntimeError("painter_b200: gradient hand-off between blocks does not match the incoming grad")
            dy = ho[1]
        else:
            dy, _ = ops.scale_cast_colsum(dx2, drop_m, N, want_colsum=need["fc2_b"], colsum_out=g["fc2_b"])
        if need["fc2_w"]:
            _wgrad(dy, hact, out=g["fc2_w"])
        dz = ops.gemm(dy, wfc2, trans_b=True, kind=EPI_DGELU, aux=z)
        if need["fc1_b"]:
            ops.colsum_bf16(dz, out=g["fc1_b"])
        if need["fc1_w"]:
            _wgrad(dz, v, out=g["fc1_w"])
        # dgrad outputs that feed a LayerNorm backward are written as bf16 (the reference's autocast Linear backward
        # rounds there too): half the store traffic of the GEMM epilogue and of the LN-backward's dy stream
        dv = ops.gemm(dz, wfc1, trans_b=True, kind=EPI_BF16)
        # LN2 backward also emits the attention branch's incoming gradient: bf16(DropPath scale * dx1) + its column sums
        dx1, da = ops.layernorm_bwd(dv, x1, mean2, rstd2, n2w, g["n2w"], g["n2b"], dres=dx2,
                                    cast=(drop_a, N, g["proj_b"]))
        # ---- attention branch ----
        if ws > 0:
            da = ops.window_partition_bf16(da, Bp, h, w, ws)
            Bw = da.shape[0] // (ws * ws)
        if need["proj_w"]:
            _wgrad(da, ao, out=g["proj_w"])
        # the rest of the chain only as far as something below needs it: dx / LN1 (x or norm1 trainable), then dqkv
        need_dx = ctx.needs_input_grad[0]
        need_du = need_dx or need["n1w"] or need["n1b"]
        if not (need_du or need["qkv_w"] or need["qkv_b"] or tables):
            if act:
                env.arena.stage_done(env.name)
            return (None, None, None, *[g[r] if need[r] else None for r in BLOCK_ROLES], None, None)
        dao = ops.gemm(da, wproj, trans_b=True, kind=EPI_BF16)
        dT = (g["rel_h"], g["rel_w"]) if tables else None
        if ws > 0:
            dqkv, _, _ = ops.attn_bwd(qkv, ao, dao, lse, th, tw, Bw, heads, ws, ws, dT_out=dT, rel=rel,
                                      table_grads=tables)
        else:
            dqkv, _, _ = ops.attn_bwd(qkv, ao, dao, lse, th, tw, Bp, heads, h, w, dT_out=dT, rel=rel,
                                      table_grads=tables)
        if need["qkv_b"]:
            ops.colsum_bf16(dqkv, out=g["qkv_b"])
        if need["qkv_w"]:
            _wgrad(dqkv, u, out=g["qkv_w"])
        dx = None
        if need_du:
            if ws > 0:
                du = ops.gemm(dqkv, wqkv, trans_b=True, kind=EPI_F32)
                du = ops.window_unpartition(du, Bp, h, w, ws)   # gradients at padded tokens are dropped
            else:
                du = ops.gemm(dqkv, wqkv, trans_b=True, kind=EPI_BF16)
            # the block below consumes dx only through bf16(its DropPath scale * dx): emit that - and the fc2 bias
            # gradient it implies, into its arena slot, unless that bias is frozen - in the same pass (with no arena
            # and a trainable bias, the block below makes its own pass)
            below = env.below if (env is not None and need_dx) else None
            if below is not None and below[0].requires_grad and not act:
                below = None
            if below is not None:
                b_fc2_b, b_drop_m, b_N = below
                dx, dxb = ops.layernorm_bwd(du, x, mean1, rstd1, n1w, g["n1w"], g["n1b"], dres=dx1,
                                            cast=(b_drop_m, b_N,
                                                  env.arena.view(b_fc2_b) if b_fc2_b.requires_grad else None))
                link.handoff = (dx, dxb)
            else:
                dx = ops.layernorm_bwd(du, x, mean1, rstd1, n1w, g["n1w"], g["n1b"], dres=dx1)
        if act:
            env.arena.stage_done(env.name)
        return (dx if need_dx else None, None, None, *[g[r] if need[r] else None for r in BLOCK_ROLES], None, None)


class MergeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        return ops.merge_halves(z)

    @staticmethod
    def backward(ctx, d):
        return ops.merge_halves_bwd(d.contiguous())


class DecoderFn(torch.autograd.Function):
    """(4 tap activations) -> (loss[1], patchified prediction [B, N, p*p*3]).  The loss's gradient with respect to
    tgts (-dpred, from the fused head backward) is returned when tgts requires grad; autograd adds it to the encoder's.
    Parameter gradients are computed only for parameters that require grad; `cat` / `g` (the operands of the
    decoder-embed and 3x3 weight gradients) are saved only if those weights require grad."""

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
        need = ctx.needs_input_grad
        ctx.save_for_backward(t0, t1, t2, t3, norm_w, cat if need[6] else None, wdec, g if need[8] else None, wd, hp,
                              c1, tgts, mask_u8, valid, coef, *[s for pair in stats for s in pair])
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
        need = ctx.needs_input_grad
        env = ctx.env
        act = env is not None and env.begin()
        G = (lambda k: env.grad(True, k)) if act else (lambda k: None)
        gscale = dloss.reshape(1).to(torch.float32).contiguous()
        head = any(need[10:14])
        dtg = None
        if need[14]:
            dc1, dhp, dtg = ops.decoder_head_bwd_dtgt(c1, tgts, mask_u8, valid, coef, gscale, hp, p, loss_kind,
                                                      params=head)
        else:
            dc1, dhp = ops.decoder_head_bwd(c1, tgts, mask_u8, valid, coef, gscale, hp, p, loss_kind, params=head)
        dc3_b = ops.colsum_bf16(dc1.view(-1, 64), out=G("c3_b")) if need[9] else None
        dc3_w = ops.conv3x3_wgrad(g, dc1, out=G("c3_w")) if need[8] else None
        ddec_w = ddec_b = dnw = dnb = None
        dts = [None] * 4
        if any(need[0:8]):
            dD = ops.conv3x3_dgrad_unshuffle(dc1, wd, p)          # [M, p*p*64] bf16, token-major
            ddec_b = ops.colsum_bf16(dD, out=G("dec_b")) if need[7] else None
            ddec_w = _wgrad(dD, cat, out=G("dec_w")) if need[6] else None
            if any(need[0:6]):
                dcat = ops.gemm(dD, wdec, trans_b=True, kind=EPI_BF16)  # [M, 4C] bf16, read by the 4 LN backwards
                if need[4]:
                    dnw = G("norm_w") if act else torch.zeros(C, dtype=torch.float32, device=dev)
                if need[5]:
                    dnb = G("norm_b") if act else torch.zeros(C, dtype=torch.float32, device=dev)
                for k in range(4):
                    dts[k] = ops.layernorm_bwd(dcat[:, k * C:(k + 1) * C], t[k], stats[2 * k], stats[2 * k + 1],
                                               norm_w, dnw, dnb)
        c3shape, c1shape = ctx.shapes
        dlw = dlb = dc1w = dc1b = None
        if act:
            if need[10]:
                dlw = G("ln_w")
                dlw.copy_(dhp[64:128])
            if need[11]:
                dlb = G("ln_b")
                dlb.copy_(dhp[128:192])
            if need[12]:
                dc1w = G("c1_w")
                dc1w.view(-1).copy_(dhp[192:384])
            if need[13]:
                dc1b = G("c1_b")
                dc1b.copy_(dhp[384:387])
            env.arena.stage_done(env.name)
        else:
            if need[10]:
                dlw = dhp[64:128].clone()
            if need[11]:
                dlb = dhp[128:192].clone()
            if need[12]:
                dc1w = dhp[192:384].reshape(c1shape).clone()
            if need[13]:
                dc1b = dhp[384:387].clone()
        return (dts[0] if need[0] else None, dts[1] if need[1] else None, dts[2] if need[2] else None,
                dts[3] if need[3] else None, dnw, dnb, ddec_w, ddec_b, dc3_w, dc3_b, dlw, dlb, dc1w, dc1b, dtg, None,
                None, None, None)
