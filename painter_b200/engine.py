"""Host-side orchestration of the hot path: one torch.autograd.Function per stage (embed, block, merge,
decoder+loss) so that autograd / DDP hooks fire block by block.  Every arithmetic step is a call into
libpainter_b200.so (painter_b200/ops.py); torch is used for memory, streams and the autograd tape only.

Stage map (reference file:line -> Function):
  EmbedFn     Painter/models_painter.py:385-409 (PatchEmbed x2, mask-token blend, segment/pos/type tokens)
  BlockFn     Painter/models_painter.py:216-235 + Attention :73-89 (+ SegGPT ensemble models_seggpt.py:220-231)
  MergeFn     Painter/models_painter.py:414-415
  DecoderFn   Painter/models_painter.py:417 (final LN taps), :420-431 (decoder), :433-462 (loss), :355-368 (patchify)

Each stage with parameters declares their roles once (ROLES, in forward-signature order from input FIRST); the module
states which parameter fills each role (models_painter.Painter.grad_stages, which also fixes the gradient arena's
layout).  A backward reads ctx.needs_input_grad as {role: bool} through _needs, gets its zero-initialised gradient
accumulators from StageEnv.targets and ends with StageEnv.done.
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
    """Per-forward bookkeeping of one stage's backward (non-tensor argument; every stage gets one when grad is
    enabled): the module's gradient arena (None: no parameter requires grad), a token that identifies the step, the
    stage's arena group name, its parameter inputs by role as the stage receives them (a resized rel-pos table is not
    the parameter), and - for a block - the block below it in the stack (whose MLP branch consumes this block's dx)
    and the forward's StepLink that carries the hand-off.  `begin`, `targets` and `done` are the whole arena protocol
    of a backward stage."""
    __slots__ = ("arena", "token", "name", "prm", "below", "link", "active")

    def __init__(self, arena, token, name, prm, below=None, link=None):
        self.arena, self.token, self.name, self.prm, self.below, self.link = arena, token, name, prm, below, link
        self.active = False

    def begin(self):
        """Starts the stage's backward; `active`: it writes parameter gradients into the arena."""
        self.active = self.arena is not None and self.arena.begin_backward(self.token)

    def targets(self, want):
        """{role: zero-initialised fp32 gradient accumulator at the input's shape, or None} over the stage's roles.
        `want`: the roles the backward writes - those that require grad, plus frozen ones a kernel reduces together
        with a trainable one.  A role gets its arena slot when this backward writes into the arena and its input is
        the arena's parameter; the others (no arena, or a resized rel-pos table, whose gradient flows on through
        autograd) share ONE zero-filled slab for the stage."""
        g = dict.fromkeys(self.prm)
        rest = []
        for r, t in self.prm.items():
            if r in want:
                if self.active and self.arena.owns(t):
                    g[r] = self.arena.view(t)
                else:
                    rest.append(r)
        if rest:
            sizes = [self.prm[r].numel() for r in rest]
            slab = torch.zeros(sum(sizes), dtype=torch.float32, device=self.prm[rest[0]].device)
            for r, t in zip(rest, torch.split(slab, sizes)):
                g[r] = t.view(self.prm[r].shape)
        return g

    def done(self, g, need, last=False):
        """Ends the stage's backward: its arena group is enqueued (and, for the last stage, the whole backward).
        Returns the parameter gradients in role order, None where the input does not require grad."""
        if self.active:
            self.arena.stage_done(self.name)
            if last:
                self.arena.end_backward()
        return tuple(g[r] if n else None for r, n in need.items())


def _needs(ctx, fn):
    """(requires-grad flags of fn's inputs before its parameters, {role: requires grad} of its parameter inputs)."""
    n = ctx.needs_input_grad
    return n[:fn.FIRST], dict(zip(fn.ROLES, n[fn.FIRST:]))


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


def _wgrad(dy_bf16, x_bf16, out):
    """dW[out, in] = dY^T . X  (both operands read MN-major; stream-K over the zero-initialised fp32 output)."""
    return ops.gemm(dy_bf16, x_bf16, trans_a=True, trans_b=True, kind=EPI_F32, out=out, accumulate=2)


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
    ROLES = ("w", "b", "mt", "sx", "sy", "tc", "ti", "pe")   # the parameter inputs Wp .. pos_embed
    FIRST = 4

    @staticmethod
    def forward(ctx, imgs, tgts, mask_u8, seg_type, Wp, bp, mask_token, seg_x, seg_y, type_cls, type_ins, pos_embed,
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
        (need_imgs, need_tgts, _, _), need = _needs(ctx, EmbedFn)
        need_type = seg_type is not None and (need["tc"] or need["ti"])
        ctx.save_for_backward(cols if need["w"] else None, mask_u8, wp if (need_imgs or need_tgts) else None,
                              seg_type.reshape(B).contiguous() if need_type else None)
        ctx.meta = (B, N, C, h, w, s, has_cls, need_type, (Cin, H, W, p))
        ctx.env = env
        return z

    @staticmethod
    def backward(ctx, dz):
        cols, mask_u8, wp, seg_type = ctx.saved_tensors
        B, N, C, h, w, s, has_cls, need_type, (Cin, H, W, p) = ctx.meta
        (need_imgs, need_tgts, _, _), need = _needs(ctx, EmbedFn)
        env = ctx.env
        env.begin()
        dz = dz.contiguous()
        # the three tokens are reduced in one pass, and so are the two type tokens, even when only one requires grad
        need_tok = need["mt"] or need["sx"] or need["sy"]
        want = {r for r, n in need.items() if n}
        if need_tok:
            want |= {"mt", "sx", "sy"}
        if need_type:
            want |= {"tc", "ti"}
        g = env.targets(want)
        tok = (g["sx"].view(C), g["sy"].view(C), g["mt"].view(C)) if need_tok else None
        typ = (seg_type, g["tc"].view(C), g["ti"].view(C)) if need_type else None
        dE, dpos, _, _, _ = ops.assemble_tokens_bwd(dz, mask_u8, B, N, C, token_grads=tok, want_tokens=need_tok,
                                                    want_pos=need["pe"], type_grads=typ)
        if need["w"]:
            _wgrad(dE, cols, out=g["w"].view(C, -1))
        if need["b"]:
            ops.colsum_bf16(dE, out=g["b"])
        if need["pe"]:
            off = 1 if has_cls else 0
            if s == h and s == w:
                g["pe"][0, off:] = dpos
            else:
                ops.bicubic_bwd(dpos.view(h, w, C), s, s, out=g["pe"][0, off:].view(s, s, C))
        dimgs = dtgts = None
        if need_imgs or need_tgts:
            # patch-embed dgrad dE . Wp of the wanted halves only (x rows -> imgs, y rows -> tgts), one GEMM over the
            # rows of both when both are wanted, then the inverse of the im2col layout
            lo, hi = (0 if need_imgs else B * N), (2 * B * N if need_tgts else B * N)
            dcols = ops.gemm(dE[lo:hi], wp, trans_b=True, kind=EPI_F32)
            dimgs, dtgts = ops.col2im_patch(dcols[:B * N] if need_imgs else None,
                                            dcols[hi - lo - B * N:] if need_tgts else None, B, Cin, H, W, p)
        return (dimgs, dtgts, None, None, *env.done(g, need, last=True), None, None, None)


class BlockFn(torch.autograd.Function):
    """x [B'*N, C] fp32 -> same.  meta = (Bp, h, w, heads, eps, ens_groups, ens_P, ws); ws > 0 = windowed block
    (vitdet_utils.window_partition / window_unpartition around the attention, models_painter.py:220-227).
    Every parameter gradient (weight-gradient GEMM, bias column sums, LayerNorm affine reductions, rel-pos table
    gradients) is computed only if that parameter requires grad, and the activations only the weight gradients read
    (u, v, hact) are saved only if qkv / fc1 / fc2 weight requires grad; the dx chain is the same either way.
    Without an env (a block applied on its own) every gradient goes to the stage's zero slab and nothing is handed
    off."""
    ROLES = ("n1w", "n1b", "rel_h", "rel_w", "qkv_w", "qkv_b", "proj_w", "proj_b", "n2w", "n2b", "fc1_w", "fc1_b",
             "fc2_w", "fc2_b")
    FIRST = 3

    @staticmethod
    def forward(ctx, x, drop_a, drop_m, n1w, n1b, rel_h, rel_w, qkv_w, qkv_b, proj_w, proj_b, n2w, n2b, fc1_w,
                fc1_b, fc2_w, fc2_b, meta, env=None):
        Bp, h, w, heads, eps, ens_groups, ens_P, ws = meta
        if env is None:
            env = StageEnv(None, None, "block", dict(zip(BlockFn.ROLES, (
                n1w, n1b, rel_h, rel_w, qkv_w, qkv_b, proj_w, proj_b, n2w, n2b, fc1_w, fc1_b, fc2_w, fc2_b))))
        ctx.env = env
        N = h * w
        M, C = x.shape
        u, mean1, rstd1 = ops.layernorm_fwd(x, n1w, n1b, eps)
        wqkv, wproj = bf16_weight(qkv_w), bf16_weight(proj_w)
        wfc1, wfc2 = bf16_weight(fc1_w), bf16_weight(fc2_w)
        th, tw = bf16_table(rel_h), bf16_table(rel_w)
        # attention geometry (batch, grid): the zero-padded windows [Bp*nW*ws*ws, C] of a windowed block, else the grid
        if ws > 0:
            u = ops.window_partition_bf16(u, Bp, h, w, ws)
            ctx.geom = (u.shape[0] // (ws * ws), ws, ws)
        else:
            ctx.geom = (Bp, h, w)
        qkv = ops.gemm(u, wqkv, kind=EPI_BF16, bias=qkv_b)
        ao, lse = ops.attn_fwd(qkv, th, tw, ctx.geom[0], heads, *ctx.geom[1:])
        if ws == 0 and ens_groups == 0:
            x1 = ops.gemm(ao, wproj, kind=EPI_RESID, bias=proj_b, aux=x, rowscale=drop_a, rows_per_group=N)
        else:
            a = ops.gemm(ao, wproj, kind=EPI_F32, bias=proj_b)
            if ens_groups > 0:   # the ensemble merges on the full token grid, after window_unpartition
                x1 = ops.ensemble_resid(ops.window_unpartition(a, Bp, h, w, ws) if ws > 0 else a, x, ens_groups,
                                        ens_P, N, C)
            else:
                x1 = ops.window_unpartition(a, Bp, h, w, ws, resid=x, rowscale=drop_a)
        v, mean2, rstd2 = ops.layernorm_fwd(x1, n2w, n2b, eps)
        z, hact = ops.gemm(v, wfc1, kind=EPI_GELU, bias=fc1_b)
        x2 = ops.gemm(hact, wfc2, kind=EPI_RESID, bias=fc2_b, aux=x1, rowscale=drop_m, rows_per_group=N)
        _, need = _needs(ctx, BlockFn)
        ctx.save_for_backward(x, mean1, rstd1, u if need["qkv_w"] else None, qkv, ao, lse, th, tw, x1, mean2, rstd2,
                              v if need["fc1_w"] else None, z, hact if need["fc2_w"] else None, wqkv, wproj, wfc1,
                              wfc2, n1w, n2w, drop_a, drop_m)
        ctx.meta = meta
        return x2

    @staticmethod
    def backward(ctx, dx2):
        (x, mean1, rstd1, u, qkv, ao, lse, th, tw, x1, mean2, rstd2, v, z, hact, wqkv, wproj, wfc1, wfc2, n1w, n2w,
         drop_a, drop_m) = ctx.saved_tensors
        Bp, h, w, heads, eps, ens_groups, ens_P, ws = ctx.meta
        if ens_groups > 0:
            raise NotImplementedError("painter_b200: backward through the SegGPT prompt ensemble is not implemented")
        N = h * w
        dx2 = dx2.contiguous()
        (need_dx, _, _), need = _needs(ctx, BlockFn)
        tables = need["rel_h"] or need["rel_w"]
        # Accumulation targets of the parameters that require grad (LN affine grads, bias grads, the four weight
        # gradients the stream-K GEMMs add into, the rel-pos table gradients); None for a frozen parameter: its
        # reduction is skipped.  The attention kernel produces both table gradients together.
        env = ctx.env
        env.begin()
        g = env.targets({r for r, n in need.items() if n} | ({"rel_h", "rel_w"} if tables else set()))
        # ---- MLP branch ----
        # bf16(DropPath scale * dx2) and its column sums (fc2 bias gradient) normally arrive from the LN1 backward of
        # the block above, which produced dx2 (hand-off through the step's StepLink); otherwise one pass over dx2 here
        link = env.link
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
        if need["proj_w"]:
            _wgrad(da, ao, out=g["proj_w"])
        # the rest of the chain only as far as something below needs it: dx / LN1 (x or norm1 trainable), then dqkv
        need_du = need_dx or need["n1w"] or need["n1b"]
        if not (need_du or need["qkv_w"] or need["qkv_b"] or tables):
            return (None, None, None, *env.done(g, need), None, None)
        dao = ops.gemm(da, wproj, trans_b=True, kind=EPI_BF16)
        Bw, gh, gw = ctx.geom
        dqkv, _, _ = ops.attn_bwd(qkv, ao, dao, lse, th, tw, Bw, heads, gh, gw,
                                  dT_out=(g["rel_h"], g["rel_w"]) if tables else None, table_grads=tables)
        if need["qkv_b"]:
            ops.colsum_bf16(dqkv, out=g["qkv_b"])
        if need["qkv_w"]:
            _wgrad(dqkv, u, out=g["qkv_w"])
        dx = None
        if need_du:
            du = ops.gemm(dqkv, wqkv, trans_b=True, kind=EPI_F32 if ws > 0 else EPI_BF16)
            if ws > 0:
                du = ops.window_unpartition(du, Bp, h, w, ws)   # gradients at padded tokens are dropped
            # the block below consumes dx only through bf16(its DropPath scale * dx): emit that - and the fc2 bias
            # gradient it implies, into its arena slot, unless that bias is frozen - in the same pass (with no arena
            # and a trainable bias, the block below makes its own pass)
            below = env.below if need_dx else None
            if below is not None and below[0].requires_grad and not env.active:
                below = None
            if below is not None:
                b_fc2_b, b_drop_m, b_N = below
                dx, dxb = ops.layernorm_bwd(du, x, mean1, rstd1, n1w, g["n1w"], g["n1b"], dres=dx1,
                                            cast=(b_drop_m, b_N,
                                                  env.arena.view(b_fc2_b) if b_fc2_b.requires_grad else None))
                link.handoff = (dx, dxb)
            else:
                dx = ops.layernorm_bwd(du, x, mean1, rstd1, n1w, g["n1w"], g["n1b"], dres=dx1)
        return (dx if need_dx else None, None, None, *env.done(g, need), None, None)


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
    Parameter gradients are computed only for parameters that require grad; `cat` / `ps` (the operands of the
    decoder-embed and 3x3 weight gradients) are saved only if those weights require grad."""
    ROLES = ("norm_w", "norm_b", "dec_w", "dec_b", "c3_w", "c3_b", "ln_w", "ln_b", "c1_w", "c1_b")
    FIRST = 5

    @staticmethod
    def forward(ctx, t0, t1, t2, t3, tgts, norm_w, norm_b, dec_w, dec_b, c3_w, c3_b, ln_w, ln_b, c1_w, c1_b, mask_u8,
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
        ps = torch.empty((B, h * p, w * p, dd), dtype=torch.bfloat16, device=dev)
        ops.gemm(cat, wdec, kind=EPI_PIXSHUF, bias=dec_b, pixshuf=(h, w, p, dd, ps))
        wf, wd = ops.conv3x3_pack(c3_w.contiguous())
        hp = ops.pack_head_params(c3_b, ln_w, ln_b, c1_w, c1_b)
        st = ops.loss_prep(tgts, mask_u8, valid, p)
        c1, patch, num = ops.decoder_head_fwd(ps, wf, hp, tgts, mask_u8, valid, p, loss_kind)
        loss, coef = ops.loss_finalize(st, num, seggpt)
        _, need = _needs(ctx, DecoderFn)
        ctx.save_for_backward(t0, t1, t2, t3, norm_w, cat if need["dec_w"] else None, wdec,
                              ps if need["c3_w"] else None, wd, hp, c1, tgts, mask_u8, valid, coef,
                              *[s for pair in stats for s in pair])
        ctx.meta = meta
        ctx.mark_non_differentiable(patch)
        return loss, patch

    @staticmethod
    def backward(ctx, dloss, _dpatch):
        sv = ctx.saved_tensors
        t = sv[0:4]
        norm_w, cat, wdec, ps, wd, hp, c1, tgts, mask_u8, valid, coef = sv[4:15]
        stats = sv[15:]
        B, h, w, p, eps, loss_kind, seggpt = ctx.meta
        C = t[0].shape[1]
        (*need_taps, need_tgts), need = _needs(ctx, DecoderFn)
        env = ctx.env
        env.begin()
        g = env.targets({r for r, n in need.items() if n})
        gscale = dloss.reshape(1).to(torch.float32).contiguous()
        head = any(need[r] for r in ops.HEAD_SLICES)
        dtg = None
        if need_tgts:
            dc1, dhp, dtg = ops.decoder_head_bwd_dtgt(c1, tgts, mask_u8, valid, coef, gscale, hp, p, loss_kind,
                                                      params=head)
        else:
            dc1, dhp = ops.decoder_head_bwd(c1, tgts, mask_u8, valid, coef, gscale, hp, p, loss_kind, params=head)
        if need["c3_b"]:
            ops.colsum_bf16(dc1.view(-1, 64), out=g["c3_b"])
        if need["c3_w"]:
            ops.conv3x3_wgrad(ps, dc1, out=g["c3_w"])
        dts = [None] * 4
        need_ln = any(need_taps) or need["norm_w"] or need["norm_b"]
        if need_ln or need["dec_w"] or need["dec_b"]:
            dD = ops.conv3x3_dgrad_unshuffle(dc1, wd, p)          # [M, p*p*64] bf16, token-major
            if need["dec_b"]:
                ops.colsum_bf16(dD, out=g["dec_b"])
            if need["dec_w"]:
                _wgrad(dD, cat, out=g["dec_w"])
            if need_ln:
                dcat = ops.gemm(dD, wdec, trans_b=True, kind=EPI_BF16)  # [M, 4C] bf16, read by the 4 LN backwards
                for k in range(4):
                    dts[k] = ops.layernorm_bwd(dcat[:, k * C:(k + 1) * C], t[k], stats[2 * k], stats[2 * k + 1],
                                               norm_w, g["norm_w"], g["norm_b"])
        for r, sl in ops.HEAD_SLICES.items():
            if need[r]:
                g[r].view(-1).copy_(dhp[sl])
        return (*[d if n else None for d, n in zip(dts, need_taps)], dtg, *env.done(g, need), None, None, None,
                None)
