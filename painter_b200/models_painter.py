"""H100-native drop-in for the reference `Painter` module (Painter/models_painter.py:238-487).

Same constructor arguments, same `forward(imgs, tgts, bool_masked_pos=None, valid=None)` ->
`(loss, patchify(pred), bool_masked_pos)`, same attributes (`patch_size`, `patch_embed.num_patches`, `blocks`,
`pos_embed`, `no_weight_decay()`, `patchify/unpatchify`) and IDENTICAL state-dict keys/shapes, so
`painter_vit_large.pth` / MAE checkpoints load and `engine_train.train_one_epoch` runs unchanged.  The
`nn.Linear / nn.LayerNorm / nn.Conv2d` children are parameter holders only: their `forward` is never called —
all arithmetic goes through painter_b200.engine (hand-written sm_90a kernels).  There is no CPU path.
"""
from functools import partial

import torch
import torch.nn as nn

from . import engine, ops
from .arena import get_arena
from .engine import BlockFn, DecoderFn, EmbedFn, MergeFn, StageEnv


def trunc_normal_(tensor, mean=0.0, std=1.0):
    return nn.init.trunc_normal_(tensor, mean=mean, std=std, a=-2.0, b=2.0)


class Mlp(nn.Module):
    """Parameter holder with timm-0.3.2 `Mlp` key names (fc1, fc2)."""

    def __init__(self, in_features, hidden_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features, in_features)


class Attention(nn.Module):
    """Parameter holder for models_painter.py:33-71 (qkv, proj, rel_pos_h, rel_pos_w)."""

    def __init__(self, dim, num_heads=8, qkv_bias=True, use_rel_pos=False, rel_pos_zero_init=True, input_size=None):
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        if head_dim != 64:
            raise NotImplementedError("painter_b200: the attention kernels are specialised for head_dim = 64")
        self.scale = head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.use_rel_pos = use_rel_pos
        if not use_rel_pos:
            raise NotImplementedError("painter_b200: use_rel_pos=False is not a configuration of the reference path")
        self.rel_pos_h = nn.Parameter(torch.zeros(2 * input_size[0] - 1, head_dim))
        self.rel_pos_w = nn.Parameter(torch.zeros(2 * input_size[1] - 1, head_dim))
        if not rel_pos_zero_init:
            trunc_normal_(self.rel_pos_h, std=0.02)
            trunc_normal_(self.rel_pos_w, std=0.02)


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4.0, qkv_bias=True, drop_path=0.0, norm_layer=nn.LayerNorm,
                 use_rel_pos=False, rel_pos_zero_init=True, window_size=0, input_size=None):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, use_rel_pos=use_rel_pos,
                              rel_pos_zero_init=rel_pos_zero_init,
                              input_size=input_size if window_size == 0 else (window_size, window_size))
        self.drop_prob = float(drop_path)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))
        self.window_size = window_size

    def params(self):
        """The block's parameters in BlockFn.ROLES order (BlockFn's parameter inputs)."""
        a, m = self.attn, self.mlp
        return (self.norm1.weight, self.norm1.bias, a.rel_pos_h, a.rel_pos_w, a.qkv.weight, a.qkv.bias,
                a.proj.weight, a.proj.bias, self.norm2.weight, self.norm2.bias, m.fc1.weight, m.fc1.bias,
                m.fc2.weight, m.fc2.bias)


class PatchEmbed(nn.Module):
    """Parameter holder for vitdet_utils.py:160-186 (proj = Conv2d(k16, s16))."""

    def __init__(self, kernel_size=(16, 16), stride=(16, 16), padding=(0, 0), in_chans=3, embed_dim=768):
        super().__init__()
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=kernel_size, stride=stride, padding=padding)


class LayerNorm2D(nn.Module):
    """Parameter holder for vitdet_utils.py:189-209."""

    def __init__(self, normalized_shape, eps=1e-6):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(normalized_shape))
        self.bias = nn.Parameter(torch.zeros(normalized_shape))
        self.eps = eps


class Painter(nn.Module):
    seggpt = False
    # arithmetic of forward: "bf16" (tensor-core operands in bf16, fp32 accumulate - the training mode), "fp32"
    # (fp32-accurate split-operand mode, painter_b200/accurate.py, forward only) or "auto": fp32-accurate when the
    # module is called the way the reference's inference code calls it - outside autocast, gradients disabled
    # (seggpt_engine.py:26,47) - and bf16 otherwise (engine_train.py:65 runs under autocast)
    precision = "auto"

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=1024, depth=24, num_heads=16,
                 mlp_ratio=4., qkv_bias=True, drop_path_rate=0., norm_layer=nn.LayerNorm, act_layer=nn.GELU,
                 use_abs_pos=True, use_rel_pos=False, rel_pos_zero_init=True, window_size=0,
                 window_block_indexes=(), residual_block_indexes=(), use_act_checkpoint=False,
                 pretrain_img_size=224, pretrain_use_cls_token=True, out_feature="last_feat",
                 decoder_embed_dim=128, loss_func="smoothl1"):
        super().__init__()
        if len(tuple(residual_block_indexes)) > 0:
            raise NotImplementedError("painter_b200: residual_block_indexes (ResBottleneckBlock) is not used by any "
                                      "reference configuration and is not implemented")
        if not use_abs_pos:
            raise NotImplementedError("painter_b200: use_abs_pos=False is not implemented")
        if depth < 24:
            raise ValueError("depth must be >= 24: the taps [5, 11, 17, 23] are hard-coded (models_painter.py:416)")
        self.pretrain_use_cls_token = pretrain_use_cls_token
        self.patch_size = patch_size
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.patch_embed = PatchEmbed(kernel_size=(patch_size, patch_size), stride=(patch_size, patch_size),
                                      in_chans=in_chans, embed_dim=embed_dim)
        self.patch_embed.num_patches = (img_size[0] // patch_size) * (img_size[1] // patch_size)
        self.mask_token = nn.Parameter(torch.zeros(1, 1, 1, embed_dim))
        self.segment_token_x = nn.Parameter(torch.zeros(1, 1, 1, embed_dim))
        self.segment_token_y = nn.Parameter(torch.zeros(1, 1, 1, embed_dim))
        self._extra_tokens(embed_dim)
        num_patches = (pretrain_img_size // patch_size) * (pretrain_img_size // patch_size)
        num_positions = (num_patches + 1) if pretrain_use_cls_token else num_patches
        self.pos_embed = nn.Parameter(torch.zeros(1, num_positions, embed_dim), requires_grad=True)

        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.blocks = nn.ModuleList()
        for i in range(depth):
            # NB: `i in window_block_indexes` is evaluated exactly like the reference (models_painter.py:307):
            # the stock factories pass a tuple of LISTS, so no block is windowed (SURVEY.md section 0.1).
            self.blocks.append(Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                                     drop_path=dpr[i], norm_layer=norm_layer, use_rel_pos=use_rel_pos,
                                     rel_pos_zero_init=rel_pos_zero_init,
                                     window_size=window_size if i in window_block_indexes else 0,
                                     input_size=(img_size[0] // patch_size, img_size[1] // patch_size)))
        self._out_feature_channels = {out_feature: embed_dim}
        self._out_feature_strides = {out_feature: patch_size}
        self._out_features = [out_feature]
        trunc_normal_(self.pos_embed, std=0.02)
        self.norm = norm_layer(embed_dim)

        self.decoder_embed_dim = decoder_embed_dim
        self.decoder_embed = nn.Linear(embed_dim * 4, patch_size ** 2 * self.decoder_embed_dim, bias=True)
        self.decoder_pred = nn.Sequential(
            nn.Conv2d(self.decoder_embed_dim, self.decoder_embed_dim, kernel_size=3, padding=1),
            LayerNorm2D(self.decoder_embed_dim),
            nn.GELU(),
            nn.Conv2d(self.decoder_embed_dim, 3, kernel_size=1, bias=True),
        )
        self.loss_func = loss_func
        if loss_func not in engine.LOSS_KINDS:
            raise ValueError(f"unknown loss_func {loss_func}")
        torch.nn.init.normal_(self.mask_token, std=.02)
        torch.nn.init.normal_(self.segment_token_x, std=.02)
        torch.nn.init.normal_(self.segment_token_y, std=.02)
        self._init_extra_tokens()
        self.apply(self._init_weights)

    # ---- hooks the SegGPT subclass overrides ----
    def _extra_tokens(self, embed_dim):
        pass

    def _init_extra_tokens(self):
        pass

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'pos_embed', 'cls_token'}

    # ---- pure layout helpers (models_painter.py:355-383) ----
    def patchify(self, imgs):
        p = self.patch_size
        assert imgs.shape[2] == 2 * imgs.shape[3] and imgs.shape[2] % p == 0
        w = imgs.shape[3] // p
        h = w * 2
        x = imgs.reshape(imgs.shape[0], 3, h, p, w, p).permute(0, 2, 4, 3, 5, 1)
        return x.reshape(imgs.shape[0], h * w, p ** 2 * 3)

    def unpatchify(self, x):
        p = self.patch_size
        w = int((x.shape[1] * 0.5) ** .5)
        h = w * 2
        assert h * w == x.shape[1]
        x = x.reshape(x.shape[0], h, w, p, p, 3).permute(0, 5, 1, 3, 2, 4)
        return x.reshape(x.shape[0], 3, h * p, w * p)

    # ---- the hot path ----
    def _draw_drop_scales(self, B, device):
        """timm DropPath (models_painter.py:199,229-230) for the whole step: per-sample scales
        floor(keep + U[0,1)) / keep.  The uniform draws are made with torch.rand in the reference's order, shapes and
        dtype (attention branch then MLP branch of every block with p > 0; batch 2B up to the early merge; the
        branch output's dtype, i.e. the autocast dtype) so that a seeded run drops the same branches as the
        reference; one kernel then turns all of them into scales.  Returns {block: (scale_attn, scale_mlp)}."""
        if not self.training:
            return {}
        dt = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float32
        draws, keeps, slots = [], [], []
        for i, blk in enumerate(self.blocks):
            p = blk.drop_prob
            if p == 0.0:
                continue
            Bp = 2 * B if i <= 2 else B
            for br in range(2):
                draws.append(torch.rand((Bp, 1, 1, 1), dtype=dt, device=device).reshape(Bp))
                keeps.append((1.0 - p, Bp))
                slots.append((i, br, Bp))
        if not draws:
            return {}
        key = (B, str(device), tuple(k for k, _ in keeps))
        cache = self.__dict__.get("_pk_keep_cache")
        if cache is None or cache[0] != key:
            kv = torch.cat([torch.full((n,), k, dtype=torch.float32) for k, n in keeps]).to(device)
            cache = (key, kv)
            self.__dict__["_pk_keep_cache"] = cache
        scales = ops.droppath_scales(torch.cat(draws), cache[1])
        out, off = {}, 0
        for i, br, Bp in slots:
            out.setdefault(i, [None, None])[br] = scales[off:off + Bp]
            off += Bp
        return {i: tuple(v) for i, v in out.items()}

    def _drop_scales(self, i, Bp, device):
        """Per-block view of the step's DropPath scales (tests replace this to replay the reference's CPU draws)."""
        return self._step_drops.get(i, (None, None))

    def grad_stages(self):
        """{stage: {role: parameter}} in backward production order (decoder, block N-1 ... block 0, embed), the roles
        of each stage in the order of its Function's parameter inputs (engine.DecoderFn / BlockFn / EmbedFn.ROLES;
        Painter has no type tokens "tc" / "ti").  The gradient arena lays its slab out in exactly this order, and
        _run hands every stage its parameters from here."""
        dp, pe = self.decoder_pred, self.patch_embed.proj
        out = {"decoder": dict(zip(DecoderFn.ROLES, (self.norm.weight, self.norm.bias, self.decoder_embed.weight,
                                                     self.decoder_embed.bias, dp[0].weight, dp[0].bias, dp[1].weight,
                                                     dp[1].bias, dp[3].weight, dp[3].bias)))}
        for i in reversed(range(len(self.blocks))):
            out[f"block{i}"] = dict(zip(BlockFn.ROLES, self.blocks[i].params()))
        emb = {"w": pe.weight, "b": pe.bias, "mt": self.mask_token, "sx": self.segment_token_x,
               "sy": self.segment_token_y}
        if self.seggpt:
            emb.update(tc=self.type_token_cls, ti=self.type_token_ins)
        emb["pe"] = self.pos_embed
        out["embed"] = emb
        return out

    def _type_inputs(self, B, seg_type, device):
        """(seg_type fp32 [B, 1] on the device, type_token_cls, type_token_ins) for SegGPT; Painter has no type tokens."""
        return None, None, None

    def _type_emb(self, B, seg_type, device):
        st, cls, ins = self._type_inputs(B, seg_type, device)
        return None if st is None else engine.type_embedding(st, cls.detach(), ins.detach())

    def _ensemble(self, i, B, merge_between_batch, prompts_per_query, merge_idx=2):
        """(groups, members) of the SegGPT prompt ensemble at block i (models_seggpt.py:220-231,:425-429); (0, 0) =
        none.  By default the ensemble averages over the whole batch, as the reference does.  With prompts_per_query
        = P the batch holds B / P queries of P prompts each, query-major ([Q][P], so [2][Q][P] before the early
        merge), and each query averages over its own P members only."""
        if merge_between_batch < 0 or i < merge_between_batch:
            return 0, 0
        P = B if prompts_per_query is None else prompts_per_query
        if P < 1 or B % P != 0:
            raise ValueError(f"painter_b200: prompts_per_query {P} does not divide the batch {B}")
        return (2 * (B // P), P) if merge_idx >= i else (B // P, P)

    def _run(self, imgs, tgts, bool_masked_pos, valid, seg_type=None, merge_between_batch=-1,
             prompts_per_query=None):
        if not imgs.is_cuda:
            raise RuntimeError("painter_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        if valid is None:
            raise ValueError("valid must be given (the reference forward_loss multiplies by it, models_painter.py:450)")
        p = self.patch_size
        B, _, H, W = imgs.shape
        h, w = H // p, W // p
        N, C = h * w, self.embed_dim
        dev = imgs.device
        # imgs and tgts are differentiable inputs, as in the reference (prompt tuning learns them with every weight
        # frozen); valid and bool_masked_pos are loss weights and a mask, not differentiable
        imgs = imgs.float().contiguous()
        tgts = tgts.float().contiguous()
        valid = valid.detach().float().contiguous()
        if valid.shape != tgts.shape:
            valid = valid.expand_as(tgts).contiguous()
        mask_u8 = bool_masked_pos.reshape(-1, N).to(torch.uint8).contiguous()
        assert mask_u8.shape[0] in (1, B), "bool_masked_pos must have batch 1 or B"
        prec = self.precision
        if prec not in ("auto", "bf16", "fp32"):
            raise ValueError(f"painter_b200: precision must be 'auto', 'bf16' or 'fp32', got {prec!r}")
        from . import accurate
        if accurate.selected(self):
            if self.training and any(b.drop_prob > 0 for b in self.blocks):
                raise NotImplementedError("painter_b200: the fp32-accurate mode is an inference mode (call .eval())")
            return accurate.forward(self, imgs.detach(), tgts.detach(), mask_u8, valid,
                                    self._type_emb(B, seg_type, dev), merge_between_batch, prompts_per_query)
        # gradient arena + per-step token (engine.StageEnv): the arena only when this forward can be followed by a
        # backward that produces parameter gradients.  A fully frozen module (e.g. for prompt tuning) has none, and
        # drops the arena of an earlier training phase.
        trainable = any(q.requires_grad for q in self.parameters())
        if not trainable:
            self.__dict__.pop("_pk_arena", None)
        arena = get_arena(self) if torch.is_grad_enabled() and trainable else None
        link = engine.StepLink() if torch.is_grad_enabled() else None   # the block backwards' hand-off
        token = object()

        def env(name, prm, below=None):
            return StageEnv(arena, token, name, prm, below, link) if link is not None else None

        stages = self.grad_stages()
        emb = stages["embed"]
        st, _, _ = self._type_inputs(B, seg_type, dev)
        z = EmbedFn.apply(imgs, tgts, mask_u8, st, *(emb.get(r) for r in EmbedFn.ROLES), p,
                          self.pretrain_use_cls_token, env("embed", emb))
        merge_idx = 2
        Bp = 2 * B
        taps = []
        self._step_drops = self._draw_drop_scales(B, dev)
        drops = [self._drop_scales(i, 2 * B if i <= merge_idx else B, dev) for i in range(len(self.blocks))]
        for i, blk in enumerate(self.blocks):
            ws = blk.window_size
            if ws > 0 and 112 % ws != 0:
                raise NotImplementedError(f"painter_b200: window_size {ws} unsupported (must divide 112: 2,4,7,8,14,28)")
            ens_g, ens_p = self._ensemble(i, B, merge_between_batch, prompts_per_query, merge_idx)
            da, dm = drops[i]
            prm = stages[f"block{i}"]
            prm["rel_h"] = engine.resize_rel_table(prm["rel_h"], ws if ws > 0 else h)
            prm["rel_w"] = engine.resize_rel_table(prm["rel_w"], ws if ws > 0 else w)
            # hand-off: block i's dx is consumed only by block i-1's MLP branch (as bf16(DropPath scale * dx)) unless
            # block i-1's output also feeds the early merge or a decoder tap
            below = None
            if i > 0 and (i - 1) != merge_idx and (i - 1) not in (5, 11, 17, 23) and ens_g == 0:
                below = (self.blocks[i - 1].mlp.fc2.bias, drops[i - 1][1], N)
            z = BlockFn.apply(z, da, dm, *prm.values(), (Bp, h, w, self.num_heads, blk.norm1.eps, ens_g, ens_p, ws),
                              env(f"block{i}", prm, below))
            if i == merge_idx:
                z = MergeFn.apply(z)
                Bp = B
            if i in (5, 11, 17, 23):
                taps.append(z)
        dec = stages["decoder"]
        loss, patch = DecoderFn.apply(*taps, tgts, *dec.values(), mask_u8, valid,
                                      (B, h, w, p, self.norm.eps, engine.LOSS_KINDS[self.loss_func], self.seggpt),
                                      env("decoder", dec))
        return loss.reshape(()), patch

    def forward(self, imgs, tgts, bool_masked_pos=None, valid=None):
        if bool_masked_pos is None:
            bool_masked_pos = torch.zeros((imgs.shape[0], self.patch_embed.num_patches), dtype=torch.bool,
                                          device=imgs.device)
        else:
            bool_masked_pos = bool_masked_pos.flatten(1).to(torch.bool)
        loss, pred = self._run(imgs, tgts, bool_masked_pos, valid)
        return loss, pred, bool_masked_pos


def painter_vit_large_patch16_input896x448_win_dec64_8glb_sl1(**kwargs):
    model = Painter(
        img_size=(896, 448), patch_size=16, embed_dim=1024, depth=24, num_heads=16,
        drop_path_rate=0.1, window_size=14, qkv_bias=True,
        mlp_ratio=4, norm_layer=partial(nn.LayerNorm, eps=1e-6),
        # kept verbatim from the reference factory (models_painter.py:481-482): a tuple of four lists, which
        # makes every block global-attention; the released checkpoints have the matching rel-pos shapes.
        window_block_indexes=(list(range(0, 2)) + list(range(3, 5)) + list(range(6, 8)) + list(range(9, 11)) +
                              list(range(12, 14)), list(range(15, 17)), list(range(18, 20)), list(range(21, 23))),
        residual_block_indexes=[], use_rel_pos=True, out_feature="last_feat",
        decoder_embed_dim=64,
        loss_func="smoothl1",
        **kwargs)
    return model
