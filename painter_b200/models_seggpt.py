"""H100-native drop-in for the reference `SegGPT` module (SegGPT/SegGPT_inference/models_seggpt.py:241-494):
Painter plus seg-type tokens (:285-286,:414-420), the multi-prompt feature ensemble (:220-231,:425-429) and the
loss without the ignore test (:448-469).  `forward(imgs, tgts, bool_masked_pos, valid, seg_type,
merge_between_batch)` keeps the positional order used by seggpt_engine.run_one_image (:47)."""
from functools import partial

import torch
import torch.nn as nn

from .models_painter import Painter


class SegGPT(Painter):
    seggpt = True

    def _extra_tokens(self, embed_dim):
        self.type_token_cls = nn.Parameter(torch.zeros(1, 1, 1, embed_dim))
        self.type_token_ins = nn.Parameter(torch.zeros(1, 1, 1, embed_dim))

    def _init_extra_tokens(self):
        torch.nn.init.normal_(self.type_token_cls, std=.02)
        torch.nn.init.normal_(self.type_token_ins, std=.02)

    def _type_inputs(self, B, seg_type, device):
        # models_seggpt.py:415-420: seg_type 0 selects type_token_cls, 1 type_token_ins, anything else neither; the
        # tokens are autograd inputs of the embedding (engine.EmbedFn), which reduces their gradients on the device
        st = seg_type.reshape(B, 1).to(device=device, dtype=torch.float32)
        return st, self.type_token_cls, self.type_token_ins

    def forward(self, imgs, tgts, bool_masked_pos=None, valid=None, seg_type=None, merge_between_batch=-1):
        if bool_masked_pos is None:
            bool_masked_pos = torch.zeros((imgs.shape[0], self.patch_embed.num_patches), dtype=torch.bool,
                                          device=imgs.device)
        else:
            bool_masked_pos = bool_masked_pos.flatten(1).to(torch.bool)
        loss, pred = self._run(imgs, tgts, bool_masked_pos, valid, seg_type, merge_between_batch)
        return loss, pred, bool_masked_pos


def seggpt_vit_large_patch16_input896x448(**kwargs):
    model = SegGPT(
        img_size=(896, 448), patch_size=16, embed_dim=1024, depth=24, num_heads=16,
        drop_path_rate=0.1, window_size=14, qkv_bias=True,
        mlp_ratio=4, norm_layer=partial(nn.LayerNorm, eps=1e-6),
        window_block_indexes=(list(range(0, 2)) + list(range(3, 5)) + list(range(6, 8)) + list(range(9, 11)) +
                              list(range(12, 14)), list(range(15, 17)), list(range(18, 20)), list(range(21, 23))),
        residual_block_indexes=[], use_rel_pos=True, out_feature="last_feat",
        decoder_embed_dim=64,
        loss_func="smoothl1",
        **kwargs)
    return model
