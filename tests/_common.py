"""Helpers shared by the GPU parity tests."""
import os

import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs, synth_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _merge(dst, src):
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(dst[k], v)
        else:
            dst[k] = v


def load_golden(name):
    """A golden file <stem>.pt, merged with its parts <stem>.part<i>.pt (nested dicts split so that every stored file
    stays below 1 MB)."""
    stem = name[:-3]
    gold = torch.load(os.path.join(GOLDEN, name), weights_only=False)
    parts = sorted(f for f in os.listdir(GOLDEN) if f.startswith(stem + ".part") and f.endswith(".pt"))
    for f in parts:
        _merge(gold, torch.load(os.path.join(GOLDEN, f), weights_only=False))
    return gold


def build_model(cfg: po.PainterConfig, seed, device="cuda", precision="bf16"):
    """painter_b200 module of the same geometry as `cfg`, loaded with the synthetic reference-format weights.
    precision: the module's arithmetic mode, pinned to "bf16" unless a test is about the fp32-accurate / auto modes."""
    from functools import partial
    from painter_b200 import models_painter, models_seggpt
    cls = models_seggpt.SegGPT if cfg.seggpt else models_painter.Painter
    m = cls(img_size=tuple(cfg.img_size), patch_size=cfg.patch_size, embed_dim=cfg.embed_dim, depth=cfg.depth,
            num_heads=cfg.num_heads, drop_path_rate=cfg.drop_path_rate, window_size=cfg.window_size, qkv_bias=True,
            mlp_ratio=cfg.mlp_ratio, norm_layer=partial(torch.nn.LayerNorm, eps=cfg.ln_eps),
            window_block_indexes=list(cfg.window_block_indexes), residual_block_indexes=[], use_rel_pos=True,
            out_feature="last_feat", decoder_embed_dim=cfg.decoder_embed_dim, loss_func=cfg.loss_func,
            pretrain_img_size=cfg.pretrain_img_size)
    sd = synth_state_dict(cfg, seed)
    m.load_state_dict(sd, strict=True)
    m.precision = precision
    return m.to(device), sd


def rel_max(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def rel_rms(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-12)).item()
