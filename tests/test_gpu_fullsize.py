"""GPU parity at the BENCHMARKED shapes against the UNMODIFIED reference executed on the same GPU (staged copy under
oracle/_ref, scripts/stage_reference.py), following the SURVEY.md section 8(c) protocol:

  * loss: |ours - ref| <= 1e-3 |ref| against the reference in fp32 (TF32 off) AND under torch.autocast('cuda', bf16);
  * logits / gradients: err(ours, fp32 reference) <= 1.5 x err(reference-bf16-autocast, fp32 reference), per
    tensor (RMS-rel) and globally; the measured ratios go to the parity report (_refmods.record_parity).

Covers BASELINE.json configs[1] (ViT-L 896x448, B=1 eval and B=8 train with the module's own CUDA DropPath draws),
configs[2] (SegGPT ViT-L through the unmodified seggpt_engine.run_one_image, 1 and 2 prompts), configs[4] (1792x896,
N=6272: full forward + one Block forward/backward) and the unmodified engine_train.train_one_epoch loop.
"""
import gc
import json
import types

import numpy as np
import pytest
import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs, synth_state_dict

from _common import build_model
from _refmods import (build_reference, grad_report, have_reference, max_rel, record_parity, rms_rel, run_module,
                      strict_fp32)

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_reference(), reason="reference tree not staged")]

LOSS_TOL = 1e-3          # north star: loss within 1e-3 relative of the reference
NOISE_RATIO = 1.5        # SURVEY 8(c): ours <= 1.5 x the reference's own bf16 error


def _record(name, payload):
    record_parity(name, payload)


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _cuda(*ts):
    return [t.cuda() for t in ts]


def _check_against_noise(tag, loss_o, pred_o, g_o, loss_b, pred_b, g_b, loss_f, pred_f, g_f, extra=None):
    rows, glob = grad_report(g_o, g_b, g_f)
    worst = sorted(rows, key=lambda r: -r[3])[:12]
    lo, lb = rms_rel(pred_o, pred_f), rms_rel(pred_b, pred_f)
    rep = {
        "loss": {"ours": loss_o.item(), "ref_fp32": loss_f.item(), "ref_bf16": loss_b.item(),
                 "rel_vs_fp32": abs(loss_o.item() - loss_f.item()) / abs(loss_f.item()),
                 "rel_vs_bf16": abs(loss_o.item() - loss_b.item()) / abs(loss_b.item()),
                 "ref_bf16_rel_vs_fp32": abs(loss_b.item() - loss_f.item()) / abs(loss_f.item())},
        "logits_rms_rel": {"ours": lo, "ref_bf16": lb, "ratio": lo / lb},
        "logits_max_rel": {"ours": max_rel(pred_o, pred_f), "ref_bf16": max_rel(pred_b, pred_f)},
        "grads_global_rms_rel": glob,
        "grads_tensors": len(rows),
        "grads_tensors_over_1p5": sum(1 for r in rows if r[3] > NOISE_RATIO),
        "grads_worst_ratio": [{"name": r[0], "ours": r[1], "ref_bf16": r[2], "ratio": r[3], "numel": r[4]}
                              for r in worst],
        "grads_median_ratio": float(np.median([r[3] for r in rows])),
    }
    if extra:
        rep.update(extra)
    _record(tag, rep)
    print(tag, json.dumps({k: rep[k] for k in ("loss", "logits_rms_rel", "grads_global_rms_rel",
                                                "grads_tensors_over_1p5", "grads_median_ratio")}))
    assert rep["loss"]["rel_vs_fp32"] <= LOSS_TOL and rep["loss"]["rel_vs_bf16"] <= LOSS_TOL, rep["loss"]
    assert lo <= NOISE_RATIO * lb, rep["logits_rms_rel"]
    assert glob["ratio"] <= NOISE_RATIO, glob
    bad = [(r[0], r[1], r[2]) for r in rows if r[3] > NOISE_RATIO]
    assert not bad, bad[:10]


def test_vitl_b1_eval_fwd_bwd_all_grads_vs_reference():
    """configs[1] geometry, B=1, eval: all 370.7 M gradients against the reference in fp32 and in bf16 autocast."""
    cfg = po.PainterConfig()
    args = _cuda(*synth_inputs(cfg, 1, 21, valid_kind="mixed"))
    ref = build_reference(cfg, 1, stock_factory=True)
    with strict_fp32():
        loss_f, pred_f, g_f = run_module(ref, args)
    loss_b, pred_b, g_b = run_module(ref, args, autocast=torch.bfloat16)
    del ref
    _free()
    model, _ = build_model(cfg, 1)
    loss_o, pred_o, g_o = run_module(model, args)
    del model
    _free()
    _check_against_noise("vitl_896x448_b1_eval", loss_o, pred_o, g_o, loss_b, pred_b, g_b, loss_f, pred_f, g_f)


def test_vitl_b8_train_step_vs_reference_same_cuda_rng():
    """configs[1]: B=8 TRAIN mode under torch.autocast(bf16) - the bench's GEMM plans (M = 25088 / 12544) and the
    module's own CUDA DropPath draws (same seed => the reference draws the same masks, timm DropPath order/dtype)."""
    cfg = po.PainterConfig()
    B, seed = 8, 1234
    args = _cuda(*synth_inputs(cfg, B, 5, valid_kind="mixed"))
    # --- ours, recording the DropPath scales the module drew on the device ---
    model, sd = build_model(cfg, 2)
    drawn = {}
    orig = model._drop_scales

    def rec(i, Bp, dev):
        out = orig(i, Bp, dev)
        drawn[i] = out
        return out

    model._drop_scales = rec
    loss_o, pred_o, g_o = run_module(model, args, train=True, autocast=torch.bfloat16, seed=seed)
    del model
    _free()
    # --- the unmodified reference module, bf16 autocast, same CUDA RNG seed ---
    ref = build_reference(cfg, 2, stock_factory=True)
    loss_b, pred_b, g_b = run_module(ref, args, train=True, autocast=torch.bfloat16, seed=seed)
    del ref
    _free()
    # --- fp32 truth: the (pinned) oracle restatement on CUDA in strict fp32 with the recorded masks ---
    drops = []
    for i in range(cfg.depth):
        Bp = 2 * B if i <= cfg.merge_idx else B
        a, m = drawn[i]
        one = torch.ones(Bp, device="cuda")
        drops.append((one if a is None else a.float(), one if m is None else m.float()))
    sdc = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
    with strict_fp32():
        loss_f, pred_f, _ = po.forward(sdc, cfg, *args, drops=drops)
        loss_f.backward()
    g_f = {k: v.grad.detach() for k, v in sdc.items()}
    loss_f, pred_f = loss_f.detach(), pred_f.detach()
    n_dropped = int(sum((d[0] == 0).sum().item() + (d[1] == 0).sum().item() for d in drops))
    _check_against_noise("vitl_896x448_b8_train", loss_o, pred_o, g_o, loss_b, pred_b, g_b, loss_f, pred_f, g_f,
                         extra={"droppath_branches_dropped": n_dropped})
    assert n_dropped > 0, "DropPath never fired: the train-mode path was not exercised"


def test_seggpt_vitl_run_one_image_unmodified_engine():
    """configs[2]: seggpt_engine.run_one_image (UNMODIFIED, seggpt_engine.py:26-53) drives the painter_b200 SegGPT
    module and the reference module on the same numpy inputs: 1 prompt (no ensemble) and 2 prompts (feature ensemble),
    both seg types."""
    from oracle import ref_loader
    se = ref_loader.seggpt_engine()
    cfg = po.PainterConfig(seggpt=True)
    dev = torch.device("cuda")
    ref = build_reference(cfg, 3, stock_factory=True).eval()
    model, _ = build_model(cfg, 3)
    model.eval()
    rep = {}
    for P, seg in ((1, "instance"), (2, "semantic")):
        x, t, _, _ = synth_inputs(cfg, P, 40 + P)
        img = x.permute(0, 2, 3, 1).double().numpy()
        tgt = t.permute(0, 2, 3, 1).double().numpy()
        ref.seg_type = model.seg_type = seg
        with strict_fp32():
            out_f = se.run_one_image(img, tgt, ref, dev)
        # the reference's own bf16 noise: run_one_image cannot run under autocast (numpy cannot take its bf16 result),
        # so the same call sequence (seggpt_engine.py:29-52) is restated around the reference MODULE for this one
        # measurement
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            bm = torch.zeros(1, ref.patch_embed.num_patches)
            bm[:, ref.patch_embed.num_patches // 2:] = 1
            xt, tt = torch.tensor(img).permute(0, 3, 1, 2), torch.tensor(tgt).permute(0, 3, 1, 2)
            sgt = torch.ones(P, 1) if seg == "instance" else torch.zeros(P, 1)
            _, yb, _ = ref(xt.float().to(dev), tt.float().to(dev), bm.to(dev), torch.ones_like(tt).float().to(dev),
                           sgt.to(dev), 0 if P > 1 else -1)
        yb = ref.unpatchify(yb.float()).permute(0, 2, 3, 1).cpu()
        out_b = torch.clip((yb[0, yb.shape[1] // 2:] * se.imagenet_std + se.imagenet_mean) * 255, 0, 255)
        out_o = se.run_one_image(img, tgt, model, dev)
        assert tuple(out_o.shape) == tuple(out_f.shape) == (448, 448, 3) and out_o.dtype == out_f.dtype
        eo, eb = rms_rel(out_o, out_f), rms_rel(out_b, out_f)
        rep[f"P{P}_{seg}"] = {"rms_rel_ours": eo, "rms_rel_ref_bf16": eb, "ratio": eo / eb,
                              "max_abs_ours_of_255": (out_o - out_f).abs().max().item(),
                              "max_abs_ref_bf16_of_255": (out_b - out_f).abs().max().item()}
        assert eo <= NOISE_RATIO * eb, rep
    _record("seggpt_vitl_run_one_image", rep)
    print(rep)


def test_long_sequence_1792x896_forward_and_block_backward():
    """configs[4]: Painter(img_size=(1792, 896)) - N = 6272 tokens, native 223/111-row tables: full forward B=1 and
    a single Block forward/backward at N = 6272 (SURVEY 8c: the full backward oracle does not fit)."""
    from oracle import ref_loader
    cfg = po.PainterConfig(img_size=(1792, 896))
    args = _cuda(*synth_inputs(cfg, 1, 77))
    ref = build_reference(cfg, 4).eval()
    with torch.no_grad():
        with strict_fp32():
            loss_f, pred_f, _ = run_module(ref, args, backward=False)
        loss_b, pred_b, _ = run_module(ref, args, autocast=torch.bfloat16, backward=False)
    del ref
    _free()
    model, sd = build_model(cfg, 4)
    model.eval()
    with torch.no_grad():
        loss_o, pred_o, _ = run_module(model, args, backward=False)
    rep = {"loss_rel_vs_fp32": abs(loss_o.item() - loss_f.item()) / abs(loss_f.item()),
           "loss_rel_vs_bf16": abs(loss_o.item() - loss_b.item()) / abs(loss_b.item()),
           "logits_rms_rel": {"ours": rms_rel(pred_o, pred_f), "ref_bf16": rms_rel(pred_b, pred_f)}}
    assert rep["loss_rel_vs_fp32"] <= LOSS_TOL and rep["loss_rel_vs_bf16"] <= LOSS_TOL, rep
    assert rep["logits_rms_rel"]["ours"] <= NOISE_RATIO * rep["logits_rms_rel"]["ref_bf16"], rep
    # ---- one Block at N = 6272, batch 2 (the x / y halves), forward + backward ----
    from painter_b200.engine import BlockFn
    h, w = cfg.grid
    C = cfg.embed_dim
    blk = model.blocks[7]
    g = torch.Generator().manual_seed(5)
    z0 = torch.randn(2, h, w, C, generator=g).cuda()
    dz = torch.randn(2, h, w, C, generator=g).cuda()
    mp = ref_loader.models_painter()
    rb = mp.Block(dim=C, num_heads=cfg.num_heads, mlp_ratio=4, qkv_bias=True, drop_path=0.0,
                  norm_layer=lambda d: torch.nn.LayerNorm(d, eps=1e-6), use_rel_pos=True, window_size=0,
                  input_size=(h, w)).cuda()
    rb.load_state_dict({k[len("blocks.7."):]: v for k, v in sd.items() if k.startswith("blocks.7.")}, strict=True)

    def ref_block(autocast):
        for p in rb.parameters():
            p.grad = None
        zin = z0.clone().requires_grad_(True)
        if autocast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                out = rb(zin)
        else:
            with strict_fp32():
                out = rb(zin)
        out.float().backward(dz)
        gr = {"blocks.7." + n: p.grad.detach().float().clone() for n, p in rb.named_parameters()}
        gr["dx"] = zin.grad.detach().clone()
        return out.detach().float(), gr

    out_f, g_f = ref_block(False)
    out_b, g_b = ref_block(True)
    del rb
    _free()
    for p in model.parameters():
        p.grad = None
    zin = z0.reshape(2 * h * w, C).clone().requires_grad_(True)
    prm = blk.params()
    out_o = BlockFn.apply(zin, None, None, *prm, (2, h, w, cfg.num_heads, 1e-6, 0, 0, 0))
    out_o.backward(dz.reshape(2 * h * w, C))
    g_o = {"blocks.7." + n: p.grad.detach().float().clone() for n, p in blk.named_parameters()}
    g_o["dx"] = zin.grad.detach().reshape(2, h, w, C)
    rows, glob = grad_report(g_o, g_b, g_f)
    rep["block_out_rms_rel"] = {"ours": rms_rel(out_o.reshape(2, h, w, C), out_f), "ref_bf16": rms_rel(out_b, out_f)}
    rep["block_grads_global"] = glob
    rep["block_grads"] = [{"name": r[0], "ours": r[1], "ref_bf16": r[2], "ratio": r[3]} for r in rows]
    _record("long_1792x896", rep)
    print(json.dumps(rep["block_grads_global"]), rep["block_out_rms_rel"])
    assert rep["block_out_rms_rel"]["ours"] <= NOISE_RATIO * rep["block_out_rms_rel"]["ref_bf16"], rep
    assert glob["ratio"] <= NOISE_RATIO, glob
    bad = [(r[0], r[1], r[2]) for r in rows if r[3] > NOISE_RATIO]
    assert not bad, bad


def test_stock_weights_on_double_resolution_input_interpolated_tables():
    """SURVEY 8(d) config 5 variant: the stock 896x448 model fed a 1792x896 canvas (rel-pos tables linearly resized
    111 -> 223 / 55 -> 111 rows, abs-pos bicubic 14x14 -> 112x56; vitdet_utils.py:75-86,141-153)."""
    cfg = po.PainterConfig()
    args = _cuda(*synth_inputs(cfg, 1, 78, size=(1792, 896)))
    ref = build_reference(cfg, 5, stock_factory=True).eval()
    with torch.no_grad():
        with strict_fp32():
            loss_f, pred_f, _ = run_module(ref, args, backward=False)
        loss_b, pred_b, _ = run_module(ref, args, autocast=torch.bfloat16, backward=False)
    del ref
    _free()
    model, _ = build_model(cfg, 5)
    model.eval()
    with torch.no_grad():
        loss_o, pred_o, _ = run_module(model, args, backward=False)
    rep = {"loss_rel_vs_fp32": abs(loss_o.item() - loss_f.item()) / abs(loss_f.item()),
           "logits_rms_rel": {"ours": rms_rel(pred_o, pred_f), "ref_bf16": rms_rel(pred_b, pred_f)}}
    _record("stock_weights_1792x896_input", rep)
    assert rep["loss_rel_vs_fp32"] <= LOSS_TOL, rep
    assert rep["logits_rms_rel"]["ours"] <= NOISE_RATIO * rep["logits_rms_rel"]["ref_bf16"], rep


def _train_args():
    return types.SimpleNamespace(accum_iter=1, clip_grad=3.0, lr=1e-4, min_lr=0.0, warmup_epochs=0, epochs=15,
                                 log_wandb=False)


def test_unmodified_train_one_epoch_drives_the_module():
    """engine_train.train_one_epoch (UNMODIFIED, engine_train.py:34-144: fp16 autocast context, loss.item(),
    NativeScalerWithGradNormCount -> GradScaler / clip_grad_norm_ / AdamW, torch.cuda.synchronize, MetricLogger) runs
    against the painter_b200 module exactly as against the reference module, on the same loader and RNG seeds."""
    from oracle import ref_loader
    et, misc = ref_loader.engine_train(), ref_loader.misc()
    lrd = ref_loader.lr_decay()
    cfg = po.PainterConfig()
    dev = torch.device("cuda")
    loader = [tuple(t.pin_memory() for t in synth_inputs(cfg, 2, 90 + i)) for i in range(2)]

    def drive(m):
        groups = lrd.param_groups_lrd(m, 0.05, no_weight_decay_list=m.no_weight_decay(), layer_decay=0.8)
        opt = torch.optim.AdamW(groups, lr=1e-4, betas=(0.9, 0.999))
        scaler = misc.NativeScalerWithGradNormCount()
        out = []
        for epoch in range(2):
            torch.manual_seed(700 + epoch)
            stats = et.train_one_epoch(m, loader[epoch:epoch + 1], opt, dev, epoch, scaler, log_writer=None,
                                       global_rank=0, args=_train_args())
            out.append(stats)
        return out

    ref = build_reference(cfg, 6, stock_factory=True)
    s_ref = drive(ref)
    del ref
    _free()
    model, _ = build_model(cfg, 6)
    s_our = drive(model)
    rep = {"ref": s_ref, "ours": s_our}
    _record("train_one_epoch_unmodified", rep)
    print(rep)
    for a, b in zip(s_our, s_ref):
        assert np.isfinite(a["loss"]) and np.isfinite(a["grad_norm"])
    # iteration 0: same weights, same batch, same DropPath draws -> same loss and gradient norm
    assert abs(s_our[0]["loss"] - s_ref[0]["loss"]) <= LOSS_TOL * abs(s_ref[0]["loss"]), rep
    if np.isfinite(s_ref[0]["grad_norm"]):   # the reference's fp16 backward may overflow at the initial loss scale
        assert abs(s_our[0]["grad_norm"] - s_ref[0]["grad_norm"]) <= 2e-2 * abs(s_ref[0]["grad_norm"]), rep
    # iteration 1 runs on the AdamW-updated weights (first Adam step ~ lr * sign(g): amplifies rounding differences)
    assert abs(s_our[1]["loss"] - s_ref[1]["loss"]) <= 1e-2 * abs(s_ref[1]["loss"]), rep
