"""Windowed attention blocks in inference: the fused fp32-accurate window-attention kernel (pk_attn_fwd_split3), the
fp32-accurate windowed Painter / SegGPT forward, and the SegGPT prompt ensemble inside windowed blocks (fp32 and
bf16), against fp64 restatements, golden vectors of the unmodified reference and the live reference."""
import types

import numpy as np
import pytest
import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs

from _common import build_model, load_golden, rel_max, rel_rms
from _refmods import build_reference, have_reference, strict_fp32

pytestmark = pytest.mark.gpu
TOL = 1e-5
LOSS_TOL, LOGIT_RMS = 1e-3, 1.5e-2        # the bf16 tolerances of test_gpu_model.test_seggpt_tiny_prompts_and_ensemble
WINDOWS_16 = (0, 1, 3, 4, 6, 7, 9, 10, 12, 13, 15, 16, 18, 19, 21, 22)   # 16 windowed + 8 global blocks


def _attn64(qkv, th, tw, B, heads, h, w):
    """fp64 restatement of models_painter.py:73-86 + vitdet_utils.py:96-125 on qkv [B*N, 3C]: (q * 0.125) k^T + rel_h
    + rel_w (on the unscaled q), softmax, . v; returns [B*N, C]."""
    N, C = h * w, heads * 64
    q, k, v = qkv.double().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    dev = qkv.device
    Rh = th.double()[torch.arange(h, device=dev)[:, None] - torch.arange(h, device=dev)[None, :] + h - 1]
    Rw = tw.double()[torch.arange(w, device=dev)[:, None] - torch.arange(w, device=dev)[None, :] + w - 1]
    out = torch.empty((B, N, heads, 64), dtype=torch.float64, device=dev)
    for b in range(B):
        rq = q[b].reshape(heads, h, w, 64)
        rel_h = torch.einsum("nhwc,hkc->nhwk", rq, Rh)
        rel_w = torch.einsum("nhwc,wkc->nhwk", rq, Rw)
        s = ((q[b] * 0.125) @ k[b].transpose(-1, -2)).reshape(heads, h, w, h, w)
        s = (s + rel_h[..., :, None] + rel_w[..., None, :]).reshape(heads, N, N)
        out[b] = (s.softmax(-1) @ v[b]).permute(1, 0, 2)
    return out.reshape(B * N, C)


def _materialised(qkv, th, tw, B, heads, h, w):
    """accurate.attention (score matrix per (window, head)) on the same qkv: an identity qkv projection reproduces it."""
    from painter_b200 import accurate
    C3 = qkv.shape[1]
    lin = types.SimpleNamespace(weight=torch.nn.Parameter(torch.eye(C3, device=qkv.device)),
                                bias=torch.zeros(C3, device=qkv.device))
    blk = types.SimpleNamespace(attn=types.SimpleNamespace(qkv=lin))
    return accurate.attention(qkv, blk, B, h, w, heads, {}, th, tw)


@pytest.mark.parametrize("B,heads,h,w", [(16, 16, 14, 14), (4, 2, 7, 7), (2, 2, 8, 8), (1, 4, 28, 28), (8, 2, 2, 2),
                                         (2, 16, 56, 28), (3, 2, 1, 1), (2, 2, 4, 4), (2, 2, 16, 16),
                                         (1, 2, 56, 56)])
def test_split3_attention_vs_fp64(B, heads, h, w):
    from painter_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + h * 10 + w)
    N, C = h * w, heads * 64
    qkv = torch.randn(B * N, 3 * C, generator=g).cuda()
    th = (torch.randn(2 * h - 1, 64, generator=g) * 0.1).cuda()
    tw = (torch.randn(2 * w - 1, 64, generator=g) * 0.1).cuda()
    ref = _attn64(qkv, th, tw, B, heads, h, w)
    out = ops.attn_fwd_split3(qkv, th, tw, B, heads, h, w)
    mat = _materialised(qkv, th, tw, B, heads, h, w)
    torch.cuda.synchronize()
    e = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    em = ((mat.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"B={B} heads={heads} {h}x{w}: fused {e:.3e}  materialised {em:.3e}")
    assert e <= TOL, (e, em)
    assert e <= 2 * em, (e, em)


def _tiny_window_painter_inputs(gold):
    cfg = po.PainterConfig(**gold["cfg"])
    return cfg, [t.cuda() for t in synth_inputs(cfg, **gold["inputs"])]


@pytest.mark.parametrize("precision", ["auto", "fp32"])
def test_painter_tiny_window_fp32_mode(precision):
    """The eval section of painter_tiny_window.pt (ws = 7 pads the 8x4 grid to 14x7): under no_grad "auto" selects the
    fp32-accurate mode, "fp32" forces it."""
    gold = load_golden("painter_tiny_window.pt")
    cfg, (imgs, tgts, mask, valid) = _tiny_window_painter_inputs(gold)
    model, _ = build_model(cfg, gold["weight_seed"], precision=precision)
    model.eval()
    assert sorted({b.window_size for b in model.blocks}) == [0, 7]
    with torch.no_grad():
        loss, pred, _ = model(imgs, tgts, mask, valid)
    ev = gold["eval"]
    le = abs(loss.item() - ev["loss"].item()) / abs(ev["loss"].item())
    pe = rel_max(pred, ev["pred"])
    print(precision, "loss rel", le, "pred max-rel", pe)
    assert le <= TOL and pe <= TOL, (le, pe)


def _seggpt_window():
    gold = load_golden("seggpt_tiny_window.pt")
    cfg = po.PainterConfig(**gold["cfg"])
    model, _ = build_model(cfg, gold["weight_seed"], precision="auto")
    model.eval()
    assert sorted({b.window_size for b in model.blocks}) == [0, 7]
    return gold, cfg, model


def _seggpt_args(cfg, c):
    h, w = cfg.grid
    x, t, _, _ = synth_inputs(cfg, c["P"], c["seed"])
    bm = torch.zeros(1, h * w)
    bm[:, h * w // 2:] = 1
    seg = torch.full((c["P"], 1), float(c["seg_type"]))
    return x.cuda(), t.cuda(), bm.cuda(), torch.ones_like(t).cuda(), seg.cuda(), c["merge_between_batch"]


def test_seggpt_tiny_window_ensemble_fp32_and_bf16():
    """Every case of seggpt_tiny_window.pt: one prompt, the ensemble over 2 / 3 prompts from block 0 (windowed blocks
    before the early merge) and from block 4 on; fp32-accurate mode to 1e-5, bf16 under autocast to the bf16 bars."""
    gold, cfg, model = _seggpt_window()
    for c in gold["cases"]:
        args = _seggpt_args(cfg, c)
        with torch.no_grad():
            loss, pred, _ = model(*args)
        le = abs(loss.item() - c["loss"].item()) / abs(c["loss"].item())
        pe = rel_max(pred, c["pred"])
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            loss_b, pred_b, _ = model(*args)
        lb = abs(loss_b.item() - c["loss"].item()) / abs(c["loss"].item())
        pb = rel_rms(pred_b, c["pred"])
        print(f"P={c['P']} merge={c['merge_between_batch']}: fp32 loss {le:.2e} pred {pe:.2e}; "
              f"bf16 loss {lb:.2e} pred rms {pb:.2e}")
        assert le <= TOL and pe <= TOL, (c["P"], c["merge_between_batch"], le, pe)
        assert lb <= LOSS_TOL and pb <= LOGIT_RMS, (c["P"], c["merge_between_batch"], lb, pb)


def test_seggpt_tiny_window_graph_replay_matches_eager_denorm():
    """seggpt_engine.run_one_image replays the forward as a CUDA graph; with P = 2 it runs the windowed blocks with the
    ensemble in the fp32-accurate mode.  Same result as an eager forward + a one-sample denorm_bottom_batched."""
    from painter_b200 import seggpt_engine
    gold, cfg, model = _seggpt_window()
    model.seg_type = "semantic"
    x, t, _, _ = synth_inputs(cfg, 2, 31)
    img = np.ascontiguousarray(x.permute(0, 2, 3, 1).double().numpy())
    tgt = np.ascontiguousarray(t.permute(0, 2, 3, 1).double().numpy())
    out_g = seggpt_engine.run_one_image(img, tgt, model, "cuda")
    out_g2 = seggpt_engine.run_one_image(img, tgt, model, "cuda")     # a second replay of the captured graph
    h, w = cfg.grid
    p = cfg.patch_size
    bm = torch.zeros(1, h * w, device="cuda")
    bm[:, h * w // 2:] = 1
    with torch.no_grad():
        _, y, _ = model(x.cuda(), t.cuda(), bm, torch.ones_like(t).cuda(), torch.zeros(2, 1, device="cuda"), 0)
        out_e, _ = seggpt_engine.denorm_bottom_batched(y, 1, h, w, p)
    out_e = out_e[0].cpu()
    tol = 1e-6 * out_e.abs().max().item()
    assert (out_g - out_e).abs().max().item() <= tol
    assert (out_g2 - out_e).abs().max().item() <= tol


@pytest.mark.skipif(not have_reference(), reason="reference tree not staged")
def test_seggpt_vitl_window_run_one_image_fp32_vs_reference():
    """SegGPT ViT-L with window_size 14 and a flat list of 16 windowed blocks, through the UNMODIFIED
    seggpt_engine.run_one_image: the module in its default precision against the reference in strict fp32."""
    from oracle import ref_loader
    se = ref_loader.seggpt_engine()
    cfg = po.PainterConfig(seggpt=True, window_size=14, window_block_indexes=WINDOWS_16)
    dev = torch.device("cuda")
    ref = build_reference(cfg, 4).eval()
    model, _ = build_model(cfg, 4, precision="auto")
    model.eval()
    assert [b.window_size for b in model.blocks] == [14 if i in WINDOWS_16 else 0 for i in range(24)]
    assert [b.window_size for b in ref.blocks] == [14 if i in WINDOWS_16 else 0 for i in range(24)]
    rep = {}
    for P, seg in ((1, "instance"), (2, "semantic")):
        x, t, _, _ = synth_inputs(cfg, P, 60 + P)
        img = np.ascontiguousarray(x.permute(0, 2, 3, 1).double().numpy())
        tgt = np.ascontiguousarray(t.permute(0, 2, 3, 1).double().numpy())
        ref.seg_type = model.seg_type = seg
        with strict_fp32():
            out_f = se.run_one_image(img, tgt, ref, dev)
        out_o = se.run_one_image(img, tgt, model, dev)
        err = ((out_o - out_f).abs().max() / 255.0).item()
        rep[f"P{P}_{seg}"] = err
        assert np.isfinite(err)
    print(rep)
    assert all(e <= TOL for e in rep.values()), rep
