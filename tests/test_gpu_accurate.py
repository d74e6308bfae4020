"""GPU parity of the fp32-ACCURATE mode (north star: 1e-5 in fp32; SURVEY.md section 8c "fp32 mode": loss rel <= 1e-5,
logits max|d| / max|ref| <= 1e-5) against golden vectors of the unmodified reference (CPU fp32) and against the
unmodified reference executed on the GPU in strict fp32 (TF32 off)."""
import pytest
import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs

from _common import build_model, load_golden, rel_max
from _refmods import build_reference, have_reference, max_rel, record_parity, run_module, strict_fp32

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _to(dev, *ts):
    return [t.to(dev) for t in ts]


def test_split_gemm_matches_fp64_matmul():
    """The building block: one pk_gemm_bf16 over [l|m|h|m|h|h] x [h|m|l|h|m|h] operands == fp32 GEMM to ~1e-6."""
    from painter_b200 import accurate
    from painter_b200.ops import EPI_F32
    g = torch.Generator().manual_seed(0)
    for M, N, K in ((300, 192, 256), (1568, 1024, 1024), (1568, 3072, 4096)):
        a = torch.randn(M, K, generator=g).cuda()
        b = (torch.randn(N, K, generator=g) * 0.05).cuda()
        bias = torch.randn(N, generator=g).cuda()
        out = accurate._gemm(accurate.split3(a), accurate.split3(b, side_b=True), kind=EPI_F32, bias=bias)
        want = (a.double() @ b.double().t() + bias.double())
        e32 = max_rel(a @ b.t() + bias, want) if True else 0.0
        e = max_rel(out, want)
        print(M, N, K, "split", e, "torch fp32 (may use TF32)", e32)
        assert e < 1e-5, (M, N, K, e)     # fp32 accumulation over K' = 6K terms; measured 1e-6 .. 5e-6


def test_painter_tiny_golden_fp32_mode():
    gold = load_golden("painter_tiny.pt")
    cfg = po.PainterConfig(**gold["cfg"])
    model, _ = build_model(cfg, gold["weight_seed"], precision="fp32")
    model.eval()
    imgs, tgts, mask, valid = _to("cuda", *synth_inputs(cfg, **gold["inputs"]))
    with torch.no_grad():
        loss, pred, _ = model(imgs, tgts, mask, valid)
    ev = gold["eval"]
    assert abs(loss.item() - ev["loss"].item()) <= TOL * abs(ev["loss"].item()), (loss.item(), ev["loss"].item())
    assert rel_max(pred, ev["pred"]) <= TOL, rel_max(pred, ev["pred"])
    it = gold["interp"]          # 64x32 input on the 128x64 model: interpolated abs-pos / rel-pos tables
    i2, t2, mk2, v2 = _to("cuda", *synth_inputs(cfg, **it["inputs"]))
    with torch.no_grad():
        loss, pred, _ = model(i2, t2, mk2, v2)
    assert abs(loss.item() - it["loss"].item()) <= TOL * abs(it["loss"].item())
    assert rel_max(pred, it["pred"]) <= TOL, rel_max(pred, it["pred"])


def test_seggpt_tiny_golden_fp32_mode_auto_selected():
    """precision = "auto": called outside autocast under no_grad (as seggpt_engine.run_one_image does) the module
    computes in the fp32-accurate mode; prompts 1/2/3 incl. the feature ensemble and both seg types."""
    gold = load_golden("seggpt_tiny.pt")
    cfg = po.PainterConfig(**gold["cfg"])
    model, _ = build_model(cfg, gold["weight_seed"], precision="auto")
    model.eval()
    h, w = cfg.grid
    for c in gold["cases"]:
        x, t, _, _ = synth_inputs(cfg, c["P"], c["seed"])
        bm = torch.zeros(1, h * w)
        bm[:, h * w // 2:] = 1
        seg = torch.full((c["P"], 1), float(c["seg_type"]))
        with torch.no_grad():
            loss, pred, _ = model(x.cuda(), t.cuda(), bm.cuda(), torch.ones_like(t).cuda(), seg.cuda(),
                                  c["merge_between_batch"])
        assert abs(loss.item() - c["loss"].item()) <= TOL * abs(c["loss"].item()), c["P"]
        assert rel_max(pred, c["pred"]) <= TOL, (c["P"], rel_max(pred, c["pred"]))
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):     # auto -> bf16 under autocast
            _, pred_b, _ = model(x.cuda(), t.cuda(), bm.cuda(), torch.ones_like(t).cuda(), seg.cuda(),
                                 c["merge_between_batch"])
        assert 1e-4 < rel_max(pred_b, c["pred"]) < 4e-2


@pytest.mark.skipif(not have_reference(), reason="reference tree not staged")
def test_seggpt_vitl_run_one_image_fp32_mode_vs_reference_fp32():
    """configs[2] at full size through the UNMODIFIED seggpt_engine.run_one_image: the module in its default "auto"
    precision against the reference module in strict fp32 on the same GPU."""
    from oracle import ref_loader
    se = ref_loader.seggpt_engine()
    cfg = po.PainterConfig(seggpt=True)
    dev = torch.device("cuda")
    ref = build_reference(cfg, 3, stock_factory=True).eval()
    model, _ = build_model(cfg, 3, precision="auto")
    model.eval()
    rep = {}
    for P, seg in ((1, "instance"), (2, "semantic")):
        x, t, _, _ = synth_inputs(cfg, P, 40 + P)
        img = x.permute(0, 2, 3, 1).double().numpy()
        tgt = t.permute(0, 2, 3, 1).double().numpy()
        ref.seg_type = model.seg_type = seg
        with strict_fp32():
            out_f = se.run_one_image(img, tgt, ref, dev)
        out_o = se.run_one_image(img, tgt, model, dev)
        err = ((out_o - out_f).abs().max() / 255.0).item()
        rep[f"P{P}_{seg}"] = {"max_abs_err_over_255": err, "max_rel": max_rel(out_o, out_f)}
        assert err <= TOL, rep
    print(rep)
    record_parity("seggpt_vitl_run_one_image_fp32_mode", rep)


@pytest.mark.skipif(not have_reference(), reason="reference tree not staged")
def test_painter_vitl_fp32_mode_vs_reference_fp32():
    cfg = po.PainterConfig()
    args = [t.cuda() for t in synth_inputs(cfg, 1, 21, valid_kind="mixed")]
    ref = build_reference(cfg, 1, stock_factory=True).eval()
    with torch.no_grad(), strict_fp32():
        loss_f, pred_f, _ = run_module(ref, args, backward=False)
    del ref
    torch.cuda.empty_cache()
    model, _ = build_model(cfg, 1, precision="fp32")
    model.eval()
    with torch.no_grad():
        loss_o, pred_o, _ = run_module(model, args, backward=False)
    le = abs(loss_o.item() - loss_f.item()) / abs(loss_f.item())
    pe = max_rel(pred_o, pred_f)
    print("fp32 mode: loss rel", le, "logits max-rel", pe)
    assert le <= TOL and pe <= TOL, (le, pe)
