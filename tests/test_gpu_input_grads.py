"""Gradients for the input images and targets, and the backward that skips frozen parameters (GPU).

1. imgs.grad / tgts.grad against the unmodified reference's (tests/golden/painter_tiny_input_grads*.pt, pinned to the
   fp32 oracle by tests/test_oracle_input_grads.py): rms-rel error <= 1.5 x the reference algorithm's own
   bf16-autocast error on the same inputs (the tests/test_gpu_model.py protocol); single-prompt SegGPT against the
   fp32 oracle the same way; the SegGPT prompt ensemble still refuses its backward.
2. A fully frozen module gives the same input gradients, bit for bit, as the same module with trainable weights; it
   has no gradient arena and leaves every p.grad None.
3. Partial freezing (frozen encoder / frozen rel-pos tables and LayerNorms): the trainable gradients equal a full
   backward's to within the run-to-run differences of two full backwards; frozen p.grad stays None; stages whose
   parameters and inputs are all frozen run no backward.
4. A frozen backward runs no parameter-gradient work and saves none of the activations only that work reads (the same
   hooks see all of them saved by a trainable module); a module frozen after training drops its gradient arena.
5. Prompt tuning lowers the loss.
"""
import pytest
import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs, synth_state_dict
from painter_b200 import engine, ops

from _common import build_model, load_golden, rel_max, rel_rms

pytestmark = pytest.mark.gpu

NOISE_RATIO = 1.5
CASES = ("eval", "train", "l1", "l2", "l1l2", "blockmask", "window")
TINY = dict(img_size=(128, 64), embed_dim=128, num_heads=2, decoder_embed_dim=64, window_size=2)


@pytest.fixture(scope="module")
def gold():
    return load_golden("painter_tiny_input_grads.pt")["cases"]


def _case_inputs(c):
    cfg = po.PainterConfig(**c["cfg"])
    imgs, tgts, mask, valid = synth_inputs(cfg, **c["inputs"])
    if c["mask"] is not None:
        mask = c["mask"]
    drops = None
    if c["train_seed"] is not None:
        torch.manual_seed(c["train_seed"])
        drops = po.draw_drop_scales(cfg, imgs.shape[0])   # the reference's CPU draws, replayed
    return cfg, imgs, tgts, mask, valid, drops


def _oracle_input_grads(cfg, sd, imgs, tgts, mask, valid, drops=None, bf16=False, **kw):
    """imgs.grad, tgts.grad of the oracle on the GPU: fp32, or under bf16 autocast (the reference's own noise)."""
    sdc = {k: v.cuda() for k, v in sd.items()}
    x, t = imgs.cuda().requires_grad_(True), tgts.cuda().requires_grad_(True)
    d = None if drops is None else [tuple(a.cuda() for a in pair) for pair in drops]
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
        loss, _, _ = po.forward(sdc, cfg, x, t, mask.cuda(), valid.cuda(), drops=d, **kw)
    loss.float().backward()
    return x.grad, t.grad


def _ours(model, imgs, tgts, mask, valid, drops=None, **kw):
    if drops is not None:
        model._drop_scales = lambda i, Bp, dev: tuple(t.to(dev) for t in drops[i])
    x, t = imgs.cuda().requires_grad_(True), tgts.cuda().requires_grad_(True)
    loss, _, _ = model(x, t, mask.cuda(), valid.cuda(), **kw)
    loss.backward()
    return loss, x.grad, t.grad


@pytest.mark.parametrize("name", CASES)
def test_input_grads_vs_reference_golden(gold, name):
    c = gold[name]
    cfg, imgs, tgts, mask, valid, drops = _case_inputs(c)
    model, sd = build_model(cfg, c["weight_seed"])
    model.train(drops is not None)
    loss, dimgs, dtgts = _ours(model, imgs, tgts, mask, valid, drops)
    assert abs(loss.item() - c["loss"].item()) <= 1e-3 * abs(c["loss"].item())
    nimgs, ntgts = _oracle_input_grads(cfg, sd, imgs, tgts, mask, valid, drops, bf16=True)
    bad = []
    for what, ours, noise, ref in (("imgs", dimgs, nimgs, c["dimgs"]), ("tgts", dtgts, ntgts, c["dtgts"])):
        e, tol = rel_rms(ours, ref), NOISE_RATIO * rel_rms(noise, ref)
        print(f"{name} {what}: rms-rel ours {e:.3e}  reference-bf16 {tol / NOISE_RATIO:.3e}")
        if not e <= tol:
            bad.append((what, e, tol))
    assert not bad, bad


def test_seggpt_single_prompt_input_grads_and_ensemble_refusal():
    cfg = po.PainterConfig(**TINY, seggpt=True)
    model, sd = build_model(cfg, 5)
    model.eval()
    model.type_token_cls.requires_grad_(False)
    model.type_token_ins.requires_grad_(False)
    h, w = cfg.grid
    x, t, _, _ = synth_inputs(cfg, 1, 101)
    bm = torch.zeros(1, h * w)
    bm[:, h * w // 2:] = 1
    valid = torch.ones_like(t)
    seg = torch.full((1, 1), 1.0)
    _, dimgs, dtgts = _ours(model, x, t, bm, valid, seg_type=seg.cuda())
    fimgs, ftgts = _oracle_input_grads(cfg, sd, x, t, bm, valid, seg_type=seg.cuda())
    nimgs, ntgts = _oracle_input_grads(cfg, sd, x, t, bm, valid, bf16=True, seg_type=seg.cuda())
    for ours, noise, ref in ((dimgs, nimgs, fimgs), (dtgts, ntgts, ftgts)):
        assert rel_rms(ours, ref) <= NOISE_RATIO * rel_rms(noise, ref), (rel_rms(ours, ref), rel_rms(noise, ref))
    # the prompt ensemble (merge_between_batch >= 0) keeps refusing its backward
    x2, t2, _, _ = synth_inputs(cfg, 2, 102)
    xi, ti = x2.cuda().requires_grad_(True), t2.cuda().requires_grad_(True)
    loss, _, _ = model(xi, ti, bm.cuda(), torch.ones_like(ti), torch.zeros(2, 1).cuda(), 0)
    with pytest.raises(NotImplementedError):
        loss.backward()


def _tiny(seed=0, **kw):
    cfg = po.PainterConfig(**TINY, **kw)
    model, _ = build_model(cfg, seed)
    model.eval()
    return cfg, model


def test_frozen_input_grads_equal_full_bit_for_bit():
    cfg, full = _tiny()
    _, frozen = _tiny()
    frozen.requires_grad_(False)
    imgs, tgts, mask, valid = synth_inputs(cfg, 2, 7, valid_kind="mixed")
    _, fi, ft = _ours(full, imgs, tgts, mask, valid)
    _, zi, zt = _ours(frozen, imgs, tgts, mask, valid)
    assert torch.equal(fi, zi) and torch.equal(ft, zt), (rel_max(zi, fi), rel_max(zt, ft))
    assert getattr(frozen, "_pk_arena", None) is None
    assert all(p.grad is None for p in frozen.parameters())
    assert all(p.grad is not None for p in full.parameters())


def _full_grads(model, imgs, tgts, mask, valid):
    for p in model.parameters():
        p.grad = None
    loss, _, _ = model(imgs.cuda(), tgts.cuda(), mask.cuda(), valid.cuda())
    loss.backward()
    out = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    for p in model.parameters():
        p.grad = None
    return out


def _encoder_params(model):
    return [model.patch_embed.proj.weight, model.patch_embed.proj.bias, model.mask_token, model.segment_token_x,
            model.segment_token_y, model.pos_embed, *model.blocks.parameters()]


def _ln_and_tables(model):
    out = [model.norm.weight, model.norm.bias, model.decoder_pred[1].weight, model.decoder_pred[1].bias]
    for b in model.blocks:
        out += [b.norm1.weight, b.norm1.bias, b.norm2.weight, b.norm2.bias, b.attn.rel_pos_h, b.attn.rel_pos_w]
    return out


@pytest.mark.parametrize("freeze", ["encoder", "layernorms_and_tables"])
def test_partial_freezing_matches_full_backward(freeze, monkeypatch):
    cfg, model = _tiny()
    imgs, tgts, mask, valid = synth_inputs(cfg, 2, 13, valid_kind="mixed")
    # run-to-run reproducibility of the full backward (the stream-K weight gradients and the atomics of some
    # reductions add in a varying order): the largest difference between any two of four full backwards.  Where that
    # is below 1e-6 of the largest element (a few fp32 ulps: the head's block-reduction atomics), the bound is 1e-6,
    # because a shorter backward schedules those atomics differently from every full run.
    fulls = [_full_grads(model, imgs, tgts, mask, valid) for _ in range(4)]
    frozen = _encoder_params(model) if freeze == "encoder" else _ln_and_tables(model)
    frozen_ids = {id(p) for p in frozen}
    for p in frozen:
        p.requires_grad_(False)
    calls = {"embed": 0, "block": 0}
    emb_bwd, blk_bwd = engine.EmbedFn.backward, engine.BlockFn.backward

    def count(key, fn):
        def wrapped(ctx, *a):
            calls[key] += 1
            return fn(ctx, *a)
        return staticmethod(wrapped)

    monkeypatch.setattr(engine.EmbedFn, "backward", count("embed", emb_bwd))
    monkeypatch.setattr(engine.BlockFn, "backward", count("block", blk_bwd))
    loss, _, _ = model(imgs.cuda(), tgts.cuda(), mask.cuda(), valid.cuda())
    loss.backward()
    bad = []
    for n, p in model.named_parameters():
        if id(p) in frozen_ids:
            if p.grad is not None:
                bad.append((n, "frozen parameter got a gradient"))
            continue
        rep = max(rel_max(a[n], b[n]) for k, a in enumerate(fulls) for b in fulls[k + 1:])
        err = min(rel_max(p.grad, f[n]) for f in fulls)
        if err > max(rep, 1e-6):
            bad.append((n, err, rep))
    assert not bad, bad[:10]
    if freeze == "encoder":
        # neither the embedding nor any block has a parameter or an input that requires grad
        assert calls == {"embed": 0, "block": 0}, calls
    else:
        assert calls["block"] == len(model.blocks) and calls["embed"] == 1, calls


def _saved_activations(model, imgs, tgts, mask, valid, monkeypatch):
    """Runs one forward with imgs / tgts requiring grad.  Returns {kind: [recorded tensor saved for backward?]} for
    the tensors only parameter gradients read: u / v and the decoder's cat (LayerNorm outputs; cat through the slice
    its first tap LayerNorm writes), hact (GELU output), g (pixel-shuffle GEMM output) and cols (im2col), and the loss.
    The recorded tensors are kept alive so that their addresses cannot be reused during the forward."""
    rec = {"layernorm": [], "hact": [], "g": [], "cols": []}
    lnf, gemm, im2col = ops.layernorm_fwd, ops.gemm, ops.im2col_patch

    def ln_fwd(*a, **k):
        r = lnf(*a, **k)
        rec["layernorm"].append(r[0])
        return r

    def gemm_rec(*a, **k):
        r = gemm(*a, **k)
        if k.get("kind") == ops.EPI_GELU:
            rec["hact"].append(r[1])
        if k.get("pixshuf") is not None:
            rec["g"].append(k["pixshuf"][4])
        return r

    def im2col_rec(*a, **k):
        r = im2col(*a, **k)
        rec["cols"].append(r)
        return r

    with monkeypatch.context() as mp:
        mp.setattr(ops, "layernorm_fwd", ln_fwd)
        mp.setattr(ops, "gemm", gemm_rec)
        mp.setattr(ops, "im2col_patch", im2col_rec)
        saved = set()

        def pack(t):
            saved.add(t.data_ptr())
            return t

        x, t = imgs.cuda().requires_grad_(True), tgts.cuda().requires_grad_(True)
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            loss, _, _ = model(x, t, mask.cuda(), valid.cuda())
    assert len(rec["layernorm"]) == 2 * len(model.blocks) + 4 and len(rec["hact"]) == len(model.blocks)
    assert len(rec["g"]) == 1 and len(rec["cols"]) == 1
    return {k: [r.data_ptr() in saved for r in v] for k, v in rec.items()}, loss, x, t


def test_frozen_backward_skips_parameter_work_and_saves(monkeypatch):
    cfg, model = _tiny()
    imgs, tgts, mask, valid = synth_inputs(cfg, 2, 17, valid_kind="mixed")
    # positive control: the same hooks see every one of these activations saved by a trainable module (u and v of
    # every block and the decoder's cat; the tap LayerNorms' other slices are views of cat)
    kept, loss, _, _ = _saved_activations(model, imgs, tgts, mask, valid, monkeypatch)
    assert sum(kept["layernorm"]) == 2 * len(model.blocks) + 1, kept["layernorm"]
    assert all(kept["hact"]) and all(kept["g"]) and all(kept["cols"]), kept
    del loss
    model.requires_grad_(False)
    counts = {"wgrad": 0, "conv3x3_wgrad": 0, "colsum": 0, "affine": 0, "tables": 0, "scale_cast": 0}
    wgrad, cw, cs, lnb, ab = engine._wgrad, ops.conv3x3_wgrad, ops.colsum_bf16, ops.layernorm_bwd, ops.attn_bwd
    scc = ops.scale_cast_colsum

    def bump(key, fn):
        def wrapped(*a, **k):
            counts[key] += 1
            return fn(*a, **k)
        return wrapped

    def ln_bwd(dy, x, mean, rstd, gamma, dgamma, dbeta, dres=None, cast=None):
        if dgamma is not None or dbeta is not None or (cast is not None and cast[2] is not None):
            counts["affine"] += 1
        return lnb(dy, x, mean, rstd, gamma, dgamma, dbeta, dres=dres, cast=cast)

    def attn_bwd(*a, **k):
        if k.get("table_grads", True):
            counts["tables"] += 1
        return ab(*a, **k)

    monkeypatch.setattr(engine, "_wgrad", bump("wgrad", wgrad))
    monkeypatch.setattr(ops, "conv3x3_wgrad", bump("conv3x3_wgrad", cw))
    monkeypatch.setattr(ops, "colsum_bf16", bump("colsum", cs))
    monkeypatch.setattr(ops, "scale_cast_colsum", bump("scale_cast", scc))
    monkeypatch.setattr(ops, "layernorm_bwd", ln_bwd)
    monkeypatch.setattr(ops, "attn_bwd", attn_bwd)
    kept, loss, x, t = _saved_activations(model, imgs, tgts, mask, valid, monkeypatch)
    assert not any(any(v) for v in kept.values()), kept
    loss.backward()
    assert x.grad is not None and t.grad is not None
    # the blocks hand bf16(scale * dx) down without a gradient arena too: only the blocks whose output also feeds the
    # early merge or a decoder tap (2, 5, 11, 17, 23) make their own pass over the incoming gradient
    assert counts == {"wgrad": 0, "conv3x3_wgrad": 0, "colsum": 0, "affine": 0, "tables": 0, "scale_cast": 5}, counts


def test_module_frozen_after_training_drops_its_gradient_arena():
    cfg, model = _tiny()
    imgs, tgts, mask, valid = (v.cuda() for v in synth_inputs(cfg, 2, 19))
    loss, _, _ = model(imgs, tgts, mask, valid)
    loss.backward()
    assert getattr(model, "_pk_arena", None) is not None
    model.zero_grad(set_to_none=True)
    model.requires_grad_(False)
    x = imgs.clone().requires_grad_(True)
    loss, _, _ = model(x, tgts, mask, valid)
    assert getattr(model, "_pk_arena", None) is None
    loss.backward()
    assert x.grad is not None and all(p.grad is None for p in model.parameters())


def test_prompt_tuning_lowers_the_loss():
    """model.requires_grad_(False); a learnable prompt image / target pair stacked above the query, bf16 autocast,
    torch.optim.AdamW on the two prompt tensors (INTEGRATION.md)."""
    cfg, model = _tiny(seed=1)
    model.requires_grad_(False)
    g = torch.Generator().manual_seed(3)
    q_img = torch.randn(2, 3, 64, 64, generator=g).cuda()
    q_tgt = torch.randn(2, 3, 64, 64, generator=g).cuda()
    prompt_img = torch.zeros(1, 3, 64, 64, device="cuda", requires_grad=True)
    prompt_tgt = torch.zeros(1, 3, 64, 64, device="cuda", requires_grad=True)
    h, w = cfg.grid
    mask = torch.zeros(2, h, w, dtype=torch.bool, device="cuda")
    mask[:, h // 2:] = True
    valid = torch.ones(2, 3, 128, 64, device="cuda")
    opt = torch.optim.AdamW([prompt_img, prompt_tgt], lr=5e-2, weight_decay=0.0)
    losses = []
    for _ in range(20):
        imgs = torch.cat([prompt_img.expand(2, -1, -1, -1), q_img], dim=2)
        tgts = torch.cat([prompt_tgt.expand(2, -1, -1, -1), q_tgt], dim=2)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss, _, _ = model(imgs, tgts, mask, valid)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(p.grad is None for p in model.parameters())
    print("prompt-tuning losses", losses[0], losses[-1])
    assert losses[-1] < 0.95 * losses[0], losses
