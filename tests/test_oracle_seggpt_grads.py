"""The CPU oracle's SegGPT training gradients against golden vectors of the unmodified reference
(scripts/make_golden_seggpt_grads.py): the loss, imgs.grad, tgts.grad, both seg-type tokens and the GRAD_KEYS
parameters, in eval and train mode (DropPath replayed), with seg types 0, 1 and 2 in one batch, another loss function
and windowed blocks.  CPU only."""
import pytest
import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs, synth_state_dict

from _common import load_golden

CASES = ("eval", "train", "mixed", "l2", "window")


@pytest.fixture(scope="module")
def gold():
    return load_golden("seggpt_tiny_grads.pt")["cases"]


def oracle_grads(c):
    """(loss, {name: gradient}) of the fp32 oracle on a golden case, for every parameter and imgs / tgts."""
    cfg = po.PainterConfig(**c["cfg"])
    sd = {k: v.requires_grad_(True) for k, v in synth_state_dict(cfg, c["weight_seed"]).items()}
    imgs, tgts, mask, valid = synth_inputs(cfg, **c["inputs"])
    drops = None
    if c["train_seed"] is not None:
        torch.manual_seed(c["train_seed"])
        drops = po.draw_drop_scales(cfg, imgs.shape[0])
    imgs.requires_grad_(True)
    tgts.requires_grad_(True)
    loss, _, _ = po.forward(sd, cfg, imgs, tgts, mask, valid, drops=drops, seg_type=c["seg_type"])
    loss.backward()
    grads = {k: v.grad for k, v in sd.items()}
    grads.update(dimgs=imgs.grad, dtgts=tgts.grad)
    return loss.detach(), grads


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def test_golden_covers_every_case(gold):
    assert sorted(gold) == sorted(CASES)
    assert gold["window"]["cfg"]["window_block_indexes"] and gold["train"]["train_seed"] is not None
    assert sorted(gold["mixed"]["seg_type"].flatten().tolist()) == [0.0, 1.0, 2.0]
    assert {gold[k]["cfg"]["loss_func"] for k in CASES} == {"smoothl1", "l2"}
    assert all(gold[k]["cfg"]["seggpt"] for k in CASES)
    for k in CASES:
        g = gold[k]["grads"]
        assert {"type_token_cls", "type_token_ins", "dimgs", "dtgts", "pos_embed"} <= set(g), sorted(g)


@pytest.mark.parametrize("name", CASES)
def test_oracle_seggpt_grads_match_reference(gold, name):
    c = gold[name]
    loss, grads = oracle_grads(c)
    assert abs(loss.item() - c["loss"].item()) < 2e-6 * abs(c["loss"].item())
    bad = [(k, _rel(grads[k], ref)) for k, ref in c["grads"].items() if not _rel(grads[k], ref) < 2e-4]
    assert not bad, bad
    for k in ("type_token_cls", "type_token_ins"):
        assert c["grads"][k].abs().max() > 0, k      # every case has a sample of each token's type
