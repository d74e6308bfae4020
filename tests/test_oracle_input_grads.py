"""The CPU oracle's input gradients (imgs.grad, tgts.grad) against golden vectors of the unmodified reference
(scripts/make_golden_input_grads.py): eval and train mode (DropPath replayed), the four loss functions, a sample that
triggers `inds_ign`, valid maps with zeros and 10s, block masks plus the half mask, and windowed blocks.  CPU only."""
import pytest
import torch

from oracle import painter_oracle as po
from oracle.synth import synth_inputs, synth_state_dict

from _common import load_golden

CASES = ("eval", "train", "l1", "l2", "l1l2", "blockmask", "window")


@pytest.fixture(scope="module")
def gold():
    return load_golden("painter_tiny_input_grads.pt")["cases"]


def oracle_input_grads(c):
    """(loss, dimgs, dtgts) of the fp32 oracle on a golden case."""
    cfg = po.PainterConfig(**c["cfg"])
    sd = synth_state_dict(cfg, c["weight_seed"])
    imgs, tgts, mask, valid = synth_inputs(cfg, **c["inputs"])
    if c["mask"] is not None:
        mask = c["mask"]
    drops = None
    if c["train_seed"] is not None:
        torch.manual_seed(c["train_seed"])
        drops = po.draw_drop_scales(cfg, imgs.shape[0])
    imgs.requires_grad_(True)
    tgts.requires_grad_(True)
    loss, _, _ = po.forward(sd, cfg, imgs, tgts, mask, valid, drops=drops)
    loss.backward()
    return loss.detach(), imgs.grad, tgts.grad


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def test_golden_covers_every_case(gold):
    assert sorted(gold) == sorted(CASES)
    assert gold["window"]["cfg"]["window_block_indexes"]
    assert gold["train"]["train_seed"] is not None
    assert {gold[k]["cfg"]["loss_func"] for k in CASES} == {"smoothl1", "l1", "l2", "l1l2"}


@pytest.mark.parametrize("name", CASES)
def test_oracle_input_grads_match_reference(gold, name):
    c = gold[name]
    loss, dimgs, dtgts = oracle_input_grads(c)
    assert abs(loss.item() - c["loss"].item()) < 2e-6 * abs(c["loss"].item())
    assert _rel(dimgs, c["dimgs"]) < 2e-4
    assert _rel(dtgts, c["dtgts"]) < 2e-4
    if c["inputs"].get("dark_sample") is not None:
        # the loss ignores the all-black sample, and samples do not mix in the encoder: its image gets no gradient
        assert c["dimgs"][c["inputs"]["dark_sample"]].abs().max() == 0
