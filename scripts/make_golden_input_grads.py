#!/usr/bin/env python
"""Golden input gradients: imgs.grad and tgts.grad of the UNMODIFIED reference `Painter` at the tiny geometry.

    python scripts/make_golden_input_grads.py      # needs the reference tree (oracle/ref_loader.py finds it)

Writes tests/golden/painter_tiny_input_grads.pt (the cases' seeds, masks and losses) and
painter_tiny_input_grads.part<i>.pt (the gradients, one case per part so that every file stays below 1 MB;
tests/_common.load_golden merges them).  Weights and inputs are regenerated from seeds by oracle/synth.py, the way
oracle/make_golden.py builds the other goldens.  Cases:
  eval / train       smoothl1, mixed valid (zeros and 10s), random mask, sample 1 all black (the `inds_ign` rule);
                     train mode draws DropPath from torch.manual_seed(train_seed) (replayed by the tests)
  l1 / l2 / l1l2     the other loss functions, same kind of inputs
  blockmask          a BEiT-style block mask on sample 0 and the half mask on sample 1
  window             real windowed blocks (ws = 7 on the 8 x 4 grid pads to 14 x 7)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import TINY, build_ref  # noqa: E402
from oracle.painter_oracle import PainterConfig  # noqa: E402
from oracle.synth import synth_inputs  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
STEM = "painter_tiny_input_grads"


def block_masks(cfg):
    """Sample 0: two rectangular blocks (BEiT MaskingGenerator style); sample 1: the bottom half (pairdataset.py)."""
    h, w = cfg.grid
    m = torch.zeros(2, h, w, dtype=torch.int32)
    m[0, 1:4, 0:3] = 1
    m[0, 5:8, 2:4] = 1
    m[1, h // 2:] = 1
    return m


def cases():
    """(name, cfg, weight seed, synth_inputs kwargs, explicit mask or None, train seed or None)"""
    inp = dict(B=2, seed=11, mask_kind="random", valid_kind="mixed", dark_sample=1)
    out = [("eval", PainterConfig(**TINY), 0, inp, None, None),
           ("train", PainterConfig(**TINY), 0, inp, None, 77)]
    for lf in ("l1", "l2", "l1l2"):
        out.append((lf, PainterConfig(**TINY, loss_func=lf), 2,
                    dict(B=2, seed=21, mask_kind="random", valid_kind="mixed", dark_sample=0), None, None))
    cfg = PainterConfig(**TINY)
    out.append(("blockmask", cfg, 0, dict(B=2, seed=31, valid_kind="mixed"), block_masks(cfg), None))
    cfgw = PainterConfig(**{**TINY, "window_size": 7}, window_block_indexes=(0, 1, 3, 4, 6, 7))
    out.append(("window", cfgw, 3, dict(B=2, seed=5, valid_kind="mixed"), None, None))
    return out


def main():
    torch.set_num_threads(8)
    meta, parts = {}, []
    for name, cfg, wseed, inp, mask, train_seed in cases():
        m = build_ref(cfg, wseed)
        m.train(train_seed is not None)
        imgs, tgts, mk, valid = synth_inputs(cfg, **inp)
        if mask is not None:
            mk = mask
        imgs.requires_grad_(True)
        tgts.requires_grad_(True)
        if train_seed is not None:
            torch.manual_seed(train_seed)
        loss, _, _ = m(imgs, tgts, mk.clone(), valid.clone())
        loss.backward()
        meta[name] = dict(cfg=cfg.__dict__, weight_seed=wseed, inputs=inp, mask=mask, train_seed=train_seed,
                          loss=loss.detach())
        parts.append({"cases": {name: dict(dimgs=imgs.grad.clone(), dtgts=tgts.grad.clone())}})
        print(f"{name}: loss {loss.item():.6f}  |dimgs| {imgs.grad.norm():.3e}  |dtgts| {tgts.grad.norm():.3e}")
    torch.save({"cases": meta}, os.path.join(GOLD, STEM + ".pt"))
    for i, part in enumerate(parts):
        torch.save(part, os.path.join(GOLD, f"{STEM}.part{i}.pt"))


if __name__ == "__main__":
    main()
