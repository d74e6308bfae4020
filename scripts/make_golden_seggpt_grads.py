#!/usr/bin/env python
"""Golden training gradients of the UNMODIFIED reference `SegGPT` at the tiny geometry, one prompt per sample.

    python scripts/make_golden_seggpt_grads.py      # needs the reference tree (oracle/ref_loader.py finds it)

Writes tests/golden/seggpt_tiny_grads.pt (each case's seeds, seg types and loss) and seggpt_tiny_grads.part<i>.pt (the
gradients: imgs.grad, tgts.grad, both type tokens and the oracle.make_golden.GRAD_KEYS parameters of at most 70000
elements, as make_golden keeps them, split so that every file stays below 1 MB; tests/_common.load_golden merges
them).  Weights and inputs are regenerated from seeds by oracle/synth.py.  Cases (random masks, valid maps with
zeros and 10s):
  eval / train       smoothl1, seg types (1, 0); train mode draws DropPath from torch.manual_seed(train_seed)
                     (replayed by the tests)
  mixed              three samples with seg types 0, 1 and 2 (type 2 selects neither token)
  l2                 another loss function
  window             real windowed blocks (ws = 7 on blocks 0, 1, 3, 4, 6, 7; the 8 x 4 grid pads to 14 x 7)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import GRAD_KEYS, TINY, build_ref  # noqa: E402
from oracle.painter_oracle import PainterConfig  # noqa: E402
from oracle.synth import synth_inputs  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
STEM = "seggpt_tiny_grads"
TYPE_KEYS = ["type_token_cls", "type_token_ins"]
PART_BYTES = 900 * 1024


def cases():
    """(name, cfg, weight seed, synth_inputs kwargs, seg types, train seed or None)"""
    cfg = PainterConfig(**TINY, seggpt=True)
    inp = dict(B=2, seed=41, mask_kind="random", valid_kind="mixed")
    out = [("eval", cfg, 5, inp, (1, 0), None),
           ("train", cfg, 5, inp, (1, 0), 78),
           ("mixed", cfg, 6, dict(B=3, seed=43, mask_kind="random", valid_kind="mixed"), (0, 1, 2), None),
           ("l2", PainterConfig(**TINY, seggpt=True, loss_func="l2"), 7,
            dict(B=2, seed=45, mask_kind="random", valid_kind="mixed"), (0, 1), None)]
    cfgw = PainterConfig(**{**TINY, "window_size": 7}, seggpt=True, window_block_indexes=(0, 1, 3, 4, 6, 7))
    out.append(("window", cfgw, 8, dict(B=2, seed=47, mask_kind="random", valid_kind="mixed"), (0, 1), None))
    return out


def split(tensors):
    """{name: tensor} -> list of dicts of at most PART_BYTES each (largest first, first fit)."""
    parts, sizes = [], []
    for k in sorted(tensors, key=lambda k: -tensors[k].numel()):
        nbytes = tensors[k].numel() * 4
        for i, s in enumerate(sizes):
            if s + nbytes <= PART_BYTES:
                parts[i][k] = tensors[k]
                sizes[i] += nbytes
                break
        else:
            parts.append({k: tensors[k]})
            sizes.append(nbytes)
    return parts


def main():
    torch.set_num_threads(8)
    meta, parts = {}, []
    for name, cfg, wseed, inp, types, train_seed in cases():
        m = build_ref(cfg, wseed)
        m.train(train_seed is not None)
        imgs, tgts, mask, valid = synth_inputs(cfg, **inp)
        seg = torch.tensor(types, dtype=torch.float32).reshape(-1, 1)
        imgs.requires_grad_(True)
        tgts.requires_grad_(True)
        if train_seed is not None:
            torch.manual_seed(train_seed)
        loss, _, _ = m(imgs, tgts, mask.clone(), valid.clone(), seg.clone())
        loss.backward()
        named = dict(m.named_parameters())
        grads = {k: named[k].grad.clone() for k in GRAD_KEYS + TYPE_KEYS if named[k].numel() <= 70000}
        grads.update(dimgs=imgs.grad.clone(), dtgts=tgts.grad.clone())
        meta[name] = dict(cfg=cfg.__dict__, weight_seed=wseed, inputs=inp, seg_type=seg, train_seed=train_seed,
                          loss=loss.detach())
        parts += [{"cases": {name: {"grads": p}}} for p in split(grads)]
        print(f"{name}: loss {loss.item():.6f}  |d cls| {grads['type_token_cls'].norm():.3e}  "
              f"|d ins| {grads['type_token_ins'].norm():.3e}  |dimgs| {imgs.grad.norm():.3e}")
    torch.save({"cases": meta}, os.path.join(GOLD, STEM + ".pt"))
    for i, part in enumerate(parts):
        torch.save(part, os.path.join(GOLD, f"{STEM}.part{i}.pt"))
    print(len(parts), "parts")


if __name__ == "__main__":
    main()
