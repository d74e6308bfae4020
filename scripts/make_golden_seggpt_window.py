"""Golden vectors of the prompt ensemble inside windowed blocks, by EXECUTING THE UNMODIFIED REFERENCE on the CPU in fp32.

    python scripts/make_golden_seggpt_window.py [OUT]      (default tests/golden/seggpt_tiny_window.pt)

Needs the reference checkout (oracle/ref_loader.py).  The model is the tiny SegGPT of oracle/make_golden.py (TINY,
built by its build_ref from seeded synthetic weights) with ws = 7 and REAL window blocks on both sides of the early
merge (ws = 7 pads the 8x4 grid to 14x7).  The forward is called as seggpt_engine.run_one_image calls it (eval, half
mask, all-valid): one prompt (ensemble off), the ensemble over 2 / 3 prompts from block 0 with both seg types, and the
ensemble from block 4 on.  The fixture stores the seeds and the reference's loss and prediction (790 KB).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import GOLD, TINY, build_ref   # noqa: E402
from oracle.painter_oracle import PainterConfig       # noqa: E402
from oracle.synth import synth_inputs                  # noqa: E402

# (prompts, seg type, merge_between_batch)
CASES = ((1, 0, -1), (2, 0, 0), (3, 1, 0), (2, 1, 4))


def make(path):
    torch.set_num_threads(8)
    cfg = PainterConfig(**{**TINY, "window_size": 7}, window_block_indexes=(0, 1, 3, 4, 6, 7), seggpt=True)
    m = build_ref(cfg, 6).eval()
    out = dict(cfg=cfg.__dict__, weight_seed=6, cases=[])
    h, w = cfg.grid
    for P, st, fe in CASES:
        x, t, _, _ = synth_inputs(cfg, P, 200 + P)
        bm = torch.zeros(1, h * w)
        bm[:, h * w // 2:] = 1
        seg = torch.full((P, 1), float(st))
        with torch.no_grad():
            loss, y, _ = m(x, t, bm, torch.ones_like(t), seg, fe)
        out["cases"].append(dict(P=P, seed=200 + P, seg_type=st, merge_between_batch=fe, loss=loss, pred=y))
        print("seggpt window P", P, "merge_between_batch", fe, "loss", loss.item())
    torch.save(out, path)


if __name__ == "__main__":
    make(sys.argv[1] if len(sys.argv) > 1 else os.path.join(GOLD, "seggpt_tiny_window.pt"))
