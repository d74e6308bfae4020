#!/usr/bin/env python
"""Step time and peak memory of a prompt-tuning step against a full training step, ViT-L 896x448.

    python scripts/prompt_tuning_step.py [--batch 8] [--steps 10] [--warmup 3] [--out result.json]

Both steps are forward + backward of the painter_b200 module under bf16 autocast on the same synthetic batch, the
module in train mode (DropPath on):
  full     every parameter requires grad (the training step without its optimizer)
  prompt   model.requires_grad_(False); only a [1, 3, 448, 448] prompt image and prompt target require grad (stacked
           above the query half of every canvas, as in INTEGRATION.md)
Time per step is the mean over `steps` warmed-up steps, measured with CUDA events; peak memory is
torch.cuda.max_memory_allocated() over those steps.  Prints the card, its power limit and max SM clock first, then
one JSON line per step kind.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def measure(model, make_inputs, params, steps, warmup):
    def step():
        imgs, tgts, mask, valid = make_inputs()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss, _, _ = model(imgs, tgts, mask, valid)
        loss.backward()
        for p in params:
            p.grad = None
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps, torch.cuda.max_memory_allocated() / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from oracle.painter_oracle import PainterConfig
    from oracle.synth import synth_inputs, synth_state_dict
    from painter_b200.models_painter import painter_vit_large_patch16_input896x448_win_dec64_8glb_sl1
    print("card (name, power limit, max SM clock):", card(), flush=True)
    cfg = PainterConfig()
    B = a.batch
    model = painter_vit_large_patch16_input896x448_win_dec64_8glb_sl1()
    model.load_state_dict(synth_state_dict(cfg, 0), strict=True)
    model = model.cuda().train()
    model.precision = "bf16"
    imgs, tgts, mask, valid = (t.cuda() for t in synth_inputs(cfg, B, 5, valid_kind="mixed"))
    mask = mask.bool()
    mask[:, :28] = False     # the prompt (top) half is never masked
    res = []
    params = list(model.parameters())
    ms, gb = measure(model, lambda: (imgs, tgts, mask, valid), params, a.steps, a.warmup)
    res.append(dict(step="full", batch=B, ms_per_step=round(ms, 2), peak_gib=round(gb, 2)))
    print(json.dumps(res[-1]), flush=True)

    model.requires_grad_(False)     # the next forward drops the gradient arena of the full steps
    torch.cuda.empty_cache()
    prompt_img = imgs[:1, :, :448].clone().requires_grad_(True)
    prompt_tgt = tgts[:1, :, :448].clone().requires_grad_(True)
    q_img, q_tgt = imgs[:, :, 448:], tgts[:, :, 448:]

    def prompt_inputs():
        return (torch.cat([prompt_img.expand(B, -1, -1, -1), q_img], dim=2),
                torch.cat([prompt_tgt.expand(B, -1, -1, -1), q_tgt], dim=2), mask, valid)

    ms, gb = measure(model, prompt_inputs, [prompt_img, prompt_tgt], a.steps, a.warmup)
    res.append(dict(step="prompt", batch=B, ms_per_step=round(ms, 2), peak_gib=round(gb, 2)))
    print(json.dumps(res[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=card(), results=res), f, indent=1)


if __name__ == "__main__":
    main()
