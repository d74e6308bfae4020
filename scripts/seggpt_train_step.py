#!/usr/bin/env python
"""Time one SegGPT fine-tuning step: ViT-L 896x448 (the released checkpoint's geometry), batch 8, bf16 autocast,
every parameter trainable, FusedAdamW over the layer-decay groups of the reference recipe, in two forms:

  eager     forward + backward + FusedAdamW.step, one iteration after another
  graphed   train_utils.GraphedTrainStep(model, optimizer)(imgs, tgts, mask, valid, seg_type): the same iteration
            replayed as one CUDA graph

    python scripts/seggpt_train_step.py [--steps 20] [--warmup 5] [--batch 8] [--out result.json]

Reports the mean step time over the timed steps (CUDA events around the whole window, inputs resident on the device),
the peak memory of each form, and the card's name, power limit and maximum SM clock read in the same run.  Weights
are random (rel-pos tables drawn too); seg types alternate semantic / instance; masks cover half the tokens at random.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from painter_b200 import models_seggpt  # noqa: E402
from painter_b200.optim import FusedAdamW  # noqa: E402
from painter_b200.train_utils import GraphedTrainStep, param_groups_lrd  # noqa: E402


def card(dev):
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    power, clock = (s.strip() for s in q.stdout.strip().split(",")) if q.returncode == 0 else (None, None)
    return {"name": torch.cuda.get_device_name(dev), "power_limit": power, "max_sm_clock": clock}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seggpt_train_step.py times the GPU step: no CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    model = models_seggpt.seggpt_vit_large_patch16_input896x448().to(dev)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "rel_pos" in n:
                p.normal_(std=0.02)
    model.train()
    groups = param_groups_lrd(model, 0.05, no_weight_decay_list=model.no_weight_decay(), layer_decay=0.75)
    opt = FusedAdamW(groups, lr=1e-5, betas=(0.9, 0.999))
    B = args.batch
    g = torch.Generator().manual_seed(1)
    imgs = torch.randn(B, 3, 896, 448, generator=g).to(dev)
    tgts = torch.randn(B, 3, 896, 448, generator=g).to(dev)
    mask = (torch.rand(B, 56, 28, generator=g) < 0.5).to(dev)
    valid = torch.ones(B, 3, 896, 448, device=dev)
    seg = (torch.arange(B) % 2).float().reshape(B, 1).to(dev)

    def eager():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss, _, _ = model(imgs, tgts, bool_masked_pos=mask, valid=valid, seg_type=seg)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    torch.cuda.reset_peak_memory_stats(dev)
    ms_eager = timed(eager, args.steps, args.warmup)
    peak_eager = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    step = GraphedTrainStep(model, opt)
    torch.cuda.reset_peak_memory_stats(dev)
    ms_graph = timed(lambda: step(imgs, tgts, mask, valid, seg), args.steps, args.warmup)
    peak_graph = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    loss = float(step(imgs, tgts, mask, valid, seg))
    res = {"workload": f"SegGPT ViT-L 896x448 train step, batch {B}, bf16 autocast, FusedAdamW",
           "steps": args.steps, "warmup": args.warmup,
           "eager": {"ms_per_step": round(ms_eager, 2), "images_per_s": round(B / ms_eager * 1e3, 1),
                     "peak_mem_gib": round(peak_eager, 1)},
           "graphed": {"ms_per_step": round(ms_graph, 2), "images_per_s": round(B / ms_graph * 1e3, 1),
                       "peak_mem_gib": round(peak_graph, 1)},
           "last_loss": loss, "card": card(dev)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
