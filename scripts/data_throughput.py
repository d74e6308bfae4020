#!/usr/bin/env python
"""Training data path throughput: the reference PairDataset (PIL + torch-CPU augmentations in the worker) against
DevicePairDataset + pair_collate + DevicePairAugment, on a synthetic JPEG/PNG dataset written to a temporary directory
(683x512 pairs of four pair types, two pairs per sample, main_train.py's stock recipe).

    python scripts/data_throughput.py [--samples 64] [--workers 8] [--steps 20] [--out result.json]

Reports host ms/sample on one core for both, device ms per batch of 8 (CUDA events) and the images/s of
GraphedTrainStep (ViT-L 896x448, bf16, batch 8) fed by the new pipeline with N DataLoader workers, next to the same
step on synthetic in-memory batches.  Needs the reference tree (oracle/ref_loader.py) for the host comparison."""
import argparse
import contextlib
import io
import json
import os
import random
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def write_synthetic(root, n=16):
    import numpy as np
    from PIL import Image
    rng = np.random.default_rng(0)
    types = ["ade20k_image2semantic", "coco_image2panoptic_sem_seg", "nyuv2_image2depth", "derain_rainy2clean"]
    lists = []
    for t in types:
        pairs = []
        for i in range(n // len(types)):
            H, W = 512, 683
            base = rng.integers(0, 255, (H // 8, W // 8, 3), dtype=np.uint8)
            Image.fromarray(base).resize((W, H), Image.BICUBIC).save(f"{root}/{t}_{i}.jpg", quality=90)
            tgt = rng.integers(0, 150, (H // 16, W // 16, 3), dtype=np.uint8)
            Image.fromarray(tgt).resize((W, H), Image.NEAREST).save(f"{root}/{t}_{i}.png")
            pairs.append({"image_path": f"{t}_{i}.jpg", "target_path": f"{t}_{i}.png", "type": t})
        with open(f"{root}/{t}.json", "w") as f:
            json.dump(pairs, f)
        lists.append(f"{root}/{t}.json")
    return lists


def host_ms(fn, n):
    for k in range(4):
        fn(k)
    t0 = time.perf_counter()
    for k in range(n):
        fn(k)
    return (time.perf_counter() - t0) / n * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from painter_b200.data_gpu import DevicePairAugment, DevicePairDataset, DevicePairPrefetcher, pair_collate
    from _augment_data import mask_generator, reference_dataset
    assert torch.cuda.is_available(), "data_throughput.py measures on the GPU"
    torch.set_num_threads(1)
    res = {"gpu": torch.cuda.get_device_name(0)}
    try:
        res["nvidia_smi"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        res["nvidia_smi"] = f"unavailable: {e}"
    with tempfile.TemporaryDirectory() as root:
        lists = write_synthetic(root)
        with contextlib.redirect_stdout(io.StringIO()):
            ref = reference_dataset(root, lists, train=True, half_mask_ratio=0.1, mask_generator=mask_generator())
        ours = DevicePairDataset(root, lists, half_mask_ratio=0.1, masked_position_generator=mask_generator())
        random.seed(0)
        torch.manual_seed(0)
        res["reference_host_ms_per_sample"] = host_ms(lambda k: ref[k % len(ref)], args.samples)
        res["device_path_host_ms_per_sample"] = host_ms(lambda k: ours[k % len(ours)], args.samples)
        t0 = time.perf_counter()
        for _ in range(8):
            pair_collate([ours[k] for k in range(8)])
        res["pair_collate_ms_per_batch_of_8_incl_getitem"] = (time.perf_counter() - t0) / 8 * 1e3
        # device time of one batch of 8
        aug = DevicePairAugment("cuda")
        packed = pair_collate([ours[k] for k in range(8)]).pin_memory()
        for _ in range(5):
            aug(packed)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(50):
            aug(packed)
        e1.record()
        torch.cuda.synchronize()
        res["device_ms_per_batch_of_8"] = e0.elapsed_time(e1) / 50
        res["packed_mb_per_batch_of_8"] = packed.buf.numel() / 1e6
        # the training step, on synthetic resident batches and fed by the pipeline
        from painter_b200 import models_painter
        from painter_b200.optim import FusedAdamW
        from painter_b200.train_utils import GraphedTrainStep, adjust_learning_rate, param_groups_lrd
        torch.manual_seed(0)
        model = models_painter.painter_vit_large_patch16_input896x448_win_dec64_8glb_sl1().cuda().train()
        groups = param_groups_lrd(model, 0.05, no_weight_decay_list=model.no_weight_decay(), layer_decay=0.8)
        opt = FusedAdamW(groups, lr=1e-4, betas=(0.9, 0.999))
        adjust_learning_rate(opt, 1.0, 1e-4, 0.0, 1, 15)
        step = GraphedTrainStep(model, opt)
        img, tgt, m, v = aug(packed)
        batch = [t.clone() for t in (img, tgt, m, v)]
        for _ in range(3):
            step(*batch)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step(*batch)
        torch.cuda.synchronize()
        res["train_img_s_synthetic_resident"] = 8 * args.steps / (time.perf_counter() - t0)
        loader = torch.utils.data.DataLoader(
            ours, batch_size=8, num_workers=args.workers, collate_fn=pair_collate, pin_memory=True, drop_last=True,
            sampler=torch.utils.data.RandomSampler(ours, replacement=True, num_samples=8 * (args.steps + 6)),
            persistent_workers=False)
        it = DevicePairPrefetcher(loader, "cuda")
        for _ in range(5):
            step(*next(it))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 0
        for b in it:
            step(*b)
            n += 1
        torch.cuda.synchronize()
        res["train_img_s_fed_by_device_pipeline"] = 8 * n / (time.perf_counter() - t0)
        res["workers"] = args.workers
        res["host_cpus"] = os.cpu_count()
    res["nvidia_smi_after"] = subprocess.run(
        ["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"], capture_output=True,
        text=True, timeout=30).stdout.strip()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
