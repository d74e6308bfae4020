"""Shared fixtures of the augmentation tests: a temporary Painter-style dataset (one json list per pair type) and
PairDataset built with main_train.py's stock transforms from the unmodified reference modules."""
import json
import os

import numpy as np

from oracle import ref_loader

TYPES = ["nyuv2_image2depth", "ade20k_image2semantic", "coco_image2panoptic_sem_seg", "coco_image2pose",
         "coco_image2panoptic_inst", "ssid_image2denoise", "derain_rainy2clean", "lol_low2image"]
# (W, H): downscale and upscale to 448 on both axes, square and very flat sources
SIZES = [(683, 512), (320, 240), (500, 700), (448, 448), (900, 300), (260, 530)]


def write_dataset(root, per_type=3, seed=0):
    from PIL import Image
    rng = np.random.RandomState(seed)
    lists = []
    for ti, t in enumerate(TYPES):
        pairs = []
        for k in range(per_type):
            W, H = SIZES[(ti + k) % len(SIZES)]
            base = rng.randint(0, 256, (H // 8 + 1, W // 8 + 1, 3)).astype(np.uint8)
            img = Image.fromarray(base).resize((W, H), Image.BICUBIC)
            noise = rng.randint(-20, 21, (H, W, 3))
            img = Image.fromarray(np.clip(np.asarray(img).astype(int) + noise, 0, 255).astype(np.uint8))
            tgt = rng.randint(0, 150, (H // 16 + 1, W // 16 + 1, 3)).astype(np.uint8)
            tgt[: tgt.shape[0] // 3] = 0                       # black: below the valid thresholds
            tgt = Image.fromarray(tgt).resize((W, H), Image.NEAREST)
            ip, tp = f"{t}_{k}.jpg", f"{t}_{k}_t.png"
            img.save(os.path.join(root, ip), quality=90)
            tgt.save(os.path.join(root, tp))
            pairs.append({"image_path": ip, "target_path": tp, "type": t})
        jp = os.path.join(root, f"{t}.json")
        with open(jp, "w") as f:
            json.dump(pairs, f)
        lists.append(jp)
    return lists[:8]


def pair_transforms():
    d = os.path.join(ref_loader.REF_ROOT, "Painter")
    return ref_loader._load("ref_pair_transforms", os.path.join(d, "data", "pair_transforms.py"), d)


def reference_dataset(root, lists, train=True, min_random_scale=0.3, half_mask_ratio=0.3, use_two_pairs=True,
                      mask_generator=None):
    """PairDataset exactly as main_train.py:232-262 builds it (input_size (896, 448))."""
    pt = pair_transforms()
    PD = ref_loader.pairdataset()
    norm = [pt.ToTensor(), pt.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])]
    plain = pt.Compose([pt.RandomResizedCrop(448, scale=(0.9999, 1.0), interpolation=3), *norm])
    if not train:
        return PD.PairDataset(root, lists, transform=plain, transform2=None, transform3=None,
                              masked_position_generator=mask_generator, use_two_pairs=use_two_pairs,
                              half_mask_ratio=half_mask_ratio)
    tr = pt.Compose([pt.RandomResizedCrop(448, scale=(min_random_scale, 1.0), interpolation=3),
                     pt.RandomApply([pt.ColorJitter(0.4, 0.4, 0.2, 0.1)], p=0.8), pt.RandomHorizontalFlip(), *norm])
    sec = pt.Compose([pt.RandomResizedCrop((896, 448), scale=(min_random_scale, 1.0), ratio=(0.3, 0.7),
                                           interpolation=3)])
    return PD.PairDataset(root, lists, transform=tr, transform2=plain,
                          transform3=pt.Compose([pt.RandomResizedCrop(448, scale=(0.9999, 1.0), interpolation=3),
                                                 *norm]),
                          transform_seccrop=sec, masked_position_generator=mask_generator,
                          use_two_pairs=use_two_pairs, half_mask_ratio=half_mask_ratio)


def mask_generator():
    MG = ref_loader.masking_generator().MaskingGenerator
    return MG((56, 28), num_masking_patches=784, max_num_patches=None, min_num_patches=16)
