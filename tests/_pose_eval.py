"""TEST INFRASTRUCTURE: the UNMODIFIED reference COCO pose files, loaded through tests/_task_eval._load from a checkout
of the reference or the staged copy under oracle/_ref (scripts/stage_reference.py), and the seeded synthetic painted
person crops the pose tests and scripts/pose_post.py run on.

    Painter/eval/mmpose_custom/model/top_down.py                 TopDownCustom.forward_pseudo_test
    Painter/eval/mmpose_custom/data/topdown_coco_dataset.py      TopDownCocoDatasetCustom.evaluate
    Painter/eval/mmpose_custom/data/pipelines/custom_transform.py  define_colors_gb_mean_sep
    Painter/eval/mmpose_custom/configs/_base_/coco.py            dataset_info (flip pairs, sigmas)

For the duration of an import only, absent modules are replaced by stand-ins: mmcv (identity decorator factories),
mmpose's registries, post-processing and base classes (oracle/mmpose_ref.py restates the mmpose 0.29 functions),
json_tricks (json) and xtcocotools.  top_down.py imports `data.pipelines.custom_transform`, a name that Painter/data
(imported by other tests) also claims: while it loads, any imported `data` package is set aside and custom_transform.py
is registered under that name.  TopDownCustom.colors is created on "cuda", so loading top_down.py needs a GPU.
"""
import json
import os
import sys
import types

import numpy as np
import torch
from PIL import Image

import _task_eval
from oracle import mmpose_ref as mr

_DIR = os.path.join("eval", "mmpose_custom")


class TopDown(mr.TopDown):
    """The detector base class; decode_images_to_heatmaps_minmax reads the palette as `TopDown.colors`."""


class _Registry:
    def register_module(self, *_a, **_k):
        return lambda cls: cls


def _identity_factory(*_a, **_k):
    return lambda fn: fn


def _unused(*_a, **_k):
    raise NotImplementedError("stand-in")


_STANDINS = [
    ("mmcv", {"Config": dict, "deprecated_api_warning": _identity_factory}),
    ("mmcv.image", {"imwrite": _unused}),
    ("mmcv.utils.misc", {"deprecated_api_warning": _identity_factory}),
    ("mmcv.visualization.image", {"imshow": _unused}),
    ("mmcv.runner", {"auto_fp16": _identity_factory}),
    ("mmpose.core", {"imshow_bboxes": _unused, "imshow_keypoints": _unused}),
    ("mmpose.core.post_processing", {"flip_back": mr.flip_back, "oks_nms": mr.oks_nms,
                                     "soft_oks_nms": mr.soft_oks_nms}),
    ("mmpose.models.builder", {"POSENETS": _Registry()}),
    ("mmpose.models.detectors", {"TopDown": TopDown}),
    ("mmpose.datasets.builder", {"DATASETS": _Registry()}),
    ("mmpose.datasets.datasets.top_down", {"TopDownCocoDataset": mr.TopDownCocoDataset}),
    ("json_tricks", {"dump": json.dump, "load": json.load, "dumps": json.dumps, "loads": json.loads}),
    ("xtcocotools.cocoeval", {"COCOeval": _unused}),
]

# configs/coco_256x192_test_offline.py
TEST_CFG = dict(flip_test=True, post_process="default", shift_heatmap=True, modulate_kernel=17)
DATA_CFG = dict(image_size=[192, 256], heatmap_size=[192, 256], num_output_channels=17, num_joints=17,
                soft_nms=False, nms_thr=1.0, oks_thr=0.9, vis_thr=0.2, use_gt_bbox=False, imagename_with_boxid=True,
                det_bbox_thr=0.0)
H, W = 256, 192


def custom_transform():
    return _task_eval._load("pose_custom_transform", os.path.join(_DIR, "data", "pipelines", "custom_transform.py"),
                            standins=[("cv2", None)])


def coco_info():
    return _task_eval._load("pose_coco_base", os.path.join(_DIR, "configs", "_base_", "coco.py")).dataset_info


def palette():
    """define_colors_gb_mean_sep() in dict order, then the background, as top_down.py builds TopDownCustom.colors."""
    return list(custom_transform().define_colors_gb_mean_sep().values()) + [(0, 0)]


def top_down():
    if "pose_top_down" in _task_eval._cache:
        return _task_eval._cache["pose_top_down"]
    ct = custom_transform()
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == "data" or k.startswith("data.")}
    pkg, pipes = types.ModuleType("data"), types.ModuleType("data.pipelines")
    pkg.__path__, pipes.__path__ = [], []
    pkg.pipelines, pipes.custom_transform = pipes, ct
    mine = {"data": pkg, "data.pipelines": pipes, "data.pipelines.custom_transform": ct}
    sys.modules.update(mine)
    try:
        mod = _task_eval._load("pose_top_down", os.path.join(_DIR, "model", "top_down.py"), standins=_STANDINS)
    finally:
        for k in mine:
            sys.modules.pop(k, None)
        sys.modules.update(saved)
    TopDown.colors = mod.TopDownCustom.colors
    return mod


def dataset_module():
    return _task_eval._load("pose_dataset", os.path.join(_DIR, "data", "topdown_coco_dataset.py"),
                            standins=_STANDINS)


def model(flip_test=True):
    cfg = dict(TEST_CFG, flip_test=flip_test)
    return top_down().TopDownCustom(backbone=None, keypoint_head=mr.TopdownHeatmapHead(cfg), test_cfg=cfg)


def dataset(ann_file, img_prefix):
    return dataset_module().TopDownCocoDatasetCustom(ann_file, img_prefix, DATA_CFG, [], dataset_info=coco_info())


def write_pngs(root, names, preds, flipped=None):
    """preds[i] as root/crops/names[i], flipped[i] as root/crops_flip/names[i] (where forward_pseudo_test looks)."""
    paths = []
    os.makedirs(os.path.join(root, "crops"), exist_ok=True)
    if flipped is not None:
        os.makedirs(os.path.join(root, "crops_flip"), exist_ok=True)
    for i, nm in enumerate(names):
        p = os.path.join(root, "crops", nm)
        Image.fromarray(np.asarray(preds[i])).save(p)
        if flipped is not None:
            Image.fromarray(np.asarray(flipped[i])).save(os.path.join(root, "crops_flip", nm))
        paths.append(p)
    return paths


def forward_pseudo_test(mdl, paths, centers, scales, box_scores, bbox_ids, flip_pairs):
    """The reference's forward_pseudo_test on the PNG files at `paths`, with the img_metas the offline pipeline
    collects (plus bbox_id)."""
    img = torch.from_numpy(np.stack([np.array(Image.open(p)) for p in paths])).cuda()
    metas = [{"image_file": p, "center": c, "scale": s, "rotation": 0, "bbox_score": b, "flip_pairs": flip_pairs,
              "bbox_id": int(i)} for p, c, s, b, i in zip(paths, centers, scales, box_scores, bbox_ids)]
    return mdl.forward_pseudo_test(img, metas)


# ---------------------------------------------------------------------------------------------------------------------
# Synthetic painted crops.

def heatmaps_numpy(images, pal):
    """decode_images_to_heatmaps_minmax restated in numpy: float32 [N, 17, H, W]."""
    x = np.asarray(images).astype(np.float32)
    d = np.abs(x[:, None, :, :, 1:] - np.asarray(pal, np.float32)[None, :, None, None, :]).sum(-1)
    cls = np.argmin(d, axis=1)
    return np.stack([(cls == k) * x[..., 0] for k in range(17)], axis=1) / 255.


def tie_colours(pal):
    """(G, B) pairs whose nearest palette colour is not unique (torch.min takes the first)."""
    pal = np.asarray(pal, dtype=np.int32)
    g, b = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    d = np.abs(g[..., None] - pal[:, 0]) + np.abs(b[..., None] - pal[:, 1])
    ties = (d == d.min(-1, keepdims=True)).sum(-1) >= 2
    return np.argwhere(ties).astype(np.int32)


EDGES_X = (0, 1, 2, W - 2, W - 1)
EDGES_Y = (0, 1, 2, H - 2, H - 1)


def _paint(rng, blobs, pal, ties, absent):
    img = np.zeros((H, W, 3), dtype=np.int32)
    img[..., 1:] = rng.integers(0, 26, size=(H, W, 2))             # background: nearest to (0, 0)
    noise = rng.random((H, W)) < 0.01                              # faint joint-coloured speckle
    img[noise, 0] = rng.integers(1, 40, size=int(noise.sum()))
    img[noise, 1:] = pal[rng.integers(0, 17, size=int(noise.sum()))]
    yy, xx = np.mgrid[:H, :W]
    for k, cy, cx, r, flat, peak in blobs:
        d = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
        inside = d < r
        R = np.clip(np.round(peak * (1.0 - np.maximum(d - flat, 0.0) / r)), 0, 255)
        img[inside, 0] = R[inside]
        img[inside, 1:] = pal[k]
        tie = inside & (rng.random((H, W)) < 0.08)                 # colours between two palette entries
        img[tie, 1:] = ties[rng.integers(0, len(ties), size=int(tie.sum()))]
    # absent joints: no pixel of their class keeps a positive R
    cls = np.argmin(np.abs(img[:, :, None, 1:] - pal[None, None]).sum(-1), axis=-1)
    img[np.isin(cls, list(absent)), 0] = 0
    return np.clip(img, 0, 255).astype(np.uint8)


def painted_pair(rng, flip_pairs=None, absent=0.15):
    """A painted crop and the painting of its flipped crop (the mirrored layout, joints swapped, peaks jittered):
    joint blobs with flat tops (argmax ties), tie colours, peaks on the border rows / columns, absent joints and
    flat R = 51 joints (maxval exactly fl32(0.2))."""
    pal = np.asarray(palette(), dtype=np.int32)
    ties = tie_colours(pal)
    pairs = flip_pairs or [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
    swap = np.arange(17)
    for a, b in pairs:
        swap[a], swap[b] = b, a
    blobs, fblobs, gone = [], [], set()
    for k in range(17):
        if rng.random() < absent:
            gone.add(k)
            continue
        cy, cx = int(rng.integers(0, H)), int(rng.integers(0, W))
        if rng.random() < 0.3:
            cx = int(rng.choice(EDGES_X))
        if rng.random() < 0.3:
            cy = int(rng.choice(EDGES_Y))
        r, flat = int(rng.integers(3, 12)), int(rng.integers(0, 3))
        peak = 51 if rng.random() < 0.15 else int(rng.integers(60, 256))
        blobs.append((k, cy, cx, r, flat, peak))
        fpeak = peak if peak == 51 else int(np.clip(peak + rng.integers(-20, 21), 52, 255))
        fblobs.append((int(swap[k]), cy, W - cx - int(rng.integers(0, 2)), r, flat, fpeak))
    return _paint(rng, blobs, pal, ties, gone), _paint(rng, fblobs, pal, ties, {int(swap[k]) for k in gone})


def boxes_for(rng, n, img_w=640, img_h=480):
    """n random person boxes [x, y, w, h] (wide, tall and 3:4 ones, fractional)."""
    w = rng.uniform(30, 300, n)
    h = w * rng.choice([0.5, 4.0 / 3.0, 2.5], n) * rng.uniform(0.9, 1.1, n)
    x, y = rng.uniform(0, img_w - 30, n), rng.uniform(0, img_h - 30, n)
    return np.stack([x, y, w, h], axis=1)


def dataset_stream(seed, counts=(3, 20, 9, 18), repeats=5):
    """Boxes of several images in a shuffled stream: per image, clusters of boxes jittered around one painted person
    (near-duplicate poses), random bbox_ids, and `repeats` boxes sent twice (sampler padding).  Returns (preds,
    flipped, centers, scales, box scores, image ids, bbox ids, PNG names)."""
    from painter_b200.pose import box_center_scale
    rng = np.random.default_rng(seed)
    entries = []
    for im, cnt in enumerate(counts):
        iid = 785 + 1000 * im
        k = max(1, cnt // 4)
        base = [(painted_pair(rng, absent=0.05), boxes_for(rng, 1)[0]) for _ in range(k)]
        for j in range(cnt):
            (p, f), b = base[j % k]
            jit = b + rng.normal(0.0, 1.0, 4) * np.array([2.0, 2.0, 3.0, 3.0]) * rng.choice([0.1, 1.0, 6.0])
            entries.append((iid, jit, p, f))
    order = rng.permutation(len(entries))
    entries = [entries[i] for i in order]
    bbox_ids = rng.permutation(len(entries))
    pick = list(range(len(entries))) + list(rng.choice(len(entries), repeats, replace=False))
    image_ids = np.array([entries[i][0] for i in pick])
    boxes = np.array([entries[i][1] for i in pick])
    c, s = box_center_scale(boxes)
    scores = np.array([rng.uniform(0.3, 1.0) for _ in range(len(entries))])[pick]
    names = [f"{image_ids[j]:012d}_box{bbox_ids[i]}_image.png" for j, i in enumerate(pick)]
    return ([entries[i][2] for i in pick], [entries[i][3] for i in pick], c, s, scores, image_ids,
            bbox_ids[pick], names)
