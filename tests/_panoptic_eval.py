"""TEST INFRASTRUCTURE: the UNMODIFIED reference COCO panoptic evaluators, loaded through tests/_task_eval._load from a
checkout of the reference or the staged copy under oracle/_ref (scripts/stage_reference.py), and the seeded synthetic
painted images the panoptic tests and scripts/panoptic_post.py run on.

    Painter/eval/coco_panoptic/COCOCAInstSegEvaluatorCustom.py   define_colors_per_location_r_gb, COCOEvaluatorCustom
                                                                 (post_process_segm_output_by_threshold / _by_minmax)
    Painter/eval/coco_panoptic/COCOInstSegEvaluatorCustom.py     COCOInstanceEvaluatorCustom.merge_inst_semseg_result
    Painter/eval/coco_panoptic/COCOPanoEvaluatorCustom.py        combine_semantic_and_instance_outputs_custom
    Painter/util/matrix_nms.py                                   mask_matrix_nms

For the duration of an import only, absent modules are replaced by stand-ins: pycocotools, detectron2's file_io,
evaluation (a base class that accepts the constructor arguments), structures (minimal working Instances and Boxes),
data and comm, mmcv.ops, the COCO dataset registration, panopticapi and matplotlib.
"""
import os

import numpy as np
import torch

import _task_eval
from oracle import ref_loader


class Instances:
    """detectron2.structures.Instances, the part the evaluators use: fields set as attributes, len, to(device)."""

    def __init__(self, image_size, **fields):
        object.__setattr__(self, "image_size", image_size)
        object.__setattr__(self, "_fields", {})
        for k, v in fields.items():
            setattr(self, k, v)

    def __setattr__(self, k, v):
        self._fields[k] = v

    def __getattr__(self, k):
        f = self.__dict__.get("_fields", {})
        if k in f:
            return f[k]
        raise AttributeError(k)

    def __len__(self):
        for v in self._fields.values():
            return len(v)
        return 0

    def to(self, device):
        return Instances(self.image_size, **{k: v.to(device) if hasattr(v, "to") else v
                                             for k, v in self._fields.items()})


class Boxes:
    def __init__(self, tensor):
        self.tensor = tensor

    def __len__(self):
        return self.tensor.shape[0]

    def to(self, device):
        return Boxes(self.tensor.to(device))


class _Evaluator:                # stand-in base class of the detectron2 evaluators
    def __init__(self, *args, **kwargs):
        self._cpu_device = torch.device("cpu")
        self._predictions = []


def _unused(*_a, **_k):
    raise NotImplementedError("stand-in")


_STANDINS = [
    ("matplotlib.pyplot", None),
    ("pycocotools.mask", None),
    ("pycocotools.coco", {"COCO": _unused}),
    ("pycocotools.cocoeval", {"COCOeval": _unused}),
    ("detectron2.utils.file_io", {"PathManager": None}),
    ("detectron2.utils.comm", None),
    ("detectron2.data", {"MetadataCatalog": None}),
    ("detectron2.structures", {"Boxes": Boxes, "BoxMode": None, "Instances": Instances, "BitMasks": None,
                               "pairwise_iou": _unused}),
    ("detectron2.evaluation", {"COCOEvaluator": _Evaluator, "COCOPanopticEvaluator": _Evaluator,
                               "SemSegEvaluator": _Evaluator}),
    ("detectron2.evaluation.coco_evaluation", {"instances_to_coco_json": _unused}),
    ("mmcv.ops", {"soft_nms": _unused}),
    ("data.register_coco_panoptic_annos_semseg", None),
    ("panopticapi.utils", {"rgb2id": None, "IdGenerator": None, "id2rgb": None}),
]


def _mod(key, rel):
    return _task_eval._load(key, os.path.join("eval", "coco_panoptic", rel), standins=_STANDINS)


def ca_inst():
    return _mod("pano_ca_inst", "COCOCAInstSegEvaluatorCustom.py")


def inst_eval():
    return _mod("pano_inst", "COCOInstSegEvaluatorCustom.py")


def pano_eval():
    return _mod("pano_pano", "COCOPanoEvaluatorCustom.py")


def mask_matrix_nms():
    mod = ref_loader._load("ref_task_matrix_nms", os.path.join(_task_eval._painter_dir(), "util", "matrix_nms.py"),
                           _task_eval._painter_dir())
    return mod.mask_matrix_nms


def palette_dict():
    return ca_inst().define_colors_per_location_r_gb()


def inst_evaluator(dist_thr=19.0, post_type="threshold", num_windows=4):
    mod = ca_inst()
    return mod.COCOEvaluatorCustom("coco_2017_val", tasks=("segm",), palette_dict=palette_dict(), pred_dir=None,
                                   num_windows=num_windows, post_type=post_type, dist_thr=dist_thr)


def semseg_evaluator(palette):
    mod = _task_eval._load("semseg_coco", _task_eval._EVALUATORS["coco"], standins=[
        ("matplotlib.pyplot", None),
        ("detectron2.evaluation", {"SemSegEvaluator": _task_eval._SemSegEvaluator}),
        ("data.register_coco_panoptic_annos_semseg", None)])
    ev = mod.SemSegEvaluatorCustom.__new__(mod.SemSegEvaluatorCustom)
    ev.palette = torch.tensor(palette, dtype=torch.float, device="cuda")
    ev.dist_type = "abs"
    return ev


def instance_evaluator(evaluator_inst, evaluator_semseg, with_nms):
    return inst_eval().COCOInstanceEvaluatorCustom("coco_2017_val", tasks=("segm",), output_dir=None,
                                                   evaluator_inst=evaluator_inst, evaluator_semseg=evaluator_semseg,
                                                   label2cat=None, with_nms=with_nms, nms_type="matrix")


# ---------------------------------------------------------------------------------------------------------------------
# Synthetic painted images.

def instance_image(rng, h, w, palette, blobs=6, jitter=6, radius=(20, 70)):
    """Discs of distinct palette colours (the later on top) on black, every pixel jittered by up to +-jitter per
    channel (clipped to 0..255)."""
    img = np.zeros((h, w, 3), dtype=np.int32)
    yy, xx = np.mgrid[:h, :w]
    for k in rng.choice(len(palette), size=blobs, replace=False):
        cy, cx, r = rng.integers(0, h), rng.integers(0, w), rng.integers(*radius)
        img[(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = palette[k]
    img += rng.integers(-jitter, jitter + 1, size=img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def semantic_image(rng, h, w, palette, regions=12, jitter=10):
    """Vertical bands of random semantic colours, with rectangles of thing colours (< 80), jittered."""
    img = np.zeros((h, w, 3), dtype=np.int32)
    edges = np.sort(rng.choice(np.arange(1, w), size=3, replace=False))
    for a, b in zip(np.r_[0, edges], np.r_[edges, w]):
        img[:, a:b] = palette[rng.integers(80, len(palette))]
    for _ in range(regions):
        y0, x0 = rng.integers(0, h - 8), rng.integers(0, w - 8)
        img[y0:y0 + rng.integers(8, h // 2), x0:x0 + rng.integers(8, w // 2)] = palette[rng.integers(0, 80)]
    img += rng.integers(-jitter, jitter + 1, size=img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def separated(values, rel=1e-4):
    """True when consecutive sorted values differ by more than rel relative."""
    v = np.sort(np.asarray(values, dtype=np.float64))
    if len(v) < 2:
        return True
    gap = np.diff(v)
    return bool(np.all(gap > rel * np.maximum(np.abs(v[1:]), 1e-30)))
