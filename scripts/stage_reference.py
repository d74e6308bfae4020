#!/usr/bin/env python
"""Stage the UNMODIFIED reference (baaivision/Painter) into the git-ignored `oracle/_ref/` so that a copy of the
tree (like the built .so files) carries it to a GPU machine that has no checkout of the reference, where it is
executed as the live oracle / reference arm:

    python scripts/stage_reference.py            # copies from $PAINTER_REFERENCE, else /root/reference

The reference is pure Python with no setup.py, so `pip install --target oracle/_ref <reference>` has nothing to
build (recorded in DESIGN.md); this script is the install step.  Only the files of the hot path, its two engines,
the runtime utilities they import, the task eval scripts (for their run_one_image), the task evaluators and palette
generators (for the metric parity tests), the pose model, dataset, colour and keypoint definitions of
eval/mmpose_custom (for the pose parity tests), the data pipeline used by the parity tests and the SegGPT example images are
copied, byte for byte; nothing under oracle/_ref is tracked by git or imported by the product path.
"""
import filecmp
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")

FILES = [
    "LICENSE",
    "Painter/models_painter.py",
    "Painter/engine_train.py",
    "Painter/main_train.py",
    "Painter/util",                       # misc, lr_sched, lr_decay, vitdet_utils, masking_generator, ...
    "Painter/data/pairdataset.py",
    "Painter/data/pair_transforms.py",
    "Painter/data/sampler.py",
    "Painter/eval/ade20k_semantic/painter_inference_segm.py",
    "Painter/eval/coco_panoptic/painter_inference_pano_semseg.py",
    "Painter/eval/coco_panoptic/painter_inference_pano_inst.py",
    "Painter/eval/mmpose_custom/painter_inference_pose.py",
    "Painter/eval/nyuv2_depth/painter_inference_depth.py",
    "Painter/eval/sidd/painter_inference_sidd.py",
    "Painter/eval/lol/painter_inference_lol.py",
    "Painter/eval/derain/painter_inference_derain.py",
    "Painter/eval/ade20k_semantic/ADE20kSemSegEvaluatorCustom.py",
    "Painter/eval/coco_panoptic/COCOPanoSemSegEvaluatorCustom.py",
    "Painter/eval/coco_panoptic/COCOCAInstSegEvaluatorCustom.py",
    "Painter/eval/coco_panoptic/COCOInstSegEvaluatorCustom.py",
    "Painter/eval/coco_panoptic/COCOPanoEvaluatorCustom.py",
    "Painter/eval/mmpose_custom/model/top_down.py",
    "Painter/eval/mmpose_custom/data/topdown_coco_dataset.py",
    "Painter/eval/mmpose_custom/data/pipelines/custom_transform.py",
    "Painter/eval/mmpose_custom/configs/_base_/coco.py",
    "Painter/eval/nyuv2_depth/eval_with_pngs.py",
    "Painter/data/ade20k/gen_color_ade20k_sem.py",
    "Painter/data/coco_semseg/gen_color_coco_panoptic_segm.py",
    "Painter/data/panoptic_coco_categories.json",
    "SegGPT/SegGPT_inference/models_seggpt.py",
    "SegGPT/SegGPT_inference/seggpt_engine.py",
    "SegGPT/SegGPT_inference/seggpt_inference.py",
    "SegGPT/SegGPT_inference/util",
    "SegGPT/SegGPT_inference/examples",
]


def source_root():
    """Where the reference checkout is read from: $PAINTER_REFERENCE, else its default location."""
    return os.environ.get("PAINTER_REFERENCE") or "/root/reference"


def stage(src_root=None, verbose=True):
    src_root = src_root or source_root()
    if not os.path.isdir(os.path.join(src_root, "Painter")):
        raise RuntimeError(f"reference tree not found at {src_root}")
    n = 0
    for rel in FILES:
        s, d = os.path.join(src_root, rel), os.path.join(DST, rel)
        if os.path.isdir(s):
            for dirpath, _, files in os.walk(s):
                for f in files:
                    if f.endswith((".pyc",)):
                        continue
                    sp = os.path.join(dirpath, f)
                    dp = os.path.join(d, os.path.relpath(sp, s))
                    n += _copy(sp, dp)
        else:
            n += _copy(s, d)
    if verbose:
        print(f"staged reference -> {DST} ({n} files copied)")
    return DST


def _copy(s, d):
    os.makedirs(os.path.dirname(d), exist_ok=True)
    if os.path.exists(d) and filecmp.cmp(s, d, shallow=False):
        return 0
    shutil.copyfile(s, d)
    return 1


if __name__ == "__main__":
    stage(sys.argv[1] if len(sys.argv) > 1 else None)
