"""TEST INFRASTRUCTURE: the UNMODIFIED reference evaluators and palette generators, loaded through oracle/ref_loader.py
from a checkout of the reference or the staged copy under oracle/_ref (scripts/stage_reference.py).  Used by
tests/test_gpu_task_metrics.py and scripts/task_metrics.py.

    Painter/eval/ade20k_semantic/ADE20kSemSegEvaluatorCustom.py      post_process_segm_output (ADE20K)
    Painter/eval/coco_panoptic/COCOPanoSemSegEvaluatorCustom.py      post_process_segm_output (COCO panoptic semseg)
    Painter/eval/nyuv2_depth/eval_with_pngs.py                       eval(), compute_errors()
    Painter/data/ade20k/gen_color_ade20k_sem.py                      the 150-colour ADE20K palette
    Painter/data/coco_semseg/gen_color_coco_panoptic_segm.py         the 133-colour COCO panoptic palette

For the duration of an import only, absent modules the files import but the functions used here do not need
(detectron2.evaluation, the COCO dataset registration, skimage.segmentation, panopticapi.utils, matplotlib) are
replaced by empty stand-ins.
"""
import argparse
import importlib
import json
import os
import sys
import types

import torch

from oracle import ref_loader

_cache = {}


def _painter_dir():
    return os.path.join(ref_loader.REF_ROOT, "Painter")


def _load(key, rel, standins=(), argv=None):
    if key in _cache:
        return _cache[key]
    injected = []

    def provide(modname, attrs=None):
        try:
            importlib.import_module(modname)
        except Exception:
            parts = modname.split(".")
            for i in range(1, len(parts) + 1):
                n = ".".join(parts[:i])
                if n not in sys.modules:
                    sys.modules[n] = types.ModuleType(n)
                    injected.append(n)
            for a, v in (attrs or {}).items():
                setattr(sys.modules[modname], a, v)

    for modname, attrs in standins:
        provide(modname, attrs)
    saved_argv = sys.argv
    if argv is not None:
        sys.argv = argv
    try:
        _cache[key] = ref_loader._load("ref_task_" + key, os.path.join(_painter_dir(), rel), _painter_dir())
    finally:
        sys.argv = saved_argv
        for n in injected:
            sys.modules.pop(n, None)
    return _cache[key]


class _SemSegEvaluator:          # stand-in base class: only post_process_segm_output is used
    pass


_EVALUATORS = {
    "ade20k": "eval/ade20k_semantic/ADE20kSemSegEvaluatorCustom.py",
    "coco": "eval/coco_panoptic/COCOPanoSemSegEvaluatorCustom.py",
}


def semseg_decoder(kind, palette, dist_type):
    """post_process_segm_output of the ADE20K or COCO evaluator, bound to `palette` and `dist_type` (its palette lives
    on the GPU, as in the reference): numpy uint8 [H, W, 3] -> numpy int [H, W]."""
    mod = _load("semseg_" + kind, _EVALUATORS[kind], standins=[
        ("matplotlib.pyplot", None),
        ("detectron2.evaluation", {"SemSegEvaluator": _SemSegEvaluator}),
        ("data.register_coco_panoptic_annos_semseg", None)])
    ev = mod.SemSegEvaluatorCustom.__new__(mod.SemSegEvaluatorCustom)
    ev.palette = torch.tensor(palette, dtype=torch.float, device="cuda")
    ev.dist_type = dist_type

    def decode(segm):
        out = ev.post_process_segm_output(segm)
        return out[0] if kind == "coco" else out       # the COCO evaluator also returns the distances
    return decode


def ade20k_palette():
    return list(_load("gen_color_ade20k", "data/ade20k/gen_color_ade20k_sem.py").define_colors_per_location_mean_sep())


def coco_palette():
    mod = _load("gen_color_coco", "data/coco_semseg/gen_color_coco_panoptic_segm.py", standins=[
        ("matplotlib.pyplot", None),
        ("skimage.segmentation", {"find_boundaries": None}),
        ("panopticapi.utils", {"rgb2id": None, "IdGenerator": None})])
    with open(os.path.join(_painter_dir(), "data", "panoptic_coco_categories.json")) as f:
        num_colors = len(json.load(f))
    return list(mod.define_colors_by_mean_sep(num_colors=num_colors).values())


def depth_eval(min_depth=1e-3, max_depth=10.0, eigen_crop=True):
    """eval_with_pngs as a module whose `args` are those of eval/nyuv2_depth/eval.sh (the script parses its arguments
    at import: it is imported with that command line).  The caller sets the globals eval() reads: gt_depths,
    missing_ids."""
    mod = _load("eval_with_pngs", "eval/nyuv2_depth/eval_with_pngs.py",
                argv=["eval_with_pngs.py", "--pred_path", "unused", "--dataset", "nyu"])
    mod.args = argparse.Namespace(pred_path="unused", gt_path=None, dataset="nyu", eigen_crop=eigen_crop,
                                  garg_crop=False, min_depth_eval=min_depth, max_depth_eval=max_depth,
                                  do_kb_crop=False)
    return mod
