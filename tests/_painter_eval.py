"""TEST INFRASTRUCTURE: the UNMODIFIED `Painter/eval/<task>/painter_inference_*.py` scripts (their run_one_image),
loaded through oracle/ref_loader.py from a checkout of the reference or the staged copy under oracle/_ref
(scripts/stage_reference.py).  Used by tests/test_gpu_painter_tasks.py and scripts/gpu_check_painter_tasks.py.
"""
import importlib
import os
import sys
import types

from oracle import ref_loader

# key -> (directory under Painter/eval, script name)
EVAL_SCRIPTS = {
    "ade20k_semantic": ("ade20k_semantic", "painter_inference_segm"),
    "pano_semseg": ("coco_panoptic", "painter_inference_pano_semseg"),
    "pano_inst": ("coco_panoptic", "painter_inference_pano_inst"),
    "pose": ("mmpose_custom", "painter_inference_pose"),
    "depth": ("nyuv2_depth", "painter_inference_depth"),
    "sidd": ("sidd", "painter_inference_sidd"),
    "lol": ("lol", "painter_inference_lol"),
    "derain": ("derain", "painter_inference_derain"),
}

_cache = {}


def _raise_unavailable(*_a, **_k):
    raise RuntimeError("skimage.metrics is not installed: this stand-in only lets the eval script import")


def painter_eval(task):
    """Painter/eval/<dir>/<script>.py for a key of EVAL_SCRIPTS.

    The scripts import matplotlib.pyplot (unused by run_one_image), their sibling `models_painter` by bare name, and
    the restoration scripts skimage.metrics' peak_signal_noise_ratio / structural_similarity at module level (only
    their dataset loops call them).  For the duration of the import only, absent matplotlib / skimage modules are
    replaced by empty stand-ins (the skimage functions raise if called) and `models_painter` is the reference's."""
    if task not in _cache:
        sub, name = EVAL_SCRIPTS[task]
        d = os.path.join(ref_loader.REF_ROOT, "Painter")
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

        provide("matplotlib.pyplot")
        provide("skimage.metrics", {"peak_signal_noise_ratio": _raise_unavailable,
                                    "structural_similarity": _raise_unavailable})
        had_mp = sys.modules.get("models_painter")
        sys.modules["models_painter"] = ref_loader.models_painter()
        try:
            _cache[task] = ref_loader._load("ref_eval_" + name, os.path.join(d, "eval", sub, name + ".py"), d)
        finally:
            for n in injected:
                sys.modules.pop(n, None)
            if had_mp is None:
                sys.modules.pop("models_painter", None)
            else:
                sys.modules["models_painter"] = had_mp
    return _cache[task]
