"""Per-call time of the Painter eval scripts' `run_one_image` against the painter_b200 mirrors.

    python scripts/gpu_check_painter_tasks.py [--calls N] [--warmup W] [--sizes 448x448,640x480,...]
                                              [--precisions bf16,fp32]

For each task family (bilinear PNG: coco_panoptic/painter_inference_pano_semseg.py; nearest PNG:
painter_inference_pano_inst.py; depth PNG: nyuv2_depth/painter_inference_depth.py; restoration array:
sidd/painter_inference_sidd.py), each output size and precision "bf16" and "fp32", the unmodified reference function
driving the painter_b200 Painter ViT-L (896 x 448, seeded random weights) under torch.no_grad() is timed against the
mirror in painter_b200.painter_inference on the same module and inputs.  Both arms return host data or write a file,
so each call ends in a device synchronise; a host clock is read around every call, after a warm-up, with the two arms
alternating call by call.  Prints one JSON line per (family, size, precision) with the per-call median and mean of
both arms, and the card's name, power limit and max SM clock read in the same run.  PNGs go to a temporary directory;
nothing is written into the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = [(448, 448), (256, 256), (600, 400), (640, 480), (640, 427), (301, 523), (896, 896), (13, 9)]
# family -> (reference script key in tests/_painter_eval.EVAL_SCRIPTS, mirror, the script reads model.module.*)
FAMILIES = {
    "bilinear_png": ("pano_semseg", "run_one_image", True),
    "nearest_png": ("pano_inst", "run_one_image_nearest", True),
    "depth_png": ("depth", "run_one_image_depth", False),
    "restore_array": ("sidd", "run_one_image_restore", False),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20, help="timed calls per arm (at least 20)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sizes", default=",".join(f"{w}x{h}" for w, h in SIZES), help="WxH list of output sizes")
    ap.add_argument("--precisions", default="bf16,fp32")
    args = ap.parse_args()
    assert args.calls >= 20, "--calls: at least 20 per arm"
    import numpy as np
    import torch
    from oracle import painter_oracle as po
    from oracle import ref_loader
    from _common import build_model
    from _painter_eval import painter_eval
    from painter_b200 import painter_inference as ours

    if not torch.cuda.is_available():
        raise SystemExit("gpu_check_painter_tasks: needs a GPU")
    if not ref_loader.available():
        raise SystemExit("gpu_check_painter_tasks: reference tree not found (scripts/stage_reference.py)")
    sizes = [tuple(int(v) for v in s.split("x")) for s in args.sizes.split(",")]
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()

    class Wrapped(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.module = m

        def forward(self, *a, **k):
            return self.module(*a, **k)

    wrapped = Wrapped(model)
    dev = torch.device("cuda")
    rng = np.random.RandomState(0)
    img, tgt = rng.randn(896, 448, 3), rng.randn(896, 448, 3)
    with tempfile.TemporaryDirectory() as tmp:
        o_ref, o_our = os.path.join(tmp, "ref.png"), os.path.join(tmp, "our.png")
        for precision in args.precisions.split(","):
            model.precision = precision
            for fam, (script, mirror, use_wrapper) in FAMILIES.items():
                ref_fn = painter_eval(script).run_one_image
                our_fn = getattr(ours, mirror)
                m = wrapped if use_wrapper else model

                def ref_call(size):
                    with torch.no_grad():
                        ref_fn(img, tgt, size, m, o_ref, dev)

                def our_call(size):
                    our_fn(img, tgt, size, m, o_our, dev)
                    torch.cuda.synchronize()

                for size in sizes:
                    for _ in range(args.warmup):
                        ref_call(size)
                        our_call(size)
                    torch.cuda.synchronize()
                    t_ref, t_our = [], []
                    for _ in range(args.calls):
                        for fn, acc in ((ref_call, t_ref), (our_call, t_our)):
                            t0 = time.perf_counter()
                            fn(size)
                            acc.append((time.perf_counter() - t0) * 1e3)
                    d = {"family": fam, "reference": script, "mirror": mirror, "size": f"{size[0]}x{size[1]}",
                         "precision": precision, "calls": args.calls,
                         "ref_ms_median": round(statistics.median(t_ref), 3),
                         "mirror_ms_median": round(statistics.median(t_our), 3),
                         "ref_ms_mean": round(statistics.fmean(t_ref), 3),
                         "mirror_ms_mean": round(statistics.fmean(t_our), 3),
                         "card": info}
                    print(json.dumps(d), flush=True)


if __name__ == "__main__":
    main()
