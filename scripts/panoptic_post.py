"""COCO panoptic instance post-processing: the reference's per-image post_process_segm_output_by_threshold (the staged
copy, torch on CUDA) against painter_b200.panoptic.decode_instances on seeded synthetic 640 x 480 painted images, batch
8; the per-stage event times of one batch; and the intersection Gram kernel's achieved rate.

    python scripts/panoptic_post.py [--batch 8] [--reps 5] [--ref-images 4]

Prints the card name and power limit with the numbers.  Writes nothing into the repository (PNG files for the reference
go to a temporary directory)."""
import argparse
import ctypes
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from painter_b200 import panoptic as pn          # noqa: E402
from painter_b200._lib import check, lib        # noqa: E402

INT8_DENSE_TOPS = 1979.0                          # H100 SXM data sheet, dense int8 / fp8, 700 W


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                         # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-images", type=int, default=4)
    ap.add_argument("--blobs", type=int, default=30)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import _panoptic_eval as pe
    rng = np.random.default_rng(0)
    pal = pn.instance_palette().astype(np.int32)
    imgs = [pe.instance_image(rng, 480, 640, pal, blobs=a.blobs, jitter=8) for _ in range(a.batch)]
    dev = [torch.from_numpy(x).cuda() for x in imgs]
    print(f"card: {card()}")

    # ours: warm up, then whole batches
    for _ in range(2):
        pn.decode_instances(dev, dist_thr=19.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.reps):
        out = pn.decode_instances(dev, dist_thr=19.0)
    torch.cuda.synchronize()
    ours_ms = (time.perf_counter() - t0) * 1e3 / (a.reps * a.batch)
    print(f"ours: {ours_ms:.3f} ms per image (batch {a.batch}, {a.reps} batches, host clock around synchronised "
          f"batches; instances per image {[len(o) for o in out]})")

    # stage breakdown of one batch (events between stages; a stage includes its allocations)
    marks = []

    def tick(name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append((name, e))
    pn.decode_instances(dev, dist_thr=19.0, _timer=tick)
    torch.cuda.synchronize()
    print("stages (ms per batch):")
    for (n0, e0), (_, e1) in zip(marks, marks[1:]):
        print(f"  {n0:<11s} {e0.elapsed_time(e1):8.3f}")

    # the Gram kernel alone on the kept candidates of this batch
    from painter_b200.seggpt_engine import _stream
    n = a.batch
    ncap = pn._round128(pn.PRE_NMS_TOPK)
    words = pn._words(480 * 640)
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, (n, ncap, words), dtype=torch.int32, device="cuda")
    count = torch.full((n,), pn.PRE_NMS_TOPK, dtype=torch.int32, device="cuda")
    gram = torch.empty((n, ncap, ncap), dtype=torch.int32, device="cuda")

    def run():
        check(lib().pk_pano_gram(ctypes.c_void_p(bits.data_ptr()), n, ncap, words, ctypes.c_void_p(count.data_ptr()),
                                 ctypes.c_void_p(gram.data_ptr()), _stream()), "pk_pano_gram")
    for _ in range(3):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iters = 20
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    tiles = ncap // 128
    ops = 2.0 * n * (tiles * (tiles + 1) // 2) * 128 * 128 * words * 32      # AND + popcount per bit pair
    bytes_ = n * (tiles * (tiles + 1) // 2) * 2 * 128 * words * 4              # operand rows read per tile (L2)
    tops = ops / ms / 1e9
    print(f"gram (b1 mma.sync, {n} x {ncap} x {ncap} upper tiles x {words * 32} bits): {ms:.3f} ms per batch, "
          f"{tops:.1f} T bit-ops/s = {tops / INT8_DENSE_TOPS * 100:.1f}% of the {INT8_DENSE_TOPS:.0f} TOPS dense int8 "
          f"figure; HBM-side bound {n * ncap * words * 4 / 3.35e12 * 1e3:.3f} ms (rows read once), tile re-reads "
          f"{bytes_ / 1e9:.2f} GB from L2: compute-bound")
    # exactness spot check of the Gram against a popcount on the host
    b0 = bits[0, :64].cpu().numpy().view(np.uint32)
    pc = np.unpackbits(b0.view(np.uint8), axis=1).astype(np.int64)
    want = pc @ pc.T
    got = gram[0, :64, :64].cpu().numpy()
    iu = np.triu_indices(64)
    assert np.array_equal(got[iu], want[iu]), "gram mismatch"
    print("gram exactness spot check: ok")

    # the reference, per image (PNG round trip as eval.sh does it), on the first ref-images images
    ev = pe.inst_evaluator(dist_thr=19.0)
    from PIL import Image
    with tempfile.TemporaryDirectory() as d:
        paths = []
        for i, x in enumerate(imgs[:a.ref_images]):
            p = os.path.join(d, f"{i}.png")
            Image.fromarray(x).save(p)
            paths.append(p)
        ev.post_process_segm_output_by_threshold(paths[0], dist_thr_list=[19.0])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for p in paths:
            r = ev.post_process_segm_output_by_threshold(p, dist_thr_list=[19.0])
            r["instances"].scores.cpu()
        torch.cuda.synchronize()
        ref_ms = (time.perf_counter() - t0) * 1e3 / len(paths)
    print(f"reference: {ref_ms:.1f} ms per image ({len(paths)} images); speed-up {ref_ms / ours_ms:.1f}x")


if __name__ == "__main__":
    main()
