"""COCO pose post-processing: the reference flow (the staged top_down.py / topdown_coco_dataset.py with the restated
mmpose 0.29 pieces of oracle/mmpose_ref.py) against painter_b200.pose, both from the same seeded synthetic painted
256 x 192 crops and their flipped paintings.

    python scripts/pose_post.py [--images 40] [--boxes 24] [--reps 3]

Reference arm: the PNG pairs are written (not timed), then forward_pseudo_test in batches of 32 and evaluate, which
writes result_keypoints.json (timed).  GPU arm: decode_keypoints per batch of 32 on device tensors, then one
pose_results for the dataset (timed, host clock around synchronised runs).  Prints ms per box for each arm, whether
the two outputs are identical, and the card's name, power limit and SM clocks in the same run.  Writes nothing into
the repository (PNG and JSON files go to a temporary directory)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from painter_b200 import pose  # noqa: E402

BATCH = 32


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                         # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=40)
    ap.add_argument("--boxes", type=int, default=24, help="boxes per image")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import _pose_eval as pe
    from oracle import mmpose_ref as mr
    preds, flipped, c, s, scores, image_ids, bbox_ids, names = pe.dataset_stream(0, counts=(a.boxes,) * a.images,
                                                                                repeats=8)
    n = len(preds)
    print(f"card: {card()}")
    print(f"{n} boxes ({a.images} images, {len(set(bbox_ids.tolist()))} distinct bbox ids), 256 x 192 crops")

    with tempfile.TemporaryDirectory() as tmp:
        paths = pe.write_pngs(tmp, names, preds, flipped)
        mdl = pe.model(flip_test=True)
        ann = mr.write_image_list(os.path.join(tmp, "ann.json"), {f"{i:012d}.jpg": int(i) for i in set(image_ids)})
        ds = pe.dataset(ann, os.path.join(tmp, "crops") + "/")
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        results = []
        for b in range(0, n, BATCH):
            sl = slice(b, b + BATCH)
            results.append(pe.forward_pseudo_test(mdl, paths[sl], c[sl], s[sl], scores[sl], bbox_ids[sl],
                                                  pose.COCO_FLIP_PAIRS))
        t1 = time.perf_counter()
        mr.quiet(ds.evaluate, results, res_folder=tmp)
        t2 = time.perf_counter()
        with open(os.path.join(tmp, "result_keypoints.json")) as f:
            want = json.load(f)
    ref_ms = (t2 - t0) * 1e3 / n
    print(f"reference: {ref_ms:.3f} ms per box (forward_pseudo_test {(t1 - t0) * 1e3 / n:.3f}, evaluate "
          f"{(t2 - t1) * 1e3 / n:.3f})")

    dev = [torch.from_numpy(x).cuda() for x in preds]
    fdev = [torch.from_numpy(x).cuda() for x in flipped]

    def run():
        kp = torch.cat([pose.decode_keypoints(dev[b:b + BATCH], c[b:b + BATCH], s[b:b + BATCH],
                                              flipped=fdev[b:b + BATCH]) for b in range(0, n, BATCH)])
        return kp, pose.pose_results(kp, c, s, scores, image_ids, bbox_ids)

    for _ in range(2):
        run()
    torch.cuda.synchronize()
    best_dec = best_all = float("inf")
    for _ in range(a.reps):
        t0 = time.perf_counter()
        kp = torch.cat([pose.decode_keypoints(dev[b:b + BATCH], c[b:b + BATCH], s[b:b + BATCH],
                                              flipped=fdev[b:b + BATCH]) for b in range(0, n, BATCH)])
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        got = pose.pose_results(kp, c, s, scores, image_ids, bbox_ids)
        t2 = time.perf_counter()
        best_dec, best_all = min(best_dec, t1 - t0), min(best_all, t2 - t0)
    ours_ms = best_all * 1e3 / n
    print(f"ours: {ours_ms:.4f} ms per box (decode_keypoints {best_dec * 1e3 / n:.4f}, pose_results "
          f"{(best_all - best_dec) * 1e3 / n:.4f}; best of {a.reps})")
    same = got == want
    print(f"outputs identical: {same} ({len(got)} results, reference {len(want)}); speed-up {ref_ms / ours_ms:.1f}x")
    print(f"card after: {card()}")
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
