"""Task metrics from batched inference: the reference's PNG round trip against the device meters
(painter_b200.task_metrics), on synthetic inputs with the same Painter (full 896 x 448 geometry, seeded random
weights) for both arms.

    segm   reference: run_batch(task="segm", out_paths=...) writes the PNGs; per image a PIL read, the staged
           evaluator's post_process_segm_output (on the GPU, as the reference runs it) and np.bincount
           ours:      run_batch(task="segm") -> SemSegMeter.update on the device images
           ADE20K-sized images (683 x 512 and 512 x 683), the ADE20K palette
    depth  reference: run_batch(task="depth", out_paths=...) writes the PNGs; cv2.imread(-1) of each, then the staged
           eval_with_pngs.eval() (eval.sh's arguments)
           ours:      run_batch(task="depth") -> DepthMeter.update on the device maps
           NYUv2-sized images (640 x 480)
    derain reference: run_batch(task="restore"), the PNG painter_inference_derain.py writes ((clip(x, 0, 1) * 255)
           .astype(uint8)) written and read back with PIL, then oracle/matlab_ref.py's restatement of
           evaluate_PSNR_SSIM.m on the CPU (standing in for MATLAB)
           ours:      run_batch(task="restore") -> derain_scores
           Rain100-sized images (481 x 321 and 321 x 481)
    sidd   reference: run_batch(task="restore"), the float32 array painter_inference_sidd.py saves, then
           oracle/matlab_ref.py's restatement of eval_sidd.m's psnr / ssim on the CPU
           ours:      run_batch(task="restore") -> sidd_scores
           SIDD blocks (256 x 256)

For each task and arm it processes --images images (after one warm-up batch that captures the CUDA graph) and prints
one JSON line: images/s end to end (host clock; the metric state is on the host or synchronised at the end) and the
metric step alone in ms per image (CUDA events around the metric calls, the inference outputs already computed).  The
two semseg arms' confusion matrices are asserted equal, and the two depth arms' d1, d2, d3 (float32) likewise; the
derain and sidd arms' PSNR to 1e-13 relative and SSIM to 1e-12.  The
card's name, power limit and max SM clock come first.  Needs the staged reference (scripts/stage_reference.py).

    python scripts/task_metrics.py [--images 64] [--batch 8] [--tasks segm,depth,derain,sidd] [--out task_metrics.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64, help="images per timed window and arm")
    ap.add_argument("--batch", type=int, default=8, help="images per run_batch call")
    ap.add_argument("--tasks", default="segm,depth,derain,sidd")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import cv2
    import numpy as np
    import torch
    from PIL import Image
    import _task_eval
    from _common import build_model
    from oracle import painter_oracle as po
    from painter_b200 import painter_inference as pi
    from oracle import matlab_ref as mr
    from painter_b200.task_metrics import DepthMeter, SemSegMeter, derain_scores, sidd_scores

    if not torch.cuda.is_available():
        raise SystemExit("task_metrics: needs a GPU")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    tasks = set(args.tasks.split(","))
    n_img, B = args.images, args.batch
    n_calls = (n_img + B - 1) // B
    dev = torch.device("cuda")
    tmp = tempfile.mkdtemp()
    out_f = open(args.out, "w") if args.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out_f:
            out_f.write(line + "\n")

    model, _ = build_model(po.PainterConfig(), 1)
    model.eval()
    rng = np.random.RandomState(0)
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in range(4)]

    class Events:
        """CUDA events around each metric step; read after the window's final synchronise (no sync per step)."""
        def __init__(self):
            self.pairs = []

        def __enter__(self):
            self.pairs.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
            self.pairs[-1][0].record()

        def __exit__(self, *exc):
            self.pairs[-1][1].record()

        def ms(self):
            return sum(a.elapsed_time(b) for a, b in self.pairs)

    def run(task, sizes, k, paths=None):
        idx = [(k * B + j) % 4 for j in range(B)]
        return pi.run_batch([canv[i][0] for i in idx], [canv[i][1] for i in idx], [sizes[j % len(sizes)]
                            for j in range(B)], model, dev, task, out_paths=paths)

    # ---------------- semantic segmentation (ADE20K) ----------------
    palette = _task_eval.ade20k_palette()
    K = len(palette)
    decode = _task_eval.semseg_decoder("ade20k", palette, "abs")
    seg_sizes = [(683, 512), (512, 683)]
    gts = []
    for j in range(B):
        w, h = seg_sizes[j % 2]
        g = rng.randint(0, K, size=(h, w)).astype(np.uint8)
        g[rng.rand(h, w) < 0.05] = 255
        gts.append(g)

    def seg_reference(k, ev):
        paths = [os.path.join(tmp, f"s{k}_{j}.png") for j in range(B)]
        with torch.no_grad():
            run("segm", seg_sizes, k, paths)
        conf = np.zeros((K + 1) ** 2, dtype=np.int64)
        with ev:
            for p, g in zip(paths, gts):
                pred = decode(np.array(Image.open(p)))
                gt = g.astype(np.int64)
                gt[gt == 255] = K
                conf += np.bincount((K + 1) * pred.reshape(-1) + gt.reshape(-1), minlength=conf.size)
        return conf.reshape(K + 1, K + 1)

    def seg_ours(meter):
        def step(k, ev):
            with torch.no_grad():
                outs = run("segm", seg_sizes, k)
            with ev:
                meter.update(outs, gts)
        return step

    ref_conf = np.zeros((K + 1, K + 1), dtype=np.int64)

    def seg_ref_acc(k, ev):
        nonlocal ref_conf
        ref_conf = ref_conf + seg_reference(k, ev)

    # ---------------- NYUv2 depth ----------------
    dep_sizes = [(640, 480)]
    dgts = []
    for _ in range(B):
        g = rng.randint(0, 12001, size=(480, 640)).astype(np.uint16)
        g[rng.rand(480, 640) < 0.1] = 0
        dgts.append(g)
    ref_eval = _task_eval.depth_eval()
    ref_depth = []

    def dep_reference(k, ev):
        paths = [os.path.join(tmp, f"d{k}_{j}.png") for j in range(B)]
        with torch.no_grad():
            run("depth", dep_sizes, k, paths)
        with ev:
            preds = [cv2.imread(p, -1).astype(np.float32) / 1000.0 for p in paths]
            ref_eval.gt_depths = [g.astype(np.float32) / 1000.0 for g in dgts]
            ref_eval.missing_ids = set()
            ref_depth.append(np.stack(ref_eval.eval(preds), 1))

    def dep_ours(meter):
        def step(k, ev):
            with torch.no_grad():
                outs = run("depth", dep_sizes, k)
            with ev:
                meter.update(outs, dgts)
        return step

    def arm(task, name, step):
        step(0, Events())                        # warm-up: captures the graph, loads the modules
        torch.cuda.synchronize()
        ev = Events()
        t0 = time.perf_counter()
        for k in range(1, n_calls + 1):
            step(k, ev)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        emit({"task": task, "arm": name, "images": n_calls * B, "batch": B, "img_s": round(n_calls * B / wall, 2),
              "metric_ms_per_img": round(ev.ms() / (n_calls * B), 3)})

    if "segm" in tasks:
        arm("segm", "reference (PNG, PIL, post_process_segm_output, bincount)", seg_ref_acc)
        sm = SemSegMeter(palette)
        arm("segm", "run_batch -> SemSegMeter", seg_ours(sm))
        # both arms' state holds the warm-up batch and the timed ones: the same 1 + n_calls batches
        np.testing.assert_array_equal(sm.conf_matrix, ref_conf)
        emit({"task": "segm", "confusion_matrices_equal": True, "pixels": int(ref_conf.sum())})

    if "depth" in tasks:
        arm("depth", "reference (PNG, cv2, eval_with_pngs.eval)", dep_reference)
        dm = DepthMeter()
        arm("depth", "run_batch -> DepthMeter", dep_ours(dm))
        # columns of eval(): silog, log10, abs_rel, sq_rel, rms, log_rms, d1, d2, d3
        ref = np.concatenate(ref_depth)
        ours = dm.per_image()
        np.testing.assert_array_equal(ours[:, :3].astype(np.float32), ref[:, 6:9])
        np.testing.assert_allclose(ours[:, 3:], ref[:, [2, 3, 4, 5, 0, 1]], rtol=1e-5)
        emit({"task": "depth", "d1_d2_d3_equal": True, "others_within_1e-5": True, "images": len(ours)})

    # ---------------- derain and SIDD (scored in MATLAB by the reference) ----------------
    def restoration(task, sizes, ref_score, ours_score):
        rgts = []
        for j in range(B):
            w, h = sizes[j % len(sizes)]
            rgts.append(rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8))
        ref_out, ours_out = [], []

        def reference(k, ev):
            with torch.no_grad():
                outs = run("restore", sizes, k)
            with ev:
                ref_out.extend(ref_score(k, j, o, g) for j, (o, g) in enumerate(zip(outs, rgts)))

        def ours(k, ev):
            with torch.no_grad():
                outs = run("restore", sizes, k)
            with ev:
                ours_out.append(np.stack(ours_score(outs, rgts), 1))

        return reference, ours, ref_out, ours_out

    def derain_ref(k, j, o, g):
        path = os.path.join(tmp, f"r{k}_{j}.png")
        Image.fromarray((np.clip(o, 0, 1) * 255).astype(np.uint8)).save(path)
        return mr.derain_scores_u8(np.array(Image.open(path)), g)

    def sidd_ref(k, j, o, g):
        x, y = mr.sidd_inputs(o, g)
        return mr.sidd_psnr(x, y), mr.sidd_ssim(x, y)

    for task, sizes, ref_score, ours_score, ref_name in [
            ("derain", [(481, 321), (321, 481)], derain_ref, derain_scores,
             "reference (PNG, PIL, evaluate_PSNR_SSIM.m restated on the CPU)"),
            ("sidd", [(256, 256)], sidd_ref, sidd_scores, "reference (float32 array, eval_sidd.m restated on the CPU)")]:
        if task not in tasks:
            continue
        reference, ours, ref_out, ours_out = restoration(task, sizes, ref_score, ours_score)
        arm(task, ref_name, reference)
        arm(task, f"run_batch -> {ours_score.__name__}", ours)
        ref, mine = np.array(ref_out), np.concatenate(ours_out)
        assert ref.shape == mine.shape, (ref.shape, mine.shape)
        fin = np.isfinite(ref[:, 0])
        assert np.array_equal(np.isfinite(mine[:, 0]), fin)
        assert np.all(np.abs(mine[fin, 0] - ref[fin, 0]) <= 1e-13 * np.abs(ref[fin, 0])), "PSNR"
        assert np.all(np.abs(mine[:, 1] - ref[:, 1]) <= 1e-12), "SSIM"
        emit({"task": task, "psnr_within_1e-13_rel": True, "ssim_within_1e-12": True, "images": len(ref),
              "mean_psnr": float(np.mean(mine[:, 0])), "mean_ssim": float(np.mean(mine[:, 1]))})


if __name__ == "__main__":
    main()
