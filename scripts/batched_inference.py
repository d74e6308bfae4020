"""Batched task inference against the per-image mirrors, on synthetic inputs at the full 896 x 448 geometry with
seeded random weights: Painter's "segm" task (painter_inference.run_one_image vs run_batch, PNGs written to a
temporary directory by both) and SegGPT with P = 1 and P = 3 prompts (seggpt_engine.segment vs segment_batch, the
finished images copied to the host by both), at B = 1, 2, 4, 8, 16 images per forward, in the fp32-accurate mode
(precision "auto" under no_grad, what the mirrors select) and in bf16.

For every (workload, precision, B) it processes --images images with each arm after one warm-up batch (which captures
the CUDA graph) and prints one JSON line: images/s (host clock, finished images on the host), CUDA-event time of the
timed window, the peak of allocated / reserved device memory from the warm-up on, the fp32-accurate workspace
estimate (accurate.workspace_bytes) and whether the batched results equal the mirror's bit for bit.  A batch the
fp32-accurate memory check refuses is reported as refused.  The card's name, power limit and max SM clock come first.

    python scripts/batched_inference.py [--images 16] [--batches 1,2,4,8,16] [--out batched.jsonl]
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
    ap.add_argument("--images", type=int, default=16, help="images per timed window and arm")
    ap.add_argument("--batches", default="1,2,4,8,16")
    ap.add_argument("--precisions", default="auto,bf16")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import numpy as np
    import torch
    from oracle import painter_oracle as po
    from _common import build_model
    from painter_b200 import accurate
    from painter_b200 import painter_inference as pi
    from painter_b200 import seggpt_engine as se

    if not torch.cuda.is_available():
        raise SystemExit("batched_inference: needs a GPU")
    print("card (name, power limit, max SM clock):", card(), flush=True)
    batches = [int(b) for b in args.batches.split(",")]
    n_img = args.images
    rng = np.random.RandomState(0)
    canv = [(rng.randn(896, 448, 3), rng.randn(896, 448, 3)) for _ in range(4)]
    sizes = [(640, 427), (512, 512), (301, 523), (683, 512)]
    dev = torch.device("cuda")
    tmp = tempfile.mkdtemp()
    out_f = open(args.out, "w") if args.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if out_f:
            out_f.write(line + "\n")

    def drop(m):
        m.__dict__.pop("_pk_graphed", None)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    def timed(fn, n_calls):
        t0 = time.perf_counter()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        res = [fn(k) for k in range(n_calls)]
        e1.record()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, e0.elapsed_time(e1) / 1e3, res

    painter, _ = build_model(po.PainterConfig(), 1)
    painter.eval()
    seggpt, _ = build_model(po.PainterConfig(seggpt=True), 3)
    seggpt.eval()
    seggpt.seg_type = "instance"
    g = torch.Generator().manual_seed(0)
    queries = torch.randint(0, 256, (16, 448, 448, 3), generator=g, dtype=torch.uint8).cuda()
    prompt_set = [(torch.randint(0, 256, (448, 448, 3), generator=g, dtype=torch.uint8).cuda(),
                   torch.randint(0, 256, (448, 448, 3), generator=g, dtype=torch.uint8).cuda()) for _ in range(3)]

    def painter_arms(B):
        def one(k):
            i = k % 4
            return pi.run_one_image(canv[i][0], canv[i][1], sizes[i], painter, os.path.join(tmp, f"o{k}.png"),
                                    dev).cpu()

        def batch(k):
            idx = [(k * B + j) % 4 for j in range(B)]
            res = pi.run_batch([canv[i][0] for i in idx], [canv[i][1] for i in idx], [sizes[i] for i in idx],
                               painter, dev, "segm", out_paths=[os.path.join(tmp, f"b{k}_{j}.png") for j in range(B)])
            return [r.cpu() for r in res]
        return painter, one, batch, 1

    def seggpt_arms(P):
        def arms(B):
            prompts = prompt_set[:P]

            def one(k):
                return se.segment(seggpt, dev, queries[k % 16], prompts)[0].cpu()

            def batch(k):
                q = torch.stack([queries[(k * B + j) % 16] for j in range(B)])
                out, _ = se.segment_batch(seggpt, dev, q, prompts)
                return list(out.cpu().unbind(0))
            return seggpt, one, batch, P
        return arms

    workloads = [("painter_segm", painter_arms), ("seggpt_P1", seggpt_arms(1)), ("seggpt_P3", seggpt_arms(3))]
    for prec in args.precisions.split(","):
        for name, make in workloads:
            base = None
            for B in batches:
                model, one, batch, P = make(B)
                model.precision = prec
                rec = {"workload": name, "precision": "fp32-accurate" if prec == "auto" else prec, "B": B,
                       "members_per_forward": B * P * (2 if name.startswith("seggpt") else 1)}
                rec["est_accurate_GiB"] = round(accurate.workspace_bytes(model, B * P, 896, 448) / 2**30, 2)
                with torch.no_grad():
                    if base is None:     # the per-image mirror, measured once per workload and precision
                        drop(model)
                        torch.cuda.reset_peak_memory_stats()
                        one(0)
                        wall, gpu, ref = timed(one, n_img)
                        base = {"img_s": n_img / wall, "gpu_s": gpu, "res": ref,
                                "peak_GiB": torch.cuda.max_memory_allocated() / 2**30}
                    drop(model)
                    torch.cuda.reset_peak_memory_stats()
                    try:
                        batch(0)
                    except RuntimeError as e:
                        if "fp32-accurate forward of" not in str(e):
                            raise
                        rec["refused"] = str(e)
                        emit(rec)
                        continue
                    n_calls = max(1, n_img // B)
                    wall, gpu, res = timed(batch, n_calls)
                flat = [r for rs in res for r in rs]
                same = all(torch.equal(flat[j], base["res"][j % len(base["res"])])
                           for j in range(min(len(flat), len(base["res"]))))
                rec.update({"mirror_img_s": round(base["img_s"], 2), "batch_img_s": round(n_calls * B / wall, 2),
                            "speedup": round(n_calls * B / wall / base["img_s"], 3),
                            "mirror_gpu_ms_per_img": round(base["gpu_s"] / n_img * 1e3, 2),
                            "batch_gpu_ms_per_img": round(gpu / (n_calls * B) * 1e3, 2),
                            "mirror_peak_alloc_GiB": round(base["peak_GiB"], 2),
                            "batch_peak_alloc_GiB": round(torch.cuda.max_memory_allocated() / 2**30, 2),
                            "batch_peak_reserved_GiB": round(torch.cuda.max_memory_reserved() / 2**30, 2),
                            "bit_identical": bool(same)})
                emit(rec)
            drop(painter)
            drop(seggpt)
            painter.precision = seggpt.precision = "bf16"


if __name__ == "__main__":
    main()
