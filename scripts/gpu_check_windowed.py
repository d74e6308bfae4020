"""Timings of windowed-block inference in the fp32-accurate mode, with CUDA events.

    python scripts/gpu_check_windowed.py [--iters N] [--out FILE]

(a) the fused split attention forward (ops.attn_fwd_split3) against the materialised fp32-accurate attention
    (accurate.attention: score matrix per (window, head)) on the same qkv and tables, at the ViT-L window geometry
    (16 windows, 16 heads, 14 x 14) and at the global 56 x 28 geometry (2 samples, 16 heads), with the error of both
    against an fp64 restatement;
(b) seggpt_engine.run_one_image on SegGPT ViT-L with 16 windowed (ws = 14) and 8 global blocks, P = 1 and P = 3, in
    the fp32-accurate mode and in bf16 (synthetic weights and images).
Prints the card, its power limit and max SM clock, then one JSON line per measurement (also written to --out).
Writes nothing into the tree.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WINDOWS_16 = (0, 1, 3, 4, 6, 7, 9, 10, 12, 13, 15, 16, 18, 19, 21, 22)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, iters, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def kernels(iters, emit):
    """Errors on one qkv (the materialised path through an identity qkv projection); times of the attention including
    the qkv projection of a random C -> 3C layer, as a block runs it, and of the fused kernel alone."""
    import types
    import torch
    from painter_b200 import accurate, ops
    from painter_b200.ops import EPI_F32
    from test_gpu_windowed_inference import _attn64, _materialised
    for name, B, heads, h, w in (("window_14x14", 16, 16, 14, 14), ("global_56x28", 2, 16, 56, 28)):
        g = torch.Generator().manual_seed(1)
        N, C = h * w, heads * 64
        qkv = torch.randn(B * N, 3 * C, generator=g).cuda()
        th = (torch.randn(2 * h - 1, 64, generator=g) * 0.1).cuda()
        tw = (torch.randn(2 * w - 1, 64, generator=g) * 0.1).cuda()
        ref = _attn64(qkv, th, tw, B, heads, h, w)
        e_f = ops.attn_fwd_split3(qkv, th, tw, B, heads, h, w)
        e_m = _materialised(qkv, th, tw, B, heads, h, w)
        err = {k: ((o.double() - ref).abs().max() / ref.abs().max()).item() for k, o in (("fused", e_f),
                                                                                         ("materialised", e_m))}
        del ref, e_f, e_m
        u = torch.randn(B * N, C, generator=g).cuda()
        lin = types.SimpleNamespace(weight=torch.nn.Parameter((torch.randn(3 * C, C, generator=g) * 0.05).cuda()),
                                    bias=torch.randn(3 * C, generator=g).cuda())
        blk = types.SimpleNamespace(attn=types.SimpleNamespace(qkv=lin))
        cache = {}

        def fused_block():
            q = accurate._gemm(accurate.split3(u), accurate.split_weight(lin.weight), kind=EPI_F32, bias=lin.bias)
            return ops.attn_fwd_split3(q, th, tw, B, heads, h, w)

        tk = timed(lambda: ops.attn_fwd_split3(qkv, th, tw, B, heads, h, w), iters)
        tf = timed(fused_block, iters)
        tm = timed(lambda: accurate.attention(u, blk, B, h, w, heads, cache, th, tw), max(3, iters // 4))
        emit(dict(kind="attention", geometry=name, B=B, heads=heads, h=h, w=w, fused_kernel_ms=round(tk, 4),
                  fused_with_qkv_ms=round(tf, 4), materialised_with_qkv_ms=round(tm, 4), speedup=round(tm / tf, 2),
                  err_fused=err["fused"], err_materialised=err["materialised"]))
        del cache


def run_one_image(iters, emit):
    import numpy as np
    from oracle import painter_oracle as po
    from oracle.synth import synth_inputs
    from _common import build_model
    from painter_b200 import seggpt_engine
    cfg = po.PainterConfig(seggpt=True, window_size=14, window_block_indexes=WINDOWS_16)
    model, _ = build_model(cfg, 4, precision="fp32")
    model.eval()
    model.seg_type = "instance"
    for P in (1, 3):
        x, t, _, _ = synth_inputs(cfg, P, 80 + P)
        img = np.ascontiguousarray(x.permute(0, 2, 3, 1).double().numpy())
        tgt = np.ascontiguousarray(t.permute(0, 2, 3, 1).double().numpy())
        for prec in ("fp32", "bf16"):
            model.precision = prec
            ms = timed(lambda: seggpt_engine.run_one_image(img, tgt, model, "cuda"), iters, warmup=2)
            emit(dict(kind="run_one_image", model="seggpt_vitl_16win_8glb", P=P, precision=prec, ms=round(ms, 3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("gpu_check_windowed.py needs a GPU")
    lines = []

    def emit(d):
        d["card"] = info
        print(json.dumps(d), flush=True)
        lines.append(d)

    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    kernels(a.iters, emit)
    run_one_image(max(3, a.iters // 4), emit)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(d) for d in lines) + "\n")


if __name__ == "__main__":
    main()
