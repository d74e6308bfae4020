"""Per-shape timing of the block-level GEMMs of the training step (B = 8: M = 12544 tokens) with rotating operand
copies (working set > L2), CUDA events on the launching stream.  PK_LIB selects a tuning build.

    python scripts/time_gemms.py                      # the twelve GEMMs of one block (fwd + bwd) and their sum
    python scripts/time_gemms.py --ksweep             # + qkv-fwd- and fc2-fwd-shaped calls at K = 256 .. 4096; a
                                                      #   linear fit of time over (tiles per CTA x K-blocks) gives
                                                      #   the time per tile outside the K loop and per K-block
    python scripts/time_gemms.py --libs A.so B.so     # each library in its own process (PK_LIB), alternating
    python scripts/time_gemms.py --libs A.so B.so --rounds 2 --ksweep
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

M, C = 12544, 1024
R = 3   # rotating copies
SMS = 132


def run_cases(ksweep, cublas, iters):
    import torch
    from painter_b200 import ops

    dev = "cuda"
    torch.manual_seed(0)

    def rnd(*shape, dtype=torch.bfloat16, scale=1.0):
        return [(torch.randn(*shape, device=dev) * scale).to(dtype) for _ in range(R)]

    x, x3, x4 = rnd(M, C), rnd(M, 3 * C), rnd(M, 4 * C)
    wqkv, wproj = rnd(3 * C, C, scale=0.02), rnd(C, C, scale=0.02)
    wfc1, wfc2 = rnd(4 * C, C, scale=0.02), rnd(C, 4 * C, scale=0.02)
    b1, b3, b4 = torch.randn(C, device=dev), torch.randn(3 * C, device=dev), torch.randn(4 * C, device=dev)
    res = rnd(M, C, dtype=torch.float32)
    z = rnd(M, 4 * C)
    g4 = [torch.zeros(4 * C, C, device=dev) for _ in range(R)]
    g4t = [torch.zeros(C, 4 * C, device=dev) for _ in range(R)]
    g3 = [torch.zeros(3 * C, C, device=dev) for _ in range(R)]
    g1 = [torch.zeros(C, C, device=dev) for _ in range(R)]
    F1, F3, F4 = 2.0 * M * C * C, 2.0 * M * 3 * C * C, 2.0 * M * 4 * C * C

    # (name, flops, fn, counted in the block sum)
    cases = [
        ("qkv fwd   N=3072 K=1024 bf16+bias", F3, lambda i: ops.gemm(x[i], wqkv[i], kind=ops.EPI_BF16, bias=b3), 1),
        ("proj fwd  N=1024 K=1024 resid", F1,
         lambda i: ops.gemm(x[i], wproj[i], kind=ops.EPI_RESID, bias=b1, aux=res[i]), 1),
        ("fc1 fwd   N=4096 K=1024 gelu", F4, lambda i: ops.gemm(x[i], wfc1[i], kind=ops.EPI_GELU, bias=b4), 1),
        ("fc2 fwd   N=1024 K=4096 resid", F4,
         lambda i: ops.gemm(x4[i], wfc2[i], kind=ops.EPI_RESID, bias=b1, aux=res[i]), 1),
        ("fc2 wgrad 1024x4096 K=12544", F4,
         lambda i: ops.gemm(x[i], x4[i], trans_a=True, trans_b=True, kind=ops.EPI_F32, out=g4t[i], accumulate=2), 1),
        ("fc2 dgrad N=4096 K=1024 dgelu", F4,
         lambda i: ops.gemm(x[i], wfc2[i], trans_b=True, kind=ops.EPI_DGELU, aux=z[i]), 1),
        ("fc1 wgrad 4096x1024 K=12544", F4,
         lambda i: ops.gemm(x4[i], x[i], trans_a=True, trans_b=True, kind=ops.EPI_F32, out=g4[i], accumulate=2), 1),
        ("fc1 dgrad N=1024 K=4096 bf16", F4, lambda i: ops.gemm(x4[i], wfc1[i], trans_b=True, kind=ops.EPI_BF16), 1),
        ("proj wgrad 1024x1024 K=12544", F1,
         lambda i: ops.gemm(x[i], x[(i + 1) % R], trans_a=True, trans_b=True, kind=ops.EPI_F32, out=g1[i],
                            accumulate=2), 1),
        ("proj dgrad N=1024 K=1024 bf16", F1, lambda i: ops.gemm(x[i], wproj[i], trans_b=True, kind=ops.EPI_BF16), 1),
        ("qkv wgrad 3072x1024 K=12544", F3,
         lambda i: ops.gemm(x3[i], x[i], trans_a=True, trans_b=True, kind=ops.EPI_F32, out=g3[i], accumulate=2), 1),
        ("qkv dgrad N=1024 K=3072 bf16", F3, lambda i: ops.gemm(x3[i], wqkv[i], trans_b=True, kind=ops.EPI_BF16), 1),
        # windowed blocks keep the input gradient in fp32 (not part of the global block's sum)
        ("qkv dgrad N=1024 K=3072 f32 (windowed)", F3,
         lambda i: ops.gemm(x3[i], wqkv[i], trans_b=True, kind=ops.EPI_F32), 0),
    ]
    if ksweep:
        for K in (256, 512, 1024, 2048, 4096):
            xa = rnd(M, K)
            wa, wb = rnd(3 * C, K, scale=0.02), rnd(C, K, scale=0.02)
            cases.append((f"ksweep qkv-fwd  N=3072 K={K}", 2.0 * M * 3 * C * K,
                          (lambda xa, wa: lambda i: ops.gemm(xa[i], wa[i], kind=ops.EPI_BF16, bias=b3))(xa, wa), 0))
            cases.append((f"ksweep fc2-fwd  N=1024 K={K}", 2.0 * M * C * K,
                          (lambda xa, wb: lambda i: ops.gemm(xa[i], wb[i], kind=ops.EPI_RESID, bias=b1, aux=res[i]))(
                              xa, wb), 0))
    if cublas:
        cases += [
            ("cuBLAS    N=3072 K=1024 (torch.matmul)", F3, lambda i: torch.matmul(x[i], wqkv[i].t()), 0),
            ("cuBLAS    N=4096 K=1024 (torch.matmul)", F4, lambda i: torch.matmul(x[i], wfc1[i].t()), 0),
            ("cuBLAS    N=1024 K=4096 (torch.matmul)", F4, lambda i: torch.matmul(x4[i], wfc2[i].t()), 0),
            ("cuBLAS    N=1024 K=1024 (torch.matmul)", F1, lambda i: torch.matmul(x[i], wproj[i].t()), 0),
        ]

    out = []
    for name, flops, fn, counted in cases:
        for i in range(3):
            fn(i % R)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            fn(i % R)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / iters * 1e3
        out.append({"name": name, "us": us, "tflops": flops / us / 1e6, "counted": counted})
    return out


def ksweep_fit(rows, which):
    """Least-squares fit of us = a * tiles_per_cta + b * tiles_per_cta * K-blocks over the sweep of one shape:
    a = time per tile outside the K loop, b = time per 128 x BN x 64 K-block, both per CTA."""
    import numpy as np
    pts = []
    for r in rows:
        if r["name"].startswith(f"ksweep {which}"):
            K = int(r["name"].split("K=")[1])
            N = 3072 if which == "qkv-fwd" else 1024
            pts.append((K, N, r["us"]))
    if not pts:
        return None
    out = {}
    for bn in (128, 256):
        tiles = -(-M // 128) * pts[0][1] // bn
        tpc = -(-tiles // SMS)
        X = np.array([[tpc, tpc * (K // 64)] for K, _, _ in pts], dtype=np.float64)
        y = np.array([u for _, _, u in pts])
        (a, b), *_ = np.linalg.lstsq(X, y, rcond=None)
        out[f"BN{bn}"] = {"us_per_tile_outside_k_loop": float(a), "us_per_kblock": float(b)}
    return out


def child(args):
    rows = run_cases(args.ksweep, args.cublas, args.iters)
    print("JSON " + json.dumps(rows), flush=True)


def report(label, rows):
    tot = 0.0
    print(f"== {label}")
    for r in rows:
        if r["counted"]:
            tot += r["us"]
        print(f"  {r['name']:42s} {r['us']:8.1f} us  {r['tflops']:7.0f} TFLOP/s")
    print(f"  sum over one block's twelve GEMMs (fwd + bwd): {tot:.1f} us")
    for which in ("qkv-fwd", "fc2-fwd"):
        fit = ksweep_fit(rows, which)
        if fit:
            print(f"  ksweep fit {which}: {json.dumps(fit)}")
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ksweep", action="store_true")
    ap.add_argument("--cublas", action="store_true", default=bool(os.environ.get("PK_CUBLAS")))
    ap.add_argument("--libs", nargs="+", default=None, help="shared libraries to compare, one process each")
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child or not args.libs:
        if args.child:
            return child(args)
        return report(os.environ.get("PK_LIB", "in-tree library"), run_cases(args.ksweep, args.cublas, args.iters))
    results = {lib: [] for lib in args.libs}
    for rnd_ in range(args.rounds):
        for lib in args.libs:
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--iters", str(args.iters)]
            if args.ksweep:
                cmd.append("--ksweep")
            if args.cublas:
                cmd.append("--cublas")
            env = dict(os.environ, PK_LIB=os.path.abspath(lib))
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f"{lib}: child failed")
            rows = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("JSON ")][-1][5:])
            results[lib].append(rows)
            report(f"round {rnd_ + 1}: {lib}", rows)
    # per-shape comparison: best and worst round of each library
    print("== summary (min .. max over rounds, us)")
    names = [r["name"] for r in results[args.libs[0]][0]]
    for k, name in enumerate(names):
        cols = []
        for lib in args.libs:
            us = [rows[k]["us"] for rows in results[lib]]
            cols.append(f"{min(us):8.1f} .. {max(us):8.1f}")
        print(f"  {name:42s} " + " | ".join(cols))
    for lib in args.libs:
        sums = [sum(r["us"] for r in rows if r["counted"]) for rows in results[lib]]
        print(f"  block sum {lib}: " + ", ".join(f"{s:.1f}" for s in sums))


if __name__ == "__main__":
    main()
