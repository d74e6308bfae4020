"""GPU bring-up check of the wgmma GEMM (runs every case in a subprocess so that a trapped kernel
does not poison the rest).  Usage on the GPU box:  python scripts/gpu_check_gemm.py [--out file]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = []
# (name, M, N, K, trans_a, trans_b, kind, force_bn)
for bn in (0, 64, 128, 256):
    CASES.append((f"nt_small_bn{bn}", 256, 256, 128, 0, 0, "bf16", bn))
CASES += [
    ("nt_tail", 300, 128, 96, 0, 0, "bf16", 0),
    ("nt_f32", 384, 256, 256, 0, 0, "f32", 0),
    ("nt_f32_acc", 384, 256, 256, 0, 0, "f32acc", 0),
    ("nt_gelu", 384, 512, 128, 0, 0, "gelu", 0),
    ("nt_resid", 512, 256, 192, 0, 0, "resid", 0),
    ("nt_dgelu", 256, 512, 128, 0, 0, "dgelu", 0),
    ("nt_pixshuf", 2 * 8 * 4, 16 * 16 * 64, 128, 0, 0, "pixshuf", 0),
    ("nn_tb", 256, 256, 128, 0, 1, "bf16", 0),
    ("nn_tb_bn64", 256, 256, 128, 0, 1, "bf16", 64),
    ("nn_tb_bn256", 512, 512, 256, 0, 1, "bf16", 256),
    ("tn_ta", 256, 256, 128, 1, 0, "bf16", 0),
    ("tt_wgrad", 256, 384, 200, 1, 1, "f32", 0),
    ("tt_wgrad_big", 1024, 4096, 3136, 1, 1, "f32", 0),
    ("nt_qkv", 12544, 3072, 1024, 0, 0, "bf16", 0),
    ("nt_fc1", 12544, 4096, 1024, 0, 0, "gelu", 0),
    ("nt_fc2", 12544, 1024, 4096, 0, 0, "resid", 0),
    ("nt_proj", 12544, 1024, 1024, 0, 0, "resid", 0),
    ("nt_dec", 12544, 16384, 4096, 0, 0, "pixshuf_big", 0),
    ("nn_dgrad_fc2", 12544, 4096, 1024, 0, 1, "dgelu", 0),
    ("nn_dgrad_fc1", 12544, 1024, 4096, 0, 1, "f32", 0),
    ("tt_wgrad_fc1", 4096, 1024, 12544, 1, 1, "f32", 0),
    ("tt_wgrad_qkv", 3072, 1024, 12544, 1, 1, "f32", 0),
    ("nt_seggpt_qkv", 3136, 3072, 1024, 0, 0, "bf16", 0),
    # operand-major study at the wgrad shape (K = tokens)
    ("mj_nt", 4096, 1024, 12544, 0, 0, "f32", 0),
    ("mj_tn", 4096, 1024, 12544, 1, 0, "f32", 0),
    ("mj_nn", 4096, 1024, 12544, 0, 1, "f32", 0),
    ("mj_tt", 4096, 1024, 12544, 1, 1, "f32", 0),
    # weight-gradient GEMMs as the engine issues them (zero-initialised output, accumulate=2 -> stream-K)
    ("sk_fc1", 4096, 1024, 12544, 1, 1, "f32sk", 0),
    ("sk_fc2", 1024, 4096, 12544, 1, 1, "f32sk", 0),
    ("sk_qkv", 3072, 1024, 12544, 1, 1, "f32sk", 0),
    ("sk_proj", 1024, 1024, 12544, 1, 1, "f32sk", 0),
    ("sk_nt_fc1", 4096, 1024, 12544, 0, 0, "f32sk", 0),
]


def run_case(name, M, N, K, ta, tb, kind, bn):
    import torch
    from painter_b200 import ops, _lib
    torch.manual_seed(0)
    dev = "cuda"
    a = (torch.randn(M, K, device=dev) * 0.5).bfloat16()
    b = (torch.randn(N, K, device=dev) * 0.5).bfloat16()
    a_in = a.t().contiguous() if ta else a
    b_in = b.t().contiguous() if tb else b
    ref = a.float() @ b.float().t()
    _lib.lib().pk_gemm_force_bn(bn)
    _lib.lib().pk_gemm_force_splits(int(os.environ.get("PK_FORCE_SPLITS", "0")))   # 0 = library heuristic
    bias = torch.randn(N, device=dev)
    kw = {}
    if kind == "bf16":
        fn = lambda: ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_BF16, bias=bias)
        want = (ref + bias)
    elif kind == "f32":
        fn = lambda: ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_F32, alpha=0.5)
        want = ref * 0.5
    elif kind == "f32sk":
        acc = torch.zeros(M, N, device=dev)
        calls = [0]
        def fn():
            calls[0] += 1
            return ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_F32, out=acc, accumulate=2)
        want = ref
    elif kind == "f32acc":
        base = torch.randn(M, N, device=dev)
        def fn():
            o = base.clone()
            return ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_F32, out=o, accumulate=True)
        want = ref + base
    elif kind == "gelu":
        fn = lambda: ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_GELU, bias=bias)
        z = (ref + bias)
        want = (z, torch.nn.functional.gelu(z.bfloat16().float()))
    elif kind == "resid":
        resid = torch.randn(M, N, device=dev)
        rpg = M // 4
        rs = torch.tensor([1.0, 0.0, 1.1, 0.9], device=dev)
        fn = lambda: ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_RESID, bias=bias, aux=resid,
                              rowscale=rs, rows_per_group=rpg)
        want = resid + rs.repeat_interleave(rpg)[:, None] * (ref + bias)
    elif kind == "dgelu":
        z = torch.randn(M, N, device=dev).bfloat16()
        fn = lambda: ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_DGELU, aux=z)
        zf = z.float().requires_grad_(True)
        torch.nn.functional.gelu(zf).sum().backward()
        want = ref * zf.grad
    elif kind in ("pixshuf", "pixshuf_big"):
        h, w, p, c = (8, 4, 16, 64) if kind == "pixshuf" else (56, 28, 16, 64)
        B = M // (h * w)
        out = torch.zeros(B, h * p, w * p, c, device=dev, dtype=torch.bfloat16)
        fn = lambda: ops.gemm(a_in, b_in, trans_a=ta, trans_b=tb, kind=ops.EPI_PIXSHUF, bias=bias,
                              pixshuf=(h, w, p, c, out))
        d = (ref + bias).reshape(B, h, w, p, p, c)
        want = torch.einsum("nhwpqc->nhpwqc", d).reshape(B, h * p, w * p, c)
    got = fn()
    torch.cuda.synchronize()
    res = {"case": name, "M": M, "N": N, "K": K, "ta": ta, "tb": tb, "kind": kind, "bn": bn}
    gots = got if isinstance(got, tuple) else (got,)
    wants = want if isinstance(want, tuple) else (want,)
    errs = []
    for g_, w_ in zip(gots, wants):
        g_ = g_.float()
        errs.append(((g_ - w_).abs().max() / w_.abs().max().clamp_min(1e-6)).item())
    res["max_rel_err"] = max(errs)
    res["ok"] = bool(max(errs) < 1.5e-2)
    # timing
    if M * N * K >= 2 ** 30:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 10
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        res["ms"] = ms
        res["tflops"] = 2.0 * M * N * K / ms / 1e9
        # cuBLAS comparator (test-time only)
        af, bf = a, b
        for _ in range(3):
            af @ bf.t()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            af @ bf.t()
        e1.record()
        torch.cuda.synchronize()
        res["cublas_tflops"] = 2.0 * M * N * K / (e0.elapsed_time(e1) / iters) / 1e9
    return res


if __name__ == "__main__":
    if len(sys.argv) >= 3 and sys.argv[1] == "--case":
        idx = int(sys.argv[2])
        try:
            r = run_case(*CASES[idx])
        except Exception as ex:  # noqa
            r = {"case": CASES[idx][0], "ok": False, "error": repr(ex)[:500]}
        print("RESULT " + json.dumps(r), flush=True)
        sys.exit(0)
    out = os.path.join(ROOT, "gpurun_out", "gemm_check.jsonl")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    only = sys.argv[1:] if len(sys.argv) > 1 else None
    with open(out, "w") as f:
        for i, c in enumerate(CASES):
            if only and not any(c[0].startswith(o) for o in only):
                continue
            t0 = time.time()
            try:
                p = subprocess.run([sys.executable, __file__, "--case", str(i)], capture_output=True,
                                   text=True, timeout=180)
                line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
                r = json.loads(line[-1][7:]) if line else {"case": c[0], "ok": False, "rc": p.returncode,
                                                            "stderr": p.stderr[-600:], "stdout": p.stdout[-600:]}
            except subprocess.TimeoutExpired:
                r = {"case": c[0], "ok": False, "error": "timeout"}
            r["wall_s"] = round(time.time() - t0, 1)
            f.write(json.dumps(r) + "\n")
            f.flush()
            print(json.dumps(r), flush=True)
