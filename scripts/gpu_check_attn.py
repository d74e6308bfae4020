"""GPU bring-up check of the fused attention forward (each case in a subprocess)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, B, heads, h, w)
CASES = [
    ("tiny_8x4", 2, 2, 8, 4),
    ("tiny_4x2", 3, 1, 4, 2),
    ("win_14x14", 4, 2, 14, 14),
    ("win_7x7", 3, 2, 7, 7),
    ("partial_6x28", 2, 2, 6, 28),
    ("one_tile_4x28", 1, 1, 4, 28),
    ("mid_56x28", 1, 2, 56, 28),
    ("h_16x8", 2, 1, 16, 8),
    ("long_112x56", 1, 1, 112, 56),
    ("full_b8", 8, 16, 56, 28),
    ("full_b16", 16, 16, 56, 28),
]


def ref_attn(qkv, th, tw, B, heads, h, w):
    import torch
    N, C = h * w, heads * 64
    q, k, v = qkv.float().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q * 0.125) @ k.transpose(-1, -2)
    idx_h = torch.arange(h, device=qkv.device)[:, None] - torch.arange(h, device=qkv.device)[None, :] + h - 1
    idx_w = torch.arange(w, device=qkv.device)[:, None] - torch.arange(w, device=qkv.device)[None, :] + w - 1
    Rh = th.float()[idx_h]
    Rw = tw.float()[idx_w]
    rq = q.reshape(B, heads, h, w, 64)
    rel_h = torch.einsum("bnhwc,hkc->bnhwk", rq, Rh)
    rel_w = torch.einsum("bnhwc,wkc->bnhwk", rq, Rw)
    s = (s.reshape(B, heads, h, w, h, w) + rel_h[..., :, None] + rel_w[..., None, :]).reshape(B, heads, N, N)
    lse = torch.logsumexp(s, -1) * 1.4426950408889634
    p = s.softmax(-1)
    o = (p @ v).permute(0, 2, 1, 3).reshape(B * N, C)
    return o, lse.reshape(B * heads, N)


def check_bwd(res, qkv, th, tw, out, lse, B, heads, h, w):
    """Backward vs torch autograd through the fp32 reference (on bf16-rounded inputs)."""
    import torch
    from painter_b200 import ops
    N, C = h * w, heads * 64
    dout = (torch.randn(B * N, C, device=qkv.device) * 0.5).bfloat16()
    dqkv, dTh, dTw = ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w)
    torch.cuda.synchronize()
    if B * heads * N * N <= 2 ** 26:
        q32 = qkv.float().requires_grad_(True)
        th32 = th.float().requires_grad_(True)
        tw32 = tw.float().requires_grad_(True)
        ro, _ = ref_attn(q32, th32, tw32, B, heads, h, w)
        (ro * dout.float()).sum().backward()
        def rel(a, b):
            return ((a.float() - b).abs().max() / b.abs().max().clamp_min(1e-9)).item()
        g = q32.grad.reshape(B * N, 3, C)
        d = dqkv.float().reshape(B * N, 3, C)
        res["dq_err"] = rel(d[:, 0], g[:, 0])
        res["dk_err"] = rel(d[:, 1], g[:, 1])
        res["dv_err"] = rel(d[:, 2], g[:, 2])
        res["dTh_err"] = rel(dTh, th32.grad[: 2 * h - 1])
        res["dTw_err"] = rel(dTw, tw32.grad[: 2 * w - 1])
        res["bwd_ok"] = bool(max(res["dq_err"], res["dk_err"], res["dv_err"], res["dTh_err"], res["dTw_err"]) < 3e-2)
        res["ok"] = bool(res.get("ok", True) and res["bwd_ok"])
    else:
        res["bwd_finite"] = bool(torch.isfinite(dqkv.float()).all().item() and torch.isfinite(dTh).all().item())
    if B * heads * N * N >= 2 ** 27:
        for _ in range(3):
            ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res["bwd_ms"] = ms
        res["bwd_tflops"] = 10.0 * B * heads * N * N * 64 / ms / 1e9


def run_case(name, B, heads, h, w):
    import torch
    from painter_b200 import ops
    torch.manual_seed(0)
    dev = "cuda"
    N, C = h * w, heads * 64
    qkv = (torch.randn(B * N, 3 * C, device=dev) * 1.5).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=dev) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=dev) * 0.3)
    out, lse = ops.attn_fwd(qkv, th, tw, B, heads, h, w)
    torch.cuda.synchronize()
    res = {"case": name, "B": B, "heads": heads, "h": h, "w": w}
    try:
        _run_fwd_checks(res, qkv, th, tw, out, lse, B, heads, h, w)
    finally:
        pass
    check_bwd(res, qkv, th, tw, out, lse, B, heads, h, w)
    return res


def _run_fwd_checks(res, qkv, th, tw, out, lse, B, heads, h, w):
    import torch
    from painter_b200 import ops
    N, C = h * w, heads * 64
    if B * heads * N * N <= 2 ** 28:
        ro, rl = ref_attn(qkv, th, tw, B, heads, h, w)
        res["out_err"] = ((out.float() - ro).abs().max() / ro.abs().max()).item()
        res["lse_err"] = (lse - rl).abs().max().item()
        res["ok"] = bool(res["out_err"] < 2e-2 and res["lse_err"] < 2e-2)
    else:
        # compare one (b, head) slab against the reference
        ro, rl = ref_attn(qkv[:N], th, tw, 1, heads, h, w)
        res["out_err"] = ((out[:N].float() - ro).abs().max() / ro.abs().max()).item()
        res["lse_err"] = (lse[:heads] - rl).abs().max().item()
        res["ok"] = bool(res["out_err"] < 2e-2 and res["lse_err"] < 2e-2 and torch.isfinite(out.float()).all().item())
    if B * heads * N * N >= 2 ** 27:
        for _ in range(3):
            ops.attn_fwd(qkv, th, tw, B, heads, h, w)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ops.attn_fwd(qkv, th, tw, B, heads, h, w)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        res["ms"] = ms
        res["tflops"] = 4.0 * B * heads * N * N * 64 / ms / 1e9


# Kernel-level timing at the bench geometries of the saved-rows pair (attn_fwd(save_rel=True) + attn_bwd(rel=...))
# and of the pair the attention module runs (attn_fwd + attn_bwd, which recomputes the bias rows in its own kernel).
# `--bench LIB [LIB ...]` times each library in its own process (PK_LIB selects it), alternating over
# $ATTN_BENCH_ROUNDS rounds, and compares every arm's outputs with the first arm's on the same seeded operands.
BENCH_GEOMS = [("train_b8", 8, 16, 56, 28), ("long_b2", 2, 16, 112, 56)]


def attn_flops(B, heads, h, w):
    """(forward, backward) FLOPs as executed: 2 resp. 7 N x N x 64 products per (batch, head)."""
    n2 = B * heads * (h * w) ** 2 * 64 * 2.0
    return 2 * n2, 7 * n2


def bench_arm(geom, iters, dump):
    import torch
    from painter_b200 import ops
    name, B, heads, h, w = next(g for g in BENCH_GEOMS if g[0] == geom)
    N, C = h * w, heads * 64
    torch.manual_seed(0)
    qkv = (torch.randn(B * N, 3 * C, device="cuda") * 1.5).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device="cuda") * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device="cuda") * 0.3)
    dout = (torch.randn(B * N, C, device="cuda") * 0.5).bfloat16()

    def fwd():
        return ops.attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=True)

    out, lse, rel = fwd()

    def bwd():
        return ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, rel=rel)

    dqkv, dTh, dTw = bwd()
    if dump:
        torch.save({"out": out.cpu(), "lse": lse.cpu(), "dqkv": dqkv.cpu(), "dTh": dTh.cpu(), "dTw": dTw.cpu()}, dump)

    def timed(fn):
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    def mod_fwd():
        return ops.attn_fwd(qkv, th, tw, B, heads, h, w)

    def mod_bwd():
        return ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w)

    fwd_ms, bwd_ms = timed(fwd), timed(bwd)
    mod_fwd_ms, mod_bwd_ms = timed(mod_fwd), timed(mod_bwd)

    def shares(fn):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if ev.device_type == torch.autograd.DeviceType.CUDA and "attn" in ev.key:
                kern[ev.key] = kern.get(ev.key, 0.0) + ev.device_time_total
        tot = sum(kern.values()) or 1.0
        return {k: round(v / tot, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])}

    ff, bf = attn_flops(B, heads, h, w)
    return {"geom": name, "fwd_ms": round(fwd_ms, 4), "bwd_ms": round(bwd_ms, 4),
            "fwd_bwd_ms": round(fwd_ms + bwd_ms, 4), "fwd_tflops": round(ff / fwd_ms / 1e9, 1),
            "bwd_tflops": round(bf / bwd_ms / 1e9, 1), "bwd_kernel_share": shares(bwd),
            "module_fwd_ms": round(mod_fwd_ms, 4), "module_bwd_ms": round(mod_bwd_ms, 4),
            "module_fwd_bwd_ms": round(mod_fwd_ms + mod_bwd_ms, 4), "module_bwd_kernel_share": shares(mod_bwd)}


def compare_dumps(a, b):
    import torch
    x, y = torch.load(a), torch.load(b)
    res = {}
    for k in x:
        d = (x[k].float() - y[k].float()).abs().max().item()
        res[k] = d / max(x[k].float().abs().max().item(), 1e-9)
    return res


def run_bench(libs, rounds, iters):
    """One JSON line per (round, geometry, library) on stdout; the operand dumps live in a temporary directory."""
    import shutil
    import tempfile
    tmp = tempfile.mkdtemp(prefix="attn_bench_")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": smi}), flush=True)
    try:
        for rnd in range(rounds):
            for geom in [g[0] for g in BENCH_GEOMS]:
                for i, lib in enumerate(libs):
                    dump = os.path.join(tmp, f"{geom}_{i}.pt") if rnd == 0 else ""
                    env = dict(os.environ, PK_LIB=os.path.abspath(lib))
                    p = subprocess.run([sys.executable, __file__, "--bench-arm", geom, str(iters), dump], env=env,
                                       capture_output=True, text=True, timeout=600)
                    line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
                    r = json.loads(line[-1][7:]) if line else {"geom": geom, "rc": p.returncode,
                                                                "stderr": p.stderr[-1500:]}
                    r.update(arm=lib, round=rnd)
                    if dump and i > 0 and line:
                        r["rel_diff_vs_arm0"] = compare_dumps(os.path.join(tmp, f"{geom}_0.pt"), dump)
                    print(json.dumps(r), flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    if len(sys.argv) >= 3 and sys.argv[1] == "--bench":
        run_bench(sys.argv[2:], rounds=int(os.environ.get("ATTN_BENCH_ROUNDS", "2")),
                  iters=int(os.environ.get("ATTN_BENCH_ITERS", "50")))
        sys.exit(0)
    if len(sys.argv) >= 5 and sys.argv[1] == "--bench-arm":
        print("RESULT " + json.dumps(bench_arm(sys.argv[2], int(sys.argv[3]), sys.argv[4])), flush=True)
        sys.exit(0)
    if len(sys.argv) >= 3 and sys.argv[1] == "--case":
        idx = int(sys.argv[2])
        try:
            r = run_case(*CASES[idx])
        except Exception as ex:  # noqa
            r = {"case": CASES[idx][0], "ok": False, "error": repr(ex)[:600]}
        print("RESULT " + json.dumps(r), flush=True)
        sys.exit(0)
    out = os.path.join(ROOT, "gpurun_out", "attn_check.jsonl")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "w") as f:
        for i, c in enumerate(CASES):
            t0 = time.time()
            try:
                p = subprocess.run([sys.executable, __file__, "--case", str(i)], capture_output=True, text=True,
                                   timeout=120)
                line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
                r = json.loads(line[-1][7:]) if line else {"case": c[0], "ok": False, "rc": p.returncode,
                                                            "stderr": p.stderr[-800:], "stdout": p.stdout[-800:]}
            except subprocess.TimeoutExpired:
                r = {"case": c[0], "ok": False, "error": "timeout"}
            r["wall_s"] = round(time.time() - t0, 1)
            f.write(json.dumps(r) + "\n")
            f.flush()
            print(json.dumps(r), flush=True)
