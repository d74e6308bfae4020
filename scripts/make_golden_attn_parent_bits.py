"""Bit-exact digests of the fused attention's outputs, for tests/test_gpu_attention_parent_bits.py.

tests/golden/attn_parent_bits.json was written by this script against the library built from commit 5b00dcb (the
attention kernels before their score loops were made branch-free), selected with PK_LIB:

    PK_LIB=/path/to/libpainter_b200.so python scripts/make_golden_attn_parent_bits.py [output.json]

Each case draws its operands from a seeded CPU generator, moves them to the GPU and runs both forward/backward entry
pairs: the training pair (pk_attn_fwd_save + pk_attn_bwd_saved, bias rows kept by the forward) and the pair that
recomputes the bias rows (pk_attn_fwd + pk_attn_bwd).  The digests are SHA-256 of the raw bytes of out, lse, dqkv and
of dt_ws, the per-CTA table-gradient partials the dQ kernel writes.  dTh / dTw are summed from dt_ws by
attn_dt_reduce_kernel with float atomics, whose order is not fixed, so they are not compared bitwise."""
import ctypes
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "attn_parent_bits.json")

# (name, B, heads, h, w): the training geometry, the long one (one-stage dK/dV), partial last tiles (9 x 28, 6 x 28,
# 8 x 4), and the narrow images (w = 1 has no image-column part in the dQ kernel's E matrix)
CASES = [
    ("56x28", 2, 2, 56, 28),
    ("112x56", 1, 1, 112, 56),
    ("9x28", 1, 2, 9, 28),
    ("64x1", 2, 1, 64, 1),
    ("64x2", 1, 2, 64, 2),
    ("6x28", 2, 2, 6, 28),
    ("8x4", 2, 2, 8, 4),
]


def _digest(t):
    import torch
    t = t.detach().contiguous().cpu()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()


def _bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, rel):
    """ops.attn_bwd, keeping its dt_ws workspace"""
    import torch
    from painter_b200 import ops
    from painter_b200._lib import lib
    N, dev = h * w, qkv.device
    Np = (N + 127) // 128 * 128
    L = lib()
    L.pk_attn_bwd_ws_floats.restype = ctypes.c_longlong
    dqkv = torch.empty_like(qkv)
    dTh = torch.zeros((2 * h - 1, 64), dtype=torch.float32, device=dev)
    dTw = torch.zeros((2 * w - 1, 64), dtype=torch.float32, device=dev)
    delta = torch.empty((B * heads * N,), dtype=torch.float32, device=dev)
    dt_ws = torch.empty((int(L.pk_attn_bwd_ws_floats(B, heads, h, w)),), dtype=torch.float32, device=dev)
    p = ops._ptr
    if rel is not None:
        relh, relw = rel
        fn, name = L.pk_attn_bwd_saved, "pk_attn_bwd_saved"
    else:
        relh = torch.empty((B * heads * Np * h,), dtype=torch.float32, device=dev)
        relw = torch.empty((B * heads * Np * w,), dtype=torch.float32, device=dev)
        fn, name = L.pk_attn_bwd, "pk_attn_bwd"
    ops.check(fn(p(qkv), p(out), p(dout), p(lse), p(th), p(tw), p(dqkv), p(dTh), p(dTw), p(delta), p(relh), p(relw),
                 p(dt_ws), B, heads, h, w, th.shape[0], tw.shape[0], ops._stream()), name)
    return dqkv, dt_ws


def case_digests(name, B, heads, h, w, seed=0):
    """{pair: {tensor: sha256}} for one geometry, pair in ("saved", "recomputed")"""
    import torch
    from painter_b200 import ops
    N, C = h * w, heads * 64
    g = torch.Generator().manual_seed(seed)
    qkv = (torch.randn(B * N, 3 * C, generator=g) * 1.5).bfloat16().cuda()
    th = ops.relpos_table_bf16((torch.randn(2 * h - 1, 64, generator=g) * 0.3).cuda())
    tw = ops.relpos_table_bf16((torch.randn(2 * w - 1, 64, generator=g) * 0.3).cuda())
    dout = (torch.randn(B * N, C, generator=g) * 0.5).bfloat16().cuda()
    res = {}
    for pair in ("saved", "recomputed"):
        if pair == "saved":
            out, lse, rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=True)
        else:
            (out, lse), rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w), None
        dqkv, dt_ws = _bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, rel)
        torch.cuda.synchronize()
        res[pair] = {"out": _digest(out), "lse": _digest(lse), "dqkv": _digest(dqkv), "dt_ws": _digest(dt_ws)}
    return res


def main():
    sys.path.insert(0, ROOT)
    from painter_b200 import _lib
    data = {"library": "built from commit 5b00dcb", "cases": {}}
    for c in CASES:
        data["cases"][c[0]] = case_digests(*c)
    path = sys.argv[1] if len(sys.argv) > 1 else FIXTURE
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote the digests of {_lib.LIB_PATH} to {path}")


if __name__ == "__main__":
    main()
