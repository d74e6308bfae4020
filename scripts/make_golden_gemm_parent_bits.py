"""Bit-exact digests of the wgmma GEMM's outputs, for tests/test_gpu_gemm_parent_bits.py.

tests/golden/gemm_parent_bits.json was written by this script against the library built from commit 8c31bc7 (the
GEMM whose wgmmas ptxas serialised), selected with PK_LIB:

    PK_LIB=/path/to/libpainter_b200.so python scripts/make_golden_gemm_parent_bits.py [output.json]

Each case draws its operands from a seeded CPU generator, moves them to the GPU and runs one call: every epilogue kind
at the block shapes of the training step (M = 12544 tokens, ViT-L), forward and data gradients; decoder_embed with
the pixel-shuffle epilogue; the decoder's 3x3 convolution forward with the fused head (its conv output and patch
predictions; the loss numerator is summed with float atomics) and its data gradient; a small weight gradient the
planner runs as plain tiles; and ragged shapes.  The digests are SHA-256 of the raw output bytes.  Stream-K weight
gradients add partial tiles with float atomics, whose order is not fixed, so they are not digested."""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "gemm_parent_bits.json")

BF16, F32, GELU, RESID, DGELU, PIXSHUF = range(6)
M, C = 12544, 1024          # ViT-L at 896 x 448, batch 8: 8 x 56 x 28 tokens
DEC_B, DEC_H, DEC_W, P = 2, 896, 448, 16

# (name, M, N, K, kind, trans_b, extras): extras among "bias", "rowscale" (per-sample scales, with the residual),
# "acc" (read-modify-write fp32 output)
LINEAR = [
    ("qkv_fwd", M, 3 * C, C, BF16, False, ("bias",)),
    ("proj_fwd_f32", M, C, C, F32, False, ("bias",)),
    ("proj_fwd_resid", M, C, C, RESID, False, ("bias", "rowscale")),
    ("fc1_fwd_gelu", M, 4 * C, C, GELU, False, ("bias",)),
    ("fc2_fwd_resid", M, C, 4 * C, RESID, False, ("bias", "rowscale")),
    ("fc2_dgrad_dgelu", M, 4 * C, C, DGELU, True, ()),
    ("fc1_dgrad", M, C, 4 * C, BF16, True, ()),
    ("proj_dgrad", M, C, C, BF16, True, ()),
    ("qkv_dgrad_f32", M, C, 3 * C, F32, True, ()),
    ("ragged_bf16", 1000, 192, 200, BF16, False, ("bias",)),
    ("ragged_resid", 300, 256, 320, RESID, False, ("bias", "rowscale")),
    ("ragged_gelu", 777, 384, 136, GELU, True, ("bias",)),
    ("ragged_f32_acc", 513, 128, 1000, F32, False, ("acc",)),
]
OTHER = ["wgrad_plain_tiles", "decoder_embed_pixshuf", "conv_fwd_head", "conv_dgrad_unshuffle"]
CASES = [c[0] for c in LINEAR] + OTHER


def _digest(t):
    import torch
    t = t.detach().contiguous().cpu()
    if t.dtype == torch.bfloat16:
        t = t.view(torch.int16)
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()


def _linear(g, Mx, N, K, kind, trans_b, extras):
    import torch
    from painter_b200 import ops
    a = torch.randn(Mx, K, generator=g).bfloat16().cuda()
    w = (torch.randn(K, N, generator=g) if trans_b else torch.randn(N, K, generator=g)) * K ** -0.5
    kw = {"trans_b": trans_b, "kind": kind}
    if "bias" in extras:
        kw["bias"] = torch.randn(N, generator=g).cuda()
    if kind == RESID:
        kw["aux"] = torch.randn(Mx, N, generator=g).cuda()
    if kind == DGELU:
        kw["aux"] = torch.randn(Mx, N, generator=g).bfloat16().cuda()
    if "rowscale" in extras:
        groups = 8
        rpg = (Mx + groups - 1) // groups
        kw["rowscale"] = torch.tensor([0.0, 1.25, 1.25, 0.0, 1.25, 1.25, 1.25, 1.25])[:groups].cuda()
        kw["rows_per_group"] = rpg
    if "acc" in extras:
        kw["out"] = torch.randn(Mx, N, generator=g).cuda()
        kw["accumulate"] = True
    out = ops.gemm(a, w.bfloat16().cuda(), **kw)
    outs = out if isinstance(out, tuple) else (out,)
    return {f"out{i}": _digest(o) for i, o in enumerate(outs)}


def _other(g, name):
    import torch
    from painter_b200 import ops
    if name == "wgrad_plain_tiles":   # 2 tiles x 16 k-blocks: too small for stream-K, so no atomics
        dy = torch.randn(1024, 256, generator=g).bfloat16().cuda()
        x = torch.randn(1024, 128, generator=g).bfloat16().cuda()
        out = torch.zeros(256, 128, device="cuda")
        ops.gemm(dy, x, trans_a=True, trans_b=True, kind=F32, out=out, accumulate=2)
        return {"out0": _digest(out)}
    h, w = DEC_H // P, DEC_W // P
    if name == "decoder_embed_pixshuf":
        cat = torch.randn(DEC_B * h * w, 4 * C, generator=g).bfloat16().cuda()
        wdec = (torch.randn(P * P * 64, 4 * C, generator=g) * 0.02).bfloat16().cuda()
        bias = torch.randn(P * P * 64, generator=g).cuda()
        out = torch.empty((DEC_B, DEC_H, DEC_W, 64), dtype=torch.bfloat16, device="cuda")
        ops.gemm(cat, wdec, kind=PIXSHUF, bias=bias, pixshuf=(h, w, P, 64, out))
        return {"out0": _digest(out)}
    img = torch.randn(DEC_B, DEC_H, DEC_W, 64, generator=g).bfloat16().cuda()
    wf, wd = ops.conv3x3_pack((torch.randn(64, 64, 3, 3, generator=g) * 0.04).cuda())
    if name == "conv_fwd_head":
        hp = torch.cat([torch.randn(64, generator=g) * 0.1, 1 + 0.1 * torch.randn(64, generator=g),
                        0.1 * torch.randn(64, generator=g), 0.1 * torch.randn(192, generator=g),
                        0.1 * torch.randn(3, generator=g), torch.zeros(5)]).cuda()
        tgts = torch.randn(DEC_B, 3, DEC_H, DEC_W, generator=g).cuda()
        mask = (torch.rand(DEC_B, h * w, generator=g) < 0.75).to(torch.uint8).cuda()
        valid = (torch.rand(DEC_B, 3, DEC_H, DEC_W, generator=g) < 0.9).float().cuda()
        c1, patch, _num = ops.decoder_head_fwd(img, wf, hp, tgts, mask, valid, P, 0)
        return {"c1": _digest(c1), "patch": _digest(patch)}
    assert name == "conv_dgrad_unshuffle"
    return {"out0": _digest(ops.conv3x3_dgrad_unshuffle(img, wd, P))}


def case_digests(name, seed=0):
    """{output: sha256} of one case"""
    import torch
    g = torch.Generator().manual_seed(seed)
    lin = {c[0]: c for c in LINEAR}
    res = _linear(g, *lin[name][1:]) if name in lin else _other(g, name)
    torch.cuda.synchronize()
    return res


def main():
    sys.path.insert(0, ROOT)
    from painter_b200 import _lib
    data = {"library": "built from commit 8c31bc7", "cases": {c: case_digests(c) for c in CASES}}
    path = sys.argv[1] if len(sys.argv) > 1 else FIXTURE
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote the digests of {_lib.LIB_PATH} to {path}")


if __name__ == "__main__":
    main()
