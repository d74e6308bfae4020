"""Fused attention at geometries where the dQ kernel's one-hot bias-row product and Toeplitz table terms meet their
edge cases: w = 1 (one image column, 64 image rows per key tile), w = 2 (32 image rows per key tile) and a partial
last tile at w = 28.  Forward and backward against torch autograd through an fp32 restatement of the reference math."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def relmax(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


def ref_attn(qkv, th, tw, B, heads, h, w):
    """q*scale @ k^T + decomposed rel-pos bias (rel_h over image rows, rel_w over image columns), softmax, @ v."""
    N, C = h * w, heads * 64
    q, k, v = qkv.float().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q * 0.125) @ k.transpose(-1, -2)
    ih = torch.arange(h, device=DEV)[:, None] - torch.arange(h, device=DEV)[None, :] + h - 1
    iw = torch.arange(w, device=DEV)[:, None] - torch.arange(w, device=DEV)[None, :] + w - 1
    rq = q.reshape(B, heads, h, w, 64)
    rel_h = torch.einsum("bnhwc,hkc->bnhwk", rq, th.float()[ih])
    rel_w = torch.einsum("bnhwc,wkc->bnhwk", rq, tw.float()[iw])
    s = (s.reshape(B, heads, h, w, h, w) + rel_h[..., :, None] + rel_w[..., None, :]).reshape(B, heads, N, N)
    return (s.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * N, C)


@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 64, 1), (2, 2, 64, 2), (2, 2, 9, 28)])
def test_attention_bias_tile_edges_vs_reference_math(B, heads, h, w):
    from painter_b200 import ops
    torch.manual_seed(0)
    N, C = h * w, heads * 64
    qkv = (torch.randn(B * N, 3 * C, device=DEV) * 1.5).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=DEV) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=DEV) * 0.3)
    dout = (torch.randn(B * N, C, device=DEV) * 0.5).bfloat16()
    q32 = qkv.float().requires_grad_(True)
    t32, w32 = th.float().requires_grad_(True), tw.float().requires_grad_(True)
    ro = ref_attn(q32, t32, w32, B, heads, h, w)
    (ro * dout.float()).sum().backward()
    g = q32.grad.reshape(B * N, 3, C)
    # the module's pair (bias rows recomputed by the backward) and the training pair (rows kept by the forward)
    out, lse = ops.attn_fwd(qkv, th, tw, B, heads, h, w)
    out2, lse2, rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=True)
    assert torch.equal(out2, out) and torch.equal(lse2, lse)
    assert relmax(out, ro) < 1e-2
    for kw in ({}, {"rel": rel}):
        dqkv, dTh, dTw = ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, **kw)
        d = dqkv.float().reshape(B * N, 3, C)
        for i in range(3):
            assert relmax(d[:, i], g[:, i]) < 2e-2, "qkv"[i]
        assert relmax(dTh, t32.grad[:2 * h - 1]) < 2e-2
        # with one image column dT_w sums every row of dS, which is zero in exact arithmetic; what the backward
        # returns there is the bf16 rounding of O in delta = rowsum(dO * O), so it has no reference to match
        if w > 1:
            assert relmax(dTw, w32.grad[:2 * w - 1]) < 2e-2
