"""The fused attention backward sums the bias-row gradients without atomics, so dqkv is bitwise reproducible.  The
shapes cover both dK/dV pipeline depths (two query-tile stages at 56 x 28, one at 112 x 56) and partial tiles."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 8, 4), (1, 2, 6, 28), (2, 2, 56, 28), (1, 1, 112, 56)])
def test_attention_bwd_dqkv_is_bitwise_reproducible(B, heads, h, w):
    from painter_b200 import ops
    torch.manual_seed(0)
    N, C = h * w, heads * 64
    qkv = (torch.randn(B * N, 3 * C, device=DEV) * 1.5).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=DEV) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=DEV) * 0.3)
    dout = (torch.randn(B * N, C, device=DEV) * 0.5).bfloat16()
    out, lse, rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=True)
    first = ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, rel=rel)[0]
    for _ in range(2):
        again = ops.attn_bwd(qkv, out, dout, lse, th, tw, B, heads, h, w, rel=rel)[0]
        assert torch.equal(again, first)
    assert torch.isfinite(first.float()).all()
