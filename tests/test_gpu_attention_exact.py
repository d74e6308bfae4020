"""Fused rel-pos attention (ops.attn_fwd / ops.attn_bwd) against exact arithmetic and per-element error bounds, at every
grid the model launches and at the tile edges:
- selector inputs (tests/_attn_ref.py) on which the kernel's arithmetic is exact: out, dqkv and the table gradients
  match the construction bit for bit, lse within a few fp32 ulps, through both entry pairs and with frozen tables;
- random inputs, soft and peaked score rows: every element of out, lse, dq, dk, dv, dTh and dTw inside its forward-error
  bound around the fp64 reference (the worst bound ratio per quantity is printed);
- frozen tables give the same dqkv bits as trainable ones; a running table gradient is added to; table padding changes
  nothing; the pair that keeps the bias rows gives the same bits as the one that recomputes them."""
import pytest
import torch

import _attn_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (B, heads, h, w)
GEOMS = [
    (8, 16, 56, 28),     # Painter / SegGPT global blocks at 896 x 448, the benchmark's training step
    (1, 16, 112, 56),    # global blocks at 1792 x 896 (the one-stage dK/dV pipeline; 56 x 28 runs two stages)
    (128, 16, 14, 14),   # window_size = 14 training windows: 2048 CTAs per query-tile row
    (4, 2, 7, 7),        # the smallest window
    (2, 2, 1, 1),
    (2, 2, 64, 1),       # one image column: 64 image rows per key tile in the bias-row gradient product
    (2, 2, 64, 2),
    (2, 2, 9, 28),       # N = 252, 13 x 7 = 91: partial last query and key tiles
    (3, 1, 13, 7),
    (2, 2, 112, 1),
    (2, 2, 1, 56),       # the widest grid row the dQ kernel takes
]
GEOM_IDS = [f"{B}x{hd}-{h}x{w}" for B, hd, h, w in GEOMS]
SPREADS = {"soft": 0.3, "peaked": 1.5}
ELEMS = 24_000_000       # N x N float64 elements per reference chunk (a few GB of temporaries with the bounds)


def chunks(idx, N):
    n = max(1, ELEMS // (N * N))
    return [idx[i:i + n] for i in range(0, len(idx), n)]


def pack_heads(x, B, heads, h, w):
    """[B*heads, N, 64] -> [B*N, heads*64]"""
    return x.reshape(B, heads, h * w, 64).permute(0, 2, 1, 3).reshape(B * h * w, heads * 64)


def run(ops, qkv, th, tw, dO, B, heads, h, w, saved=False, **kw):
    if saved:
        out, lse, rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w, save_rel=True)
    else:
        (out, lse), rel = ops.attn_fwd(qkv, th, tw, B, heads, h, w), None
    dqkv, dTh, dTw = ops.attn_bwd(qkv, out, dO, lse, th, tw, B, heads, h, w, rel=rel, **kw)
    return out, lse, dqkv, dTh, dTw


def random_inputs(ops, B, heads, h, w, spread, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    N, C = h * w, heads * 64
    qkv = (torch.randn(B * N, 3 * C, device=DEV, generator=g) * spread).bfloat16()
    th = ops.relpos_table_bf16(torch.randn(2 * h - 1, 64, device=DEV, generator=g) * 0.3)
    tw = ops.relpos_table_bf16(torch.randn(2 * w - 1, 64, device=DEV, generator=g) * 0.3)
    dO = (torch.randn(B * N, C, device=DEV, generator=g) * 0.5).bfloat16()
    return qkv, th, tw, dO


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("twohot", [False, True], ids=["onehot", "twohot"])
@pytest.mark.parametrize("B,heads,h,w", GEOMS, ids=GEOM_IDS)
def test_selector_inputs_bitwise(B, heads, h, w, twohot):
    """out == V[sel] (or the mean of two), dqkv == bf16_rn(exact), dTh / dTw == exact, lse within 8 fp32 ulps (of
    max(|lse|, 1)), for both entry pairs and both table-gradient settings.  Zeros compare equal whatever their sign."""
    from painter_b200 import ops
    N, C, Pn = h * w, heads * 64, B * heads
    inp = R.selector_inputs(B, heads, h, w, twohot, seed=N + 7 * B * heads + twohot, device=DEV)
    ex = {key: [] for key in ("out", "lse", "dq", "dk", "dv")}
    dTh = torch.zeros(2 * h - 1, 64, dtype=torch.float64, device=DEV)
    dTw = torch.zeros(2 * w - 1, 64, dtype=torch.float64, device=DEV)
    for c in chunks(torch.arange(Pn, device=DEV), N):
        r = R.selector_expected(inp, B, heads, h, w, pairs=c)
        for key in ex:
            ex[key].append(r[key])
        dTh += r["dTh"].sum(0)
        dTw += r["dTw"].sum(0)
        del r
    ex = {key: torch.cat(v) for key, v in ex.items()}
    want_out = pack_heads(ex["out"], B, heads, h, w).float().bfloat16()
    want_dqkv = torch.cat([pack_heads(ex[key], B, heads, h, w) for key in ("dq", "dk", "dv")], 1).float().bfloat16()
    tol = 2.0 ** -20 * ex["lse"].abs().clamp_min(1.0)
    for saved in (False, True):
        for tg in (True, False):
            out, lse, dqkv, gh, gw = run(ops, inp["qkv"], inp["th"], inp["tw"], inp["dO"], B, heads, h, w,
                                         saved=saved, table_grads=tg)
            what = f"saved={saved} table_grads={tg}"
            assert torch.equal(out, want_out), what
            assert bool(((lse.double() - ex["lse"]).abs() <= tol).all()), what
            d, want = dqkv.reshape(B * N, 3, C), want_dqkv.reshape(B * N, 3, C)
            for i in range(3):
                bad = (d[:, i] != want[:, i]).sum().item()
                assert bad == 0, f"{what}: {bad} elements of d{'qkv'[i]} differ"
            if tg:
                assert torch.equal(gh.double(), dTh) and torch.equal(gw.double(), dTw), what
            else:
                assert gh is None and gw is None


# ---------------------------------------------------------------------------------------------------------------
def sampled_pairs(Pn, N, seed):
    """Every pair of a small call; else the first, the middle and the last, and five more drawn at random when N is
    small enough for the fp64 reference to be cheap."""
    if Pn <= 8:
        return list(range(Pn))
    s = {0, Pn // 2, Pn - 1}
    if N <= 2000:
        g = torch.Generator().manual_seed(seed)
        s |= set(torch.randperm(Pn, generator=g)[:5].tolist())
    return sorted(s)


@pytest.mark.parametrize("spread", list(SPREADS))
@pytest.mark.parametrize("B,heads,h,w", GEOMS, ids=GEOM_IDS)
def test_random_inputs_within_error_bounds(B, heads, h, w, spread):
    from painter_b200 import ops
    N, Pn = h * w, B * heads
    nt = (N + 63) // 64
    qkv, th, tw, dO = random_inputs(ops, B, heads, h, w, SPREADS[spread], seed=N + Pn)
    out, lse, dqkv, dTh, dTw = run(ops, qkv, th, tw, dO, B, heads, h, w)
    # the training pair (bias rows kept by the forward) computes the same bits
    out2, lse2, dqkv2, _, _ = run(ops, qkv, th, tw, dO, B, heads, h, w, saved=True)
    assert torch.equal(out2, out) and torch.equal(lse2, lse) and torch.equal(dqkv2, dqkv)
    pairs = sampled_pairs(Pn, N, seed=N)
    if len(pairs) < Pn:
        # the table gradients sum over every pair: take them from a call whose dO is zero outside the sampled pairs
        keep = torch.zeros(Pn, device=DEV, dtype=torch.bfloat16)
        keep[pairs] = 1
        dOm = (dO.reshape(B, N, heads, 64) * keep.reshape(B, 1, heads, 1)).reshape(B * N, heads * 64)
        _, _, dqkv_m, dTh, dTw = run(ops, qkv, th, tw, dOm, B, heads, h, w)
        q_m = R.split_qkv(dqkv_m, B, heads, h, w)
        q_f = R.split_qkv(dqkv, B, heads, h, w)
        for a, b in zip(q_m, q_f):   # the masked call computes the sampled pairs' dqkv bit for bit
            assert torch.equal(a[pairs], b[pairs])
    q, k, v = R.split_qkv(qkv, B, heads, h, w)
    dO64 = R.split_heads(dO, B, heads, h, w)
    got = dict(zip(("dq", "dk", "dv"), R.split_qkv(dqkv, B, heads, h, w)))
    got["out"] = R.split_heads(out, B, heads, h, w)
    got["lse"] = lse.double()
    th64, tw64 = th.double(), tw.double()
    worst = {key: 0.0 for key in ("out", "lse", "dq", "dk", "dv", "dTh", "dTw")}
    sums = {key: 0.0 for key in ("dTh", "dTw", "dTh_E", "dTh_M", "dTw_E", "dTw_M")}
    for c in chunks(torch.tensor(pairs, device=DEV), N):
        r = R.reference(q[c], k[c], v[c], th64, tw64, dO64[c], h, w)
        b = R.error_bounds(r, q[c], k[c], v[c], th64, tw64, dO64[c], h, w)
        for key in ("out", "lse", "dq", "dk", "dv"):
            worst[key] = max(worst[key], ((got[key][c] - r[key]).abs() / b[key]).max().item())
        for key in ("dTh", "dTw"):
            sums[key] = sums[key] + r[key].sum(0)
            sums[key + "_E"] = sums[key + "_E"] + b[key + "_E"].sum(0)
            sums[key + "_M"] = sums[key + "_M"] + b[key + "_M"].sum(0)
        del r, b
    for key, g_ in (("dTh", dTh), ("dTw", dTw)):
        bound = R.table_grad_bound(sums[key + "_E"], sums[key + "_M"], Pn * nt)
        worst[key] = ((g_.double() - sums[key]).abs() / bound).max().item()
    print(f"\n[attention bound ratio] B={B} heads={heads} {h}x{w} {spread} ({len(pairs)}/{Pn} pairs): "
          + " ".join(f"{key}={val:.3f}" for key, val in worst.items()))
    assert all(val < 1.0 for val in worst.values()), worst


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 16, 16), (2, 2, 9, 28), (8, 16, 56, 28)], ids=["full-tiles",
                                                                                             "partial-tiles", "bench"])
def test_frozen_tables_same_dqkv_bits(B, heads, h, w):
    """table_grads=False runs attn_bwd_dq_kernel<false>, which leaves out the table-gradient partials; dQ comes from
    the same instructions in the same order, so dqkv is bit-identical to table_grads=True (both entry pairs)."""
    from painter_b200 import ops
    qkv, th, tw, dO = random_inputs(ops, B, heads, h, w, 1.5, seed=3)
    for saved in (False, True):
        _, _, d1, _, _ = run(ops, qkv, th, tw, dO, B, heads, h, w, saved=saved, table_grads=True)
        _, _, d0, gh, gw = run(ops, qkv, th, tw, dO, B, heads, h, w, saved=saved, table_grads=False)
        assert gh is None and gw is None
        assert torch.equal(d0, d1), f"saved={saved}"


@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 9, 28), (8, 16, 56, 28), (1, 2, 1, 56)])
def test_running_table_gradient_is_added_to(B, heads, h, w):
    """dT_out pre-filled with X (the engine passes gradient-arena slots) comes back as X + dT.  The reduction adds its
    four stripe sums into each entry with fp32 atomics in no fixed order, so the result is X + dT up to five fp32
    roundings of partial sums bounded by a few times |X| + max|dT|: checked to 2^-20 (|X| + max|dT|) per element."""
    from painter_b200 import ops
    qkv, th, tw, dO = random_inputs(ops, B, heads, h, w, 1.5, seed=4)
    out, lse = ops.attn_fwd(qkv, th, tw, B, heads, h, w)
    _, dTh, dTw = ops.attn_bwd(qkv, out, dO, lse, th, tw, B, heads, h, w)
    g = torch.Generator(device=DEV).manual_seed(5)
    Xh = torch.randn(dTh.shape, device=DEV, generator=g) * dTh.abs().max()
    Xw = torch.randn(dTw.shape, device=DEV, generator=g) * dTw.abs().max()
    acc = (Xh.clone(), Xw.clone())
    _, gh, gw = ops.attn_bwd(qkv, out, dO, lse, th, tw, B, heads, h, w, dT_out=acc)
    assert gh is acc[0] and gw is acc[1]
    for X, d, got in ((Xh, dTh, gh), (Xw, dTw, gw)):
        tol = 2.0 ** -20 * (X.abs() + d.abs().max())
        err = (got - (X + d)).abs()
        assert bool((err <= tol).all()), (err / tol).max().item()
    assert bool((gh != Xh).any()) or bool((gw != Xw).any())   # the gradient was actually added


@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 9, 28), (3, 1, 13, 7), (2, 2, 1, 56), (2, 2, 112, 1),
                                         (1, 2, 56, 28)])
def test_table_padding_changes_nothing(B, heads, h, w):
    """Tables zero-padded to the minimum (2n - 1 rounded up to 16 rows) and to the maximum the kernel accepts
    (224 / 112 rows) give bit-identical out, lse and dqkv through both entry pairs."""
    from painter_b200 import ops
    qkv, th, tw, dO = random_inputs(ops, B, heads, h, w, 1.5, seed=6)
    thx = torch.zeros(224, 64, dtype=torch.bfloat16, device=DEV)
    twx = torch.zeros(112, 64, dtype=torch.bfloat16, device=DEV)
    thx[:th.shape[0]] = th
    twx[:tw.shape[0]] = tw
    for saved in (False, True):
        a = run(ops, qkv, th, tw, dO, B, heads, h, w, saved=saved)
        b = run(ops, qkv, thx, twx, dO, B, heads, h, w, saved=saved)
        for i, name in enumerate(("out", "lse", "dqkv")):
            assert torch.equal(a[i], b[i]), f"{name} saved={saved}"
