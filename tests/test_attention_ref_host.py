"""CPU checks of the attention test helpers (tests/_attn_ref.py), before any GPU runs them:
- the fp64 reference equals an independent restatement (einsum form, torch autograd for the gradients);
- a torch emulation of the fused kernel's rounding points (bf16 P before P V with fp32 l, bf16 O, delta from the bf16
  O, bf16 dS and P^T, bf16 G, bf16 dqkv) stays inside the per-element error bounds;
- plausible kernel bugs applied to that emulation exceed the bounds, so the GPU suite would catch them;
- the selector inputs select what their closed form says, with an unambiguous argmax (or an exact two-way tie)."""
import math

import pytest
import torch

import _attn_ref as R

SPREADS = {"soft": 0.3, "peaked": 1.5}
# every (h, w) the GPU suite runs: the model's grids and the tile edges
GEOMS_HW = [(56, 28), (112, 56), (14, 14), (7, 7), (1, 1), (64, 1), (64, 2), (9, 28), (13, 7), (112, 1), (1, 56)]


def random_inputs(B, heads, h, w, spread, seed):
    """bf16-valued float64 q, k, v, dO [B*heads, N, 64] and tables, as the GPU tests draw them."""
    g = torch.Generator().manual_seed(seed)
    N, Pn = h * w, B * heads

    def bf(x):
        return x.to(torch.bfloat16).double()

    q, k, v = (bf(torch.randn(Pn, N, 64, generator=g) * spread) for _ in range(3))
    th = bf(torch.randn(2 * h - 1, 64, generator=g) * 0.3)
    tw = bf(torch.randn(2 * w - 1, 64, generator=g) * 0.3)
    dO = bf(torch.randn(Pn, N, 64, generator=g) * 0.5)
    return q, k, v, th, tw, dO


def emulate(q, k, v, th, tw, dO, h, w, bug=None):
    """The fused kernel's arithmetic restated in fp32 torch with its bf16 rounding points (global row maximum instead
    of the online one: a legitimate reordering the bounds cover).  `bug` injects one plausible kernel defect."""
    bf = lambda x: x.to(torch.bfloat16).float()   # noqa: E731
    N, Lh, Lw = h * w, 2 * h - 1, 2 * w - 1
    last = N // 64 * 64                            # first row of the last, partial, 64-row tile
    q, k, v, dO = q.float(), k.float(), v.float(), dO.float()
    th, tw = th[:Lh].float(), tw[:Lw].float()
    if bug == "toeplitz":                          # bias gathered from table row i_q - i + h instead of + h - 1
        th = torch.cat([th[1:], th[-1:]])
    ki, kj = R.coords(h, w, "cpu")
    rh, rw = R.bias_rows(q, th, tw, h, w)
    log2e = torch.tensor(R.LOG2E, dtype=torch.float32)
    s = (q @ k.transpose(1, 2)) * torch.tensor(0.125 * R.LOG2E, dtype=torch.float32) \
        + ((rh * log2e)[:, :, ki] + (rw * log2e)[:, :, kj])
    sf = s.clone()
    if bug == "drop_key_tile":
        sf[:, :, last:] = -math.inf
    m = sf.amax(2, keepdim=True)
    p = torch.exp2(sf - m)
    l = p.sum(2, keepdim=True)
    o = (bf(p) @ v) * (1.0 / l)
    if bug == "scale_q_tile":
        o[:, last:] *= 1 + 2.0 ** -6
    O = bf(o)
    lse = (m + torch.log2(l)).squeeze(2)
    if bug == "lse":
        lse = lse + 2.0 ** -12
    delta = (dO * O).sum(2)
    pb = torch.exp2(s - lse[..., None])
    dS = bf(pb * (dO @ v.transpose(1, 2) - delta[..., None]))
    Pb = bf(pb)
    if bug == "dv_q_tile":
        Pb[:, :64] = 0
    dv = bf(Pb.transpose(1, 2) @ dO)
    dk = bf(0.125 * (dS.transpose(1, 2) @ q))
    dRh, dRw = R.rel_grads(dS, h, w)
    if bug == "dtw_k_tile":
        dSx = dS.clone()
        dSx[:, :, :64] = 0
        dRw = R.rel_grads(dSx, h, w)[1]
    Gh, Gw = R.toeplitz_grads(bf(dRh), bf(dRw), h, w)
    dq = bf(0.125 * (dS @ k) + Gh @ th + Gw @ tw)
    return {"out": O, "lse": lse, "dq": dq, "dk": dk, "dv": dv,
            "dTh": (Gh.transpose(1, 2) @ q).sum(0), "dTw": (Gw.transpose(1, 2) @ q).sum(0)}


def bound_ratios(got, ref, bnd, h, w):
    """max |got - ref| / bound per quantity (dT compared as the sum over pairs, like the kernel returns it)."""
    nctas = ref["out"].shape[0] * ((h * w + 63) // 64)
    out = {}
    for key in ("out", "lse", "dq", "dk", "dv"):
        out[key] = ((got[key].double() - ref[key]).abs() / bnd[key]).max().item()
    for t in ("dTh", "dTw"):
        b = R.table_grad_bound(bnd[t + "_E"].sum(0), bnd[t + "_M"].sum(0), nctas)
        out[t] = ((got[t].double() - ref[t].sum(0)).abs() / b).max().item()
    return out


# ---------------------------------------------------------------------------------------------------------------
def restated(qkv, th, tw, B, heads, h, w):
    """models_painter.py:73-86 + vitdet_utils.py:96-125 in the einsum form of tests/test_gpu_attention_bias_tiles.py."""
    N, C = h * w, heads * 64
    q, k, v = qkv.reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4)
    s = (q * 0.125) @ k.transpose(-1, -2)
    ih = torch.arange(h)[:, None] - torch.arange(h)[None, :] + h - 1
    iw = torch.arange(w)[:, None] - torch.arange(w)[None, :] + w - 1
    rq = q.reshape(B, heads, h, w, 64)
    rel_h = torch.einsum("bnhwc,hkc->bnhwk", rq, th[ih])
    rel_w = torch.einsum("bnhwc,wkc->bnhwk", rq, tw[iw])
    s = (s.reshape(B, heads, h, w, h, w) + rel_h[..., :, None] + rel_w[..., None, :]).reshape(B, heads, N, N)
    lse = torch.logsumexp(s, -1).reshape(B * heads, N) * R.LOG2E
    return (s.softmax(-1) @ v).permute(0, 2, 1, 3).reshape(B * N, C), lse


@pytest.mark.parametrize("B,heads,h,w", [(2, 2, 6, 5), (1, 3, 9, 28), (2, 1, 13, 7), (1, 2, 8, 1), (1, 2, 1, 9)])
def test_reference_matches_autograd_restatement(B, heads, h, w):
    q, k, v, th, tw, dO = random_inputs(B, heads, h, w, 1.0, seed=h * 100 + w)
    r = R.reference(q, k, v, th, tw, dO, h, w)

    def pack(x):
        return x.reshape(B, heads, h * w, 64).permute(0, 2, 1, 3).reshape(B * h * w, heads * 64)

    qkv = torch.cat([pack(q), pack(k), pack(v)], 1).requires_grad_(True)
    t1, t2 = th.clone().requires_grad_(True), tw.clone().requires_grad_(True)
    out, lse = restated(qkv, t1, t2, B, heads, h, w)
    (out * pack(dO)).sum().backward()
    C = heads * 64

    def close(a, b, scale=None):
        scale = b.abs().max() if scale is None else scale
        return ((a - b).abs().max() / scale).item() < 1e-12

    assert close(pack(r["out"]), out.detach())
    assert close(r["lse"], lse.detach())
    for i, key in enumerate(("dq", "dk", "dv")):
        assert close(pack(r[key]), qkv.grad[:, i * C:(i + 1) * C]), key
    # with one image column (or row) the exact dT_w (dT_h) is zero: every row of dS sums to 0
    scale = max(t1.grad.abs().max(), t2.grad.abs().max())
    assert close(r["dTh"].sum(0), t1.grad, scale) and close(r["dTw"].sum(0), t2.grad, scale)


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spread", list(SPREADS))
@pytest.mark.parametrize("B,heads,h,w", [(1, 2, 9, 28), (2, 2, 13, 7), (1, 2, 64, 2), (1, 2, 1, 56), (2, 1, 7, 7),
                                         (1, 1, 112, 1)])
def test_emulated_kernel_rounding_stays_inside_bounds(B, heads, h, w, spread):
    q, k, v, th, tw, dO = random_inputs(B, heads, h, w, SPREADS[spread], seed=7 * h + w)
    ref = R.reference(q, k, v, th, tw, dO, h, w)
    bnd = R.error_bounds(ref, q, k, v, th, tw, dO, h, w)
    ratios = bound_ratios(emulate(q, k, v, th, tw, dO, h, w), ref, bnd, h, w)
    print(f"\n[bound ratio, emulation] {B}x{heads} {h}x{w} {spread}: "
          + " ".join(f"{k_}={v_:.3f}" for k_, v_ in ratios.items()))
    assert all(x < 1.0 for x in ratios.values()), ratios


# bug -> the quantity it has to be caught in
CONTROLS = {"toeplitz": "out", "drop_key_tile": "out", "scale_q_tile": "out", "swap_heads": "out", "lse": "lse",
            "dv_q_tile": "dv", "dtw_k_tile": "dTw"}


@pytest.mark.parametrize("bug", list(CONTROLS))
def test_negative_controls_exceed_bounds(bug):
    """Each bug, applied to the emulation at 9 x 28 (252 tokens: a partial last query and key tile), moves some element
    of the quantity it corrupts past its bound under at least one of the two score spreads the GPU tests use."""
    B, heads, h, w = 1, 2, 9, 28
    key = CONTROLS[bug]
    worst = {}
    for spread, sd in SPREADS.items():
        q, k, v, th, tw, dO = random_inputs(B, heads, h, w, sd, seed=3)
        ref = R.reference(q, k, v, th, tw, dO, h, w)
        bnd = R.error_bounds(ref, q, k, v, th, tw, dO, h, w)
        if bug == "swap_heads":
            got = emulate(q, k, v[[1, 0]], th, tw, dO, h, w)
        else:
            got = emulate(q, k, v, th, tw, dO, h, w, bug=bug)
        worst[spread] = bound_ratios(got, ref, bnd, h, w)[key]
    print(f"\n[negative control] {bug}: worst {key} bound ratio " + " ".join(f"{s}={r:.2f}" for s, r in worst.items()))
    assert max(worst.values()) > 1.0, worst


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("twohot", [False, True], ids=["onehot", "twohot"])
@pytest.mark.parametrize("h,w", GEOMS_HW)
def test_selector_inputs_select_their_closed_form(h, w, twohot):
    B, heads = (1, 1) if h * w > 2000 else (2, 2)
    inp = R.selector_inputs(B, heads, h, w, twohot, seed=h * 1000 + w)
    q, k, _ = R.split_qkv(inp["qkv"], B, heads, h, w)
    s2 = R.LOG2E * R.scores(q, k, inp["th"].double(), inp["tw"].double(), h, w)
    sel = inp["sel"]
    two = sel[..., 1] >= 0
    top = s2.amax(2)
    # argmax of the fp64 scores: one key per query, or exactly two tied ones where the closed form says two
    at_top = s2 == top[..., None]
    cnt = at_top.sum(2)
    assert torch.equal(cnt, 1 + two.long())
    assert torch.equal(torch.gather(at_top, 2, sel[..., :1]).squeeze(2), torch.ones_like(two))
    assert bool(torch.gather(at_top, 2, sel[..., 1:].clamp_min(0)).squeeze(2)[two].all())
    # every other key at least 127 below the maximum in the log2 domain (ex2.approx.ftz gives exactly 0 there)
    masked = s2.masked_fill(at_top, -math.inf)
    if h * w > 1:
        gap = (top - masked.amax(2)).min().item()
        assert gap >= 127.0, gap
    if twohot and h * w >= 4:
        assert bool(two.any()), "no query splits between two keys"
    if not twohot:
        assert not bool(two.any())


@pytest.mark.parametrize("twohot", [False, True], ids=["onehot", "twohot"])
@pytest.mark.parametrize("h,w", [(9, 28), (13, 7), (64, 2), (1, 56), (7, 7), (1, 1)])
def test_selector_expected_values(h, w, twohot):
    """The exact expected values agree with the fp64 reference run on the same inputs (whose exp(-128 ...) tails are
    not exactly zero), are small dyadic numbers, and vanish where the construction says so."""
    B, heads = 2, 2
    inp = R.selector_inputs(B, heads, h, w, twohot, seed=11)
    q, k, v = R.split_qkv(inp["qkv"], B, heads, h, w)
    dO = R.split_heads(inp["dO"], B, heads, h, w)
    th, tw = inp["th"].double(), inp["tw"].double()
    ex = R.selector_expected(inp, B, heads, h, w)
    ref = R.reference(q, k, v, th, tw, dO, h, w)
    for key in ("out", "lse", "dq", "dk", "dv", "dTh", "dTw"):
        scale = ex[key].abs().max().clamp_min(1.0)
        assert (ex[key] - ref[key]).abs().max().item() <= 1e-9 * scale.item(), key
    # the kernel's accumulators (8 dq = dS K + 8 G T, 8 dk = dS^T Q, dv, dT) hold integers or halves below 2^23:
    # every fp32 partial sum of their products is exact
    for key in ("dq", "dk", "dv", "dTh", "dTw"):
        x = ex[key] * 8
        assert torch.equal(x, x.round()) and x.abs().max().item() < 2 ** 24, key
    assert (ex["dS"].abs().max().item() <= 16.0)
    if not twohot:
        for key in ("dq", "dk", "dTh", "dTw"):
            assert not bool(ex[key].any()), key
