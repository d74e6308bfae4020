"""Shared helpers for the exact-arithmetic and per-element error-bound tests of the fused rel-pos attention
(ops.attn_fwd / ops.attn_bwd, painter_b200/csrc/attention.cu).  Nothing here needs a GPU: every function runs on the
device its tensors live on, in the dtype they carry (float64 for the reference and the bounds).

Tensors of one call are batched over a leading "pair" dimension, one entry per (sample, head): q, k, v, dO are
[P, N, 64] with N = h * w, the tables are shared ([2h - 1, 64] / [2w - 1, 64]).

(a) `reference`: forward and backward of models_painter.py:73-86 (q * scale @ k^T, decomposed rel-pos bias, softmax,
    @ v; scale = 64^-0.5 = 1/8) and vitdet_utils.py:96-125 (rel_h[q, i] = q . T_h[i_q - i + h - 1], rel_w[q, j] =
    q . T_w[j_q - j + w - 1], added over image rows / columns of the keys), evaluated in float64 on the bf16 values of
    qkv, the tables and dO.  The backward is written out by hand (dS = P (dP - delta), the bias-row gradients summed
    over image rows / columns, and their Toeplitz scatter G for dQ += G T and dT = G^T Q), so it fits in memory one
    (sample, head) chunk at a time at 112 x 56.
(b) `error_bounds`: per-element forward-error bounds of what the kernel returns, read off its rounding points.
(c) `selector_inputs`: qkv, tables and dO on which the kernel's arithmetic is exact, so results compare bit for bit.
(d) `selector_probs` + `backward`: the exact expected values on those inputs.
"""
import math

import torch

LOG2E = math.log2(math.e)
LN2 = math.log(2.0)
U_BF16 = 2.0 ** -8    # bf16 round to nearest: 8 significant bits
U_F32 = 2.0 ** -24    # fp32 round to nearest (CUDA-core adds, multiplies, fma, 1/l, log2f within 1 ulp)
# wgmma fp32 accumulation: products of bf16 operands are exact; the adds are taken to truncate (2 u_f32) and to lose
# up to another factor 2 aligning the product terms, so each add of a sum contributes 2^-22 of the sum's magnitude
U_TC = 2.0 ** -22
# ex2.approx.ftz.f32: the PTX manual gives a maximum relative error of 2^-22 over the range used; taken with a factor 2
U_EX2 = 2.0 ** -21
# the bounds below are first order in the unit roundoffs; products of two of them (2^-16 relative at most) are covered
# by this factor
SLACK = 1.0 + 2.0 ** -5


def gamma(n, u=U_TC):
    """Standard bound on the relative error of an n-term sum: |fl(sum x) - sum x| <= gamma(n) sum |x|."""
    return n * u / (1.0 - n * u)


def pad16(n):
    return (n + 15) // 16 * 16


def coords(h, w, device):
    """Image (row, column) of every token of an h x w grid, row-major."""
    t = torch.arange(h * w, device=device)
    return t // w, t % w


def toeplitz(n, device):
    """[n, n] table row of (query row, key row): i_q - i + n - 1."""
    a = torch.arange(n, device=device)
    return a[:, None] - a[None, :] + n - 1


def split_qkv(qkv, B, heads, h, w):
    """bf16 [B*N, 3*heads*64] -> float64 q, k, v [B*heads, N, 64]."""
    N = h * w
    x = qkv.double().reshape(B, N, 3, heads, 64).permute(2, 0, 3, 1, 4).reshape(3, B * heads, N, 64)
    return x[0], x[1], x[2]


def split_heads(x, B, heads, h, w):
    """[B*N, heads*64] -> float64 [B*heads, N, 64]."""
    N = h * w
    return x.double().reshape(B, N, heads, 64).permute(0, 2, 1, 3).reshape(B * heads, N, 64)


def bias_rows(q, th, tw, h, w):
    """rel_h [P, N, h] and rel_w [P, N, w]: rel_h[q, i] = q . T_h[i_q - i + h - 1], rel_w[q, j] = q . T_w[j_q - j + w - 1]."""
    P_, N, _ = q.shape
    qg = q.reshape(P_, h, w, 64)
    rh = torch.einsum("pijc,ikc->pijk", qg, th[toeplitz(h, q.device)]).reshape(P_, N, h)
    rw = torch.einsum("pijc,jkc->pijk", qg, tw[toeplitz(w, q.device)]).reshape(P_, N, w)
    return rh, rw


def rel_grads(dS, h, w):
    """Bias-row gradients: dRh[q, i] = sum of dS[q, k] over the keys k of image row i, dRw[q, j] over image column j."""
    P_, N, _ = dS.shape
    ki, kj = coords(h, w, dS.device)
    dRh = dS.new_zeros(P_, N, h).index_add_(2, ki, dS)
    dRw = dS.new_zeros(P_, N, w).index_add_(2, kj, dS)
    return dRh, dRw


def toeplitz_grads(dRh, dRw, h, w):
    """G_h [P, N, 2h-1] with G_h[q, i_q - i + h - 1] = dRh[q, i] (zero elsewhere), likewise G_w: dQ += G_h T_h + G_w T_w,
    dT_h = G_h^T Q."""
    P_, N, _ = dRh.shape
    qi, qj = coords(h, w, dRh.device)
    Gh = dRh.new_zeros(P_, N, 2 * h - 1).scatter_(2, toeplitz(h, dRh.device)[qi].expand(P_, N, h), dRh)
    Gw = dRw.new_zeros(P_, N, 2 * w - 1).scatter_(2, toeplitz(w, dRw.device)[qj].expand(P_, N, w), dRw)
    return Gh, Gw


def scores(q, k, th, tw, h, w):
    """Natural-log-domain scores S [P, N, N] = q k^T / 8 + rel_h[q, i_k] + rel_w[q, j_k]."""
    ki, kj = coords(h, w, q.device)
    rh, rw = bias_rows(q, th, tw, h, w)
    return 0.125 * q @ k.transpose(1, 2) + rh[:, :, ki] + rw[:, :, kj]


def backward(P, O, q, k, v, th, tw, dO, h, w):
    """Gradients of sum(O * dO) through softmax(S) @ v, given the probabilities P [P, N, N] and O = P v."""
    Lh, Lw = 2 * h - 1, 2 * w - 1
    th, tw = th[:Lh], tw[:Lw]
    dv = P.transpose(1, 2) @ dO
    dP = dO @ v.transpose(1, 2)
    delta = (dO * O).sum(2)
    dS = P * (dP - delta[..., None])
    dRh, dRw = rel_grads(dS, h, w)
    Gh, Gw = toeplitz_grads(dRh, dRw, h, w)
    dq = 0.125 * dS @ k + Gh @ th + Gw @ tw
    dk = 0.125 * dS.transpose(1, 2) @ q
    return {"dq": dq, "dk": dk, "dv": dv, "dTh": Gh.transpose(1, 2) @ q, "dTw": Gw.transpose(1, 2) @ q,
            "dP": dP, "delta": delta, "dS": dS, "dRh": dRh, "dRw": dRw}


def reference(q, k, v, th, tw, dO, h, w):
    """fp64 forward and backward of one chunk of (sample, head) pairs.  Returns a dict with out [P, N, 64], lse [P, N]
    (log2 domain, like the kernel: log2 sum_k 2^(S log2 e)), dq, dk, dv [P, N, 64], the per-pair table gradients dTh
    [P, 2h-1, 64] / dTw [P, 2w-1, 64] (the kernel's dT is their sum over pairs) and the intermediates the bounds use."""
    Lh, Lw = 2 * h - 1, 2 * w - 1
    th, tw = th[:Lh], tw[:Lw]
    S = scores(q, k, th, tw, h, w)
    m = S.amax(2, keepdim=True)
    e = torch.exp(S - m)
    l = e.sum(2, keepdim=True)
    P = e / l
    O = P @ v
    r = backward(P, O, q, k, v, th, tw, dO, h, w)
    r.update(out=O, lse=LOG2E * (m + torch.log(l)).squeeze(2), S=S, P=P)
    return r


def error_bounds(r, q, k, v, th, tw, dO, h, w):
    """Per-element bounds on |kernel - reference| for out, lse, dq, dk, dv, and the per-pair parts of the dTh / dTw
    bounds (`table_grad_bound` combines them), from the reference dict `r` of the same inputs.

    Notation: u_b = U_BF16, u = U_F32, g(n) = gamma(n) (tensor-core sums), |x| elementwise magnitudes, n_t = ceil(N/64)
    key tiles, s2 = S log2 e the log2-domain scores.  Each rounding point adds one unit roundoff times the magnitude
    that flows through it; the terms are first order, SLACK covers the rest.

    Forward (attn_fwd_kernel)
      Scores.  s^ = fma(acc(q.k), fl(log2e/8), fl(fl(acc(q.T_h) log2e) + fl(acc(q.T_w) log2e))), every acc a 64-term
        tensor-core sum.  |s^ - s2| <= Es = log2e (g(64) + u) (|q||k|/8 + |q||T_h| + |q||T_w|)
                                            + u (3 |rel_h2| + 3 |rel_w2| + |s2|).
      Probabilities.  p^ = ex2.approx(s^ - m), the running maximum m shared by the whole row (it cancels in O), alpha =
        ex2(m_old - m_new) applied to o and l once per key tile.  Relative error of p^ against the exact weight:
        eta = ln2 (Es + u (|s2 - m2| + range of s2 over the row)) + (n_t + 1) u_ex2 + 2 n_t u.
      out.  O^ = bf16(o / l) with o = sum bf16(p^) v (tensor core, N terms + n_t rescales) and l = sum p^ (fp32, N/4 + n_t
        + 2 adds per row, unrounded p).  The weight errors move O by sum_k P_k (eta_k - eta_bar)(V_k - O), bounded by
        (P eta)|V| + eta_bar (P|V| + 2|O|), eta_bar = sum_k P_k eta_k.
        b_out = u_b |O| (store) + u_b P|V| (P rounded to bf16) + (P eta)|V| + eta_bar (P|V| + 2|O|)
                + (g(N) + n_t u) P|V| + (gamma(N/4 + n_t + 2, u) + 2u) |O|.
      lse = m^ + log2f(l^) = lse2 + log2(1 + sum_k P_k eta_k') + (sum error of l) / ln 2:
        b_lse = log2e (eta_bar + gamma(N/4 + n_t + 2, u)) + 2u (|lse2| + |m2| + 1).
    Backward (attn_bwd_dq_kernel, attn_bwd_dkv_kernel, attn_delta_kernel)
      delta = sum dO O^ in fp32 from the bf16 O^ of the forward: b_delta = |dO| b_out + gamma(64, u) |dO| (|O| + b_out).
      dP = dO . v (tensor core): E_dP = g(64) |dO||V|^T.
      P in the backward: ex2(s^ - lse^), relative error rho = ln2 (Es + u |s2 - lse2| + b_lse) + u_ex2.
      dS^ = p^ (dP^ - delta^) (two fp32 roundings): E_dS = P ((rho + 2u) |dP - delta| + (1 + rho + 2u)(E_dP + b_delta)),
        and the bf16 dS operand of dS K, dS E and dS^T Q: F = E_dS + u_b (|dS| + E_dS).
      dv = bf16(P^T dO) with P^T rounded to bf16: E_P = P (rho + u_b (1 + rho)),
        b_dv = e + u_b (|dv| + e),  e = E_P^T |dO| + g(N) (P + E_P)^T |dO|.
      dk = bf16(dS^T Q / 8): e = (F^T |Q| + g(N) (|dS| + F)^T |Q|) / 8, b_dk = e + u_b (|dk| + e).
      Bias-row gradients dRh, dRw: sums of the bf16 dS over the keys of an image row / column (dS E per key tile, then
        fp32 adds across tiles; with w = 1 dRw is the fp32 sum of dRh): E_R = sum F + g(N + n_t + h) sum (|dS| + F).
        G is rounded to bf16 for both G T and G^T Q: E_G = E_R + u_b (|dR| + E_R), scattered to table rows.
      dq = bf16(dS K / 8 + G [T_h; T_w]): e = F|K|/8 + E_Gh|T_h| + E_Gw|T_w|
                                             + g(N + 2h-1 + 2w-1) ((|dS| + F)|K|/8 + |G~h||T_h| + |G~w||T_w|),
        |G~| = |G| + E_G,  b_dq = e + u_b (|dq| + e).
      dT = G^T Q in fp32 (64 queries per dQ CTA on the tensor core, then a sum over the CTAs' partials and four
        atomic stripes): per pair E_G^T |Q| and |G~|^T |Q|; `table_grad_bound` adds g(64 + CTAs + 24) of the latter.
    """
    N = h * w
    nt = (N + 63) // 64
    Lh, Lw = 2 * h - 1, 2 * w - 1
    th, tw = th[:Lh], tw[:Lw]
    ki, kj = coords(h, w, q.device)
    aq, ak, av, adO, ath, atw = q.abs(), k.abs(), v.abs(), dO.abs(), th.abs(), tw.abs()
    u = U_F32
    # forward
    A = 0.125 * aq @ ak.transpose(1, 2)
    Bh, Bw = bias_rows(aq, ath, atw, h, w)
    rh, rw = bias_rows(q, th, tw, h, w)
    rh2, rw2 = LOG2E * rh.abs()[:, :, ki], LOG2E * rw.abs()[:, :, kj]
    s2 = LOG2E * r["S"]
    m2 = s2.amax(2, keepdim=True)
    rng = m2 - s2.amin(2, keepdim=True)
    Es = LOG2E * (gamma(64) + u) * (A + Bh[:, :, ki] + Bw[:, :, kj]) + u * (3 * rh2 + 3 * rw2 + s2.abs())
    del A, rh2, rw2
    eta = LN2 * (Es + u * ((s2 - m2).abs() + rng)) + (nt + 1) * U_EX2 + 2 * nt * u
    P, O = r["P"], r["out"]
    aO = O.abs()
    Peta = P * eta
    del eta
    etabar = Peta.sum(2, keepdim=True)
    PaV = P @ av
    gl = gamma((N + 3) // 4 + nt + 2, u)
    b_out = SLACK * (U_BF16 * (aO + PaV) + Peta @ av + etabar * (PaV + 2 * aO) + (gamma(N) + nt * u) * PaV
                     + (gl + 2 * u) * aO)
    del Peta
    lse2 = r["lse"]
    b_lse = SLACK * (LOG2E * (etabar.squeeze(2) + gl) + 2 * u * (lse2.abs() + m2.squeeze(2).abs() + 1.0))
    # backward
    b_delta = (adO * b_out).sum(2) + gamma(64, u) * (adO * (aO + b_out)).sum(2)
    E_dP = gamma(64) * adO @ av.transpose(1, 2)
    rho = LN2 * (Es + u * (s2 - lse2[..., None]).abs() + b_lse[..., None]) + U_EX2
    del Es, s2
    D = (r["dP"] - r["delta"][..., None]).abs()
    E_dS = P * ((rho + 2 * u) * D + (1 + rho + 2 * u) * (E_dP + b_delta[..., None]))
    del D, E_dP
    adS = r["dS"].abs()
    F = E_dS + U_BF16 * (adS + E_dS)
    del E_dS
    dSm = adS + F
    E_P = P * (rho + U_BF16 * (1 + rho))
    del rho
    e = E_P.transpose(1, 2) @ adO + gamma(N) * (P + E_P).transpose(1, 2) @ adO
    del E_P
    b_dv = SLACK * (e + U_BF16 * (r["dv"].abs() + e))
    e = 0.125 * (F.transpose(1, 2) @ aq + gamma(N) * dSm.transpose(1, 2) @ aq)
    b_dk = SLACK * (e + U_BF16 * (r["dk"].abs() + e))
    Fh, Fw = rel_grads(F, h, w)
    Mh, Mw = rel_grads(dSm, h, w)
    nr = N + nt + h
    ERh, ERw = Fh + gamma(nr) * Mh, Fw + gamma(nr) * Mw
    EGh_, EGw_ = ERh + U_BF16 * (r["dRh"].abs() + ERh), ERw + U_BF16 * (r["dRw"].abs() + ERw)
    EGh, EGw = toeplitz_grads(EGh_, EGw_, h, w)
    MGh, MGw = toeplitz_grads(r["dRh"].abs() + EGh_, r["dRw"].abs() + EGw_, h, w)
    e = (0.125 * F @ ak + EGh @ ath + EGw @ atw
         + gamma(N + Lh + Lw) * (0.125 * dSm @ ak + MGh @ ath + MGw @ atw))
    b_dq = SLACK * (e + U_BF16 * (r["dq"].abs() + e))
    return {"out": b_out, "lse": b_lse, "dq": b_dq, "dk": b_dk, "dv": b_dv,
            "dTh_E": EGh.transpose(1, 2) @ aq, "dTh_M": MGh.transpose(1, 2) @ aq,
            "dTw_E": EGw.transpose(1, 2) @ aq, "dTw_M": MGw.transpose(1, 2) @ aq}


def table_grad_bound(E, M, nctas):
    """Bound on the kernel's table gradient from the per-pair parts summed over the pairs of the call (E, M: sums of
    error_bounds' dTh_E / dTh_M or dTw_E / dTw_M); nctas = B * heads * ceil(N / 64) partial slices."""
    return SLACK * (E + gamma(64 + nctas + 24) * M)


# ----------------------------------------------------------------------------------------------------------------
# (c) selector inputs
# ----------------------------------------------------------------------------------------------------------------
PEAK = 128.0   # table slope: the next-best key scores 128 below the selected one, 128 log2 e = 184.7 in log2 units


def selector_inputs(B, heads, h, w, twohot, seed=0, device="cpu"):
    """qkv (bf16 [B*N, 3*heads*64]), tables (bf16, zero-padded to 16 rows), dO (bf16 [B*N, heads*64]) on which the
    kernel's arithmetic is exact, and the keys every query selects: sel [B*heads, N, 2] (second entry -1 for a single
    key).

    Construction.  Table columns d = 0..15 are peaked, T[r, d] = -128 |r - r0_d| (integers times 128 up to 128 * 222:
    bf16-exact for every row of a 112 x 56 grid); dims 16..63 of both tables are zero.  Every query's q is one-hot over
    dims 0..15 (value 1 at a dim d drawn per (sample, head, query)), so its bias rows are exactly column d of the
    tables: rel_h[q, i] + rel_w[q, j] = -128 (|i - (i_q + h-1 - r0h_d)| + |j - (j_q + w-1 - r0w_d)|), largest (0) at
    the nearest valid key to the peak, every other key at least 128 below.  k is zero on dims 0..15.  One-hot variant:
    dims 16..63 of q and k are in {-1, 0, 1}, so q.k/8 is an exact multiple of 1/8 of magnitude <= 6 and moves no key
    across the 128 gap.  Two-hot variant: dims 8..15 get a second peak at r1 = r0 + sep (1 <= sep <= n) in the table
    of the longer image axis; q is zero on dims 16..63, so a query whose two peaks both fall inside the grid scores
    both keys exactly 0 and splits 1/2 : 1/2 (with sep <= n, a query with a peak outside the grid still has a unique
    nearest key).  Every other key lies >= 127 below the maximum in the log2 domain, where ex2.approx.ftz flushes to 0.

    Magnitudes.  One-hot: v in [-8, 8], dO in {-1, 0, 1}; dS = 0 (dP - delta = 0 with O exact), so dq = dk = dT = 0 and
    dv = sum of dO over the queries selecting the key.  Two-hot: v in {0, 4}, dO in {-1, 0, 1} on dims 0..15 only, so
    O = (V1 + V2)/2 is exact, dS = +-(1/4) dO.(V1 - V2) is an integer of magnitude <= 16, 8 G T (the dQ tail's
    operands) an integer < 2^23, and every fp32 partial sum of every product is an integer or a half below 2^24: exact.
    The kernel's results are then bf16_rn(exact) (dqkv, out) and exact (dTh, dTw).

    One assumption is unmeasured: that ex2.approx.ftz.f32(0) is exactly 1 (and ex2(-1) exactly 1/2).  The construction
    does not depend on it: a p of 1 - eps (eps ~ 2^-22) rounds to 1 in bf16 before P V and P^T dO, scales O and dS by
    1 + O(eps) before their bf16 rounding, and moves the integer or half-integer results by far less than half a bf16
    ulp, so the bf16 outputs are the same.
    """
    g = torch.Generator().manual_seed(seed)
    N, Pn, Lh, Lw = h * w, B * heads, 2 * h - 1, 2 * w - 1
    r0h = torch.randint(0, Lh, (16,), generator=g)
    r0w = torch.randint(0, Lw, (16,), generator=g)
    ax = ("h" if h >= 2 else "w" if w >= 2 else None) if twohot else None
    two = torch.zeros(16, dtype=torch.bool)
    r1 = torch.full((16,), -1, dtype=torch.long)
    if ax is not None:
        n = h if ax == "h" else w
        sep = torch.randint(1, n + 1, (8,), generator=g)
        r0 = (torch.rand(8, generator=g) * (2 * n - 1 - sep)).long()   # r0 in [0, 2n - 2 - sep]
        (r0h if ax == "h" else r0w)[8:] = r0
        r1[8:] = r0 + sep
        two[8:] = True
    rows = torch.arange(Lh)[:, None].double()
    cols = torch.arange(Lw)[:, None].double()
    th = torch.zeros(pad16(Lh), 64, dtype=torch.float64)
    tw = torch.zeros(pad16(Lw), 64, dtype=torch.float64)
    th[:Lh, :16] = -PEAK * (rows - r0h[None].double()).abs()
    tw[:Lw, :16] = -PEAK * (cols - r0w[None].double()).abs()
    if ax is not None:
        t2, L2 = (th, Lh) if ax == "h" else (tw, Lw)
        rr = torch.arange(L2)[:, None].double()
        t2[:L2, 8:16] = -PEAK * torch.minimum((rr - r0[None].double()).abs(), (rr - r1[8:][None].double()).abs())
    dsel = torch.randint(0, 16, (Pn, N), generator=g)
    q = torch.zeros(Pn, N, 64, dtype=torch.float64)
    q.scatter_(2, dsel[..., None], 1.0)
    k = torch.zeros(Pn, N, 64, dtype=torch.float64)
    k[:, :, 16:] = torch.randint(-1, 2, (Pn, N, 48), generator=g).double()
    dO = torch.zeros(Pn, N, 64, dtype=torch.float64)
    if twohot:
        v = 4.0 * torch.randint(0, 2, (Pn, N, 64), generator=g).double()
        dO[:, :, :16] = torch.randint(-1, 2, (Pn, N, 16), generator=g).double()
    else:
        q[:, :, 16:] = torch.randint(-1, 2, (Pn, N, 48), generator=g).double()
        v = torch.randint(-8, 9, (Pn, N, 64), generator=g).double()
        dO[:] = torch.randint(-1, 2, (Pn, N, 64), generator=g).double()
    # closed-form selection
    qi, qj = coords(h, w, "cpu")
    ah = qi[None] + h - 1 - r0h[dsel]          # peak key row / column of every query
    aw = qj[None] + w - 1 - r0w[dsel]
    rowa, cola = ah.clamp(0, h - 1), aw.clamp(0, w - 1)
    sel = torch.stack([rowa * w + cola, torch.full_like(rowa, -1)], 2)
    if ax is not None:
        a0, n = (ah, h) if ax == "h" else (aw, w)
        a1 = a0 - (r1[dsel] - (r0h if ax == "h" else r0w)[dsel])
        ok0, ok1 = (a0 >= 0) & (a0 < n), (a1 >= 0) & (a1 < n)
        isw = two[dsel]
        alt = a1.clamp(0, n - 1)
        second = alt * w + cola if ax == "h" else rowa * w + alt
        both = isw & ok0 & ok1
        only1 = isw & ~ok0 & ok1
        sel[..., 0] = torch.where(only1, second, sel[..., 0])
        sel[..., 1] = torch.where(both, second, sel[..., 1])

    def pack(x):      # [B*heads, N, 64] -> [B*N, heads*64]
        return x.reshape(B, heads, N, 64).permute(0, 2, 1, 3).reshape(B * N, heads * 64)

    qkv = torch.cat([pack(q), pack(k), pack(v)], 1).to(torch.bfloat16)
    return {"qkv": qkv.to(device), "th": th.to(torch.bfloat16).to(device), "tw": tw.to(torch.bfloat16).to(device),
            "dO": pack(dO).to(torch.bfloat16).to(device), "sel": sel.to(device)}


def selector_probs(sel, N):
    """Exact probabilities [P, N, N] of a selection map: 1 on the selected key, 1/2 on each of two."""
    Pn = sel.shape[0]
    P = torch.zeros(Pn, N, N, dtype=torch.float64, device=sel.device)
    two = sel[..., 1] >= 0
    P.scatter_(2, sel[..., :1], torch.where(two, 0.5, 1.0)[..., None].double())
    P.scatter_add_(2, sel[..., 1:].clamp_min(0), two[..., None].double() * 0.5)
    return P


def selector_expected(inp, B, heads, h, w, pairs=None):
    """Exact expected kernel results on selector inputs for the pairs `pairs` (a slice or index tensor of the
    B*heads pairs; default all): out, lse (fp64; the kernel's fp32 lse is compared within a few ulps), dq, dk, dv
    [P, N, 64] (exact; the kernel returns their bf16 rounding) and the per-pair dTh, dTw (exact sums)."""
    N = h * w
    q, k, v = split_qkv(inp["qkv"], B, heads, h, w)
    dO = split_heads(inp["dO"], B, heads, h, w)
    sel = inp["sel"]
    if pairs is not None:
        q, k, v, dO, sel = q[pairs], k[pairs], v[pairs], dO[pairs], sel[pairs]
    th, tw = inp["th"].double(), inp["tw"].double()
    P = selector_probs(sel, N)
    O = P @ v
    r = backward(P, O, q, k, v, th, tw, dO, h, w)
    # score of the (first) selected key: q.k / 8 plus its bias, which is -128 times its distance to a peak outside the grid
    s0 = sel[..., :1]
    rh, rw = bias_rows(q, th[:2 * h - 1], tw[:2 * w - 1], h, w)
    s = (0.125 * (q * torch.gather(k, 1, s0.expand(-1, -1, 64))).sum(2) + torch.gather(rh, 2, s0 // w).squeeze(2)
         + torch.gather(rw, 2, s0 % w).squeeze(2))
    r.update(out=O, lse=LOG2E * s + torch.where(sel[..., 1] >= 0, 1.0, 0.0).double())
    return r
