"""Exact-arithmetic tests of the wgmma GEMM (ops.gemm) and of the decoder's implicit-GEMM 3x3 convolutions.

The operands are small integers stored as bf16 and every accumulator stays below 2^16 (below 2^24 for the fp32
weight gradient of the convolution), so each partial sum is an integer that fp32 holds exactly, whatever the
summation order, the tile width, split-K or the stream-K atomics.  The reference is the same product in float64 on
the GPU.  fp32 outputs must equal it cast to fp32; bf16 outputs must equal it cast to fp32 and then rounded to bf16
(round to nearest even in both code paths).  So a kernel that reorders its sums passes and a kernel with one wrong
element fails.  Every buffer a call writes is filled with NaN beyond the view the kernel is given (a row above, 130
rows below, and the columns around the view when it is a column slice); those sentinels must survive the call.

The GELU / GELU' epilogues are transcendental.  Every bf16 value in [-10, 10] is driven through them and compared
per element with float64 x Phi(x) and Phi(x) + x phi(x), at the accuracy common.cuh documents for the fitted
polynomial (2.5e-5 and 1.1e-4 absolute), on top of one bf16 ulp for the stored result."""
import contextlib
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32
DROP_SCALES = (0.0, 0.5, 1.0, 1.25)   # DropPath row scales (keep probability 0.8 gives 1.25)


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)


def _lib():
    from painter_b200 import _lib
    return _lib.lib()


def _ints(shape, lim, dtype=BF16, device=DEV):
    return torch.randint(-lim, lim + 1, tuple(shape), device=device).to(dtype)


def _nan_view(rows, cols, dtype, strided=False):
    """(buffer, view, region): a NaN-filled buffer and a [rows, cols] view of it, buffer[region].  The row stride is
    a multiple of 8 elements (16 bytes, as TMA and the vector stores need).  The buffer has one row above the view and
    130 below it (past the next 128-row tile).  strided: the view is a column slice that starts 8 elements in and has
    24 more columns to its right."""
    c0 = 8 if strided else 0
    ld = c0 + -(-cols // 8) * 8 + (24 if strided else 0)
    buf = torch.full((rows + 131, ld), float("nan"), dtype=dtype, device=DEV)
    region = (slice(1, rows + 1), slice(c0, c0 + cols))
    return buf, buf[region], region


def _nan_flat(shape, dtype):
    """(buffer, view, region) for a contiguous output: the view sits between two runs of 64 NaN elements."""
    n = math.prod(shape)
    buf = torch.full((n + 128,), float("nan"), dtype=dtype, device=DEV)
    region = (slice(64, 64 + n),)
    return buf, buf[region].view(shape), region


def _assert_equal(got, want, what):
    if torch.equal(got, want):
        return
    bad = (got != want).nonzero()
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{what}: {bad.shape[0]} of {got.numel()} elements differ; first at {i}: got "
                         f"{got[i].item()}, want {want[i].item()}")


def _assert_sentinels(buf, region, what):
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[region] = False
    written = outside & ~buf.isnan()
    if written.any():
        i = tuple(written.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(written.sum())} elements written outside the view, first at buffer "
                             f"index {i} (view {region})")


@contextlib.contextmanager
def _forced(bn=0, splits=0):
    lib = _lib()
    lib.pk_gemm_force_bn(bn)
    lib.pk_gemm_force_splits(splits)
    try:
        yield
    finally:
        lib.pk_gemm_force_bn(0)
        lib.pk_gemm_force_splits(0)


def _plan(M, N, K, kind, accumulate):
    """the planner's decisions for a call (the same host code pk_gemm_bf16 runs, honouring forced settings)"""
    out = (ctypes.c_int * 9)()
    assert _lib().pk_gemm_plan(M, N, K, kind, accumulate, out) == 0
    return dict(zip(["pair", "BN", "mt", "nt", "splits", "kbps", "sk_units", "group_m", "workers"], list(out)))


# ------------------------------------------------------ GELU references ------------------------------------------
def _gelu64(x):
    return x * torch.special.ndtr(x)


def _gelu_grad64(x):
    return torch.special.ndtr(x) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def _ulp_bf16(r):
    """spacing of bf16 numbers at |r| (r a bf16 tensor), as float64"""
    _, e = torch.frexp(r.double())
    ulp = torch.ldexp(torch.ones_like(r, dtype=torch.float64), e - 8).clamp_min(2.0 ** -133)
    return torch.where(r == 0, 2.0 ** -133, ulp)


GELU_SLACK, GELU_GRAD_SLACK = 2.0 ** -15, 2.0 ** -13   # cover the fit's documented 2.5e-5 and 1.1e-4


def _gelu_errors(got, x, grad):
    """(|got - ref|, bar, ref) per element; ref = bf16(float64 GELU or GELU' of x)"""
    ref = (_gelu_grad64 if grad else _gelu64)(x.double()).float().bfloat16()
    err = (got.double() - ref.double()).abs()
    bar = _ulp_bf16(ref) + (GELU_GRAD_SLACK if grad else GELU_SLACK)
    return err, bar, ref


def _assert_gelu_within_bar(got, z, grad, what):
    err, bar, ref = _gelu_errors(got, z, grad)
    bad = ~(err <= bar)
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} elements beyond 1 ulp + {'2^-13' if grad else '2^-15'}; "
                             f"first at {i}: x = {z[i].item()}, got {got[i].item()}, want {ref[i].item()}")


# ------------------------------------------------------ exact GEMM probes ----------------------------------------
KINDS = {   # name: (epilogue kind, accumulate)
    "bf16": (0, 0), "f32": (1, 0), "f32_acc": (1, 1), "wgrad": (1, 2), "gelu": (2, 0), "resid": (3, 0),
    "dgelu": (4, 0), "pixshuf": (5, 0),
}


def _check_gemm(M, N, K, kind, ta=False, tb=False, strided=False, rows_per_group=None, pixshuf=None):
    """One ops.gemm call with integer operands against the float64 product, every output element exact and every
    sentinel around the outputs intact.  kind: a key of KINDS ("wgrad": zero-initialised fp32 output with split-K /
    stream-K atomics, called twice so that the second call adds).  strided: A, B, out and aux are column slices of
    wider buffers.  rows_per_group: the residual epilogue's DropPath row scales (None: no row scale).  pixshuf:
    (B, h, w, p, c) of the pixel-shuffle epilogue."""
    from painter_b200 import ops
    lim = 4 if K <= 2048 else 2                   # |acc| <= K lim^2 <= 2^15
    _, a, _ = _nan_view(*((K, M) if ta else (M, K)), BF16, strided)
    _, b, _ = _nan_view(*((K, N) if tb else (N, K)), BF16, strided)
    a.copy_(_ints(a.shape, lim))
    b.copy_(_ints(b.shape, lim))
    acc = (a.double().t() if ta else a.double()) @ (b.double() if tb else b.double().t())
    bias = _ints((N,), 16, F32)
    kw = dict(trans_a=ta, trans_b=tb, kind=KINDS[kind][0])
    checks = []   # (name, buffer, region, view, exact reference)
    if kind in ("bf16", "f32", "f32_acc", "wgrad", "resid", "dgelu", "gelu"):
        odt = F32 if kind in ("f32", "f32_acc", "wgrad", "resid") else BF16
        obuf, out, oreg = _nan_view(M, N, odt, strided)
        kw["out"] = out
    if kind == "bf16":
        kw["bias"] = bias
        checks.append(("out", obuf, oreg, out, (acc + bias.double()).float().bfloat16()))
    elif kind == "f32":
        kw["bias"] = bias
        checks.append(("out", obuf, oreg, out, (acc + bias.double()).float()))
    elif kind == "f32_acc":
        init = _ints((M, N), 64, F32)
        out.copy_(init)
        kw.update(bias=bias, accumulate=1)
        checks.append(("out", obuf, oreg, out, (init.double() + acc + bias.double()).float()))
    elif kind == "wgrad":
        out.zero_()
        kw["accumulate"] = 2
        checks.append(("out", obuf, oreg, out, (2 * acc).float()))
    elif kind == "resid":
        _, aux, _ = _nan_view(M, N, F32, strided)
        aux.copy_(_ints((M, N), 64, F32))
        kw.update(bias=bias, aux=aux)
        scale = torch.ones(M, 1, dtype=torch.float64, device=DEV)
        if rows_per_group is not None:
            groups = -(-M // rows_per_group)
            rs = torch.tensor(DROP_SCALES, device=DEV)[torch.randint(0, 4, (groups,), device=DEV)]
            kw.update(rowscale=rs, rows_per_group=rows_per_group)
            scale = rs.double().repeat_interleave(rows_per_group)[:M, None]
        checks.append(("out", obuf, oreg, out, (aux.double() + scale * (acc + bias.double())).float()))
    elif kind == "dgelu":
        # GELU'(0) = 0.5 and GELU'(16) = 1 (to 1e-55), so the product stays exact; which of the two each element
        # gets checks that the saved pre-activation is read at the right place
        _, aux, _ = _nan_view(M, N, BF16, strided)
        aux.copy_((torch.randint(0, 2, (M, N), device=DEV) * 16).to(BF16))
        kw["aux"] = aux
        checks.append(("out", obuf, oreg, out, (acc * torch.where(aux.double() > 0, 1.0, 0.5)).float().bfloat16()))
    elif kind == "gelu":
        hbuf, hact, hreg = _nan_view(M, N, BF16, strided)
        kw.update(bias=bias, out2=hact)
        checks.append(("z", obuf, oreg, out, (acc + bias.double()).float().bfloat16()))
    else:
        assert kind == "pixshuf"
        B, h, w, p, c = pixshuf
        assert M == B * h * w and N == p * p * c
        obuf, out, oreg = _nan_flat((B, h * p, w * p, c), BF16)
        kw.update(bias=bias, pixshuf=(h, w, p, c, out))
        want = (acc + bias.double()).reshape(B, h, w, p, p, c).permute(0, 1, 3, 2, 4, 5).reshape(B, h * p, w * p, c)
        checks.append(("out", obuf, oreg, out, want.float().bfloat16()))

    ops.gemm(a, b, **kw)
    if kind == "wgrad":
        ops.gemm(a, b, **kw)
    torch.cuda.synchronize()
    what = f"{kind} M={M} N={N} K={K} ta={int(ta)} tb={int(tb)} strided={int(strided)}"
    for name, buf, region, view, want in checks:
        _assert_equal(view, want, f"{what}: {name}")
        _assert_sentinels(buf, region, f"{what}: {name}")
    if kind == "gelu":
        _assert_gelu_within_bar(hact, out, False, f"{what}: gelu(z)")
        _assert_sentinels(hbuf, hreg, f"{what}: gelu(z)")


LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]


@pytest.mark.parametrize("kind", ["bf16", "f32", "f32_acc", "resid", "gelu", "dgelu", "pixshuf"])
@pytest.mark.parametrize("ta,tb", LAYOUTS)
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_gemm_exact_every_tile_width_and_layout(bn, ta, tb, kind):
    """Every epilogue at every tile width and operand layout, on strided views (lda, ldb, ldc, ld_aux beyond the
    matrix), with a ragged M (three row blocks, the last one 44 rows) and a ragged K (the last K-block 8 deep)."""
    M, N, K = 300, 1024, 200
    with _forced(bn=bn):
        assert _plan(M, N, K, *KINDS[kind])["BN"] == bn
        _check_gemm(M, N, K, kind, ta, tb, strided=True, rows_per_group=37, pixshuf=(3, 10, 10, 4, 64))


RAGGED = [   # (M, N, K, trans_a, trans_b): every M in {1, 127, 129, 300, 4000}, K in {8, 72, 200, 1000},
    (1, 64, 8, False, False),       # N in {64, 192, 320, 1024, 3072}, each operand layout
    (1, 3072, 1000, True, True),
    (127, 192, 72, True, False),
    (127, 1024, 200, False, True),
    (129, 320, 1000, False, False),
    (129, 64, 72, True, True),
    (129, 1024, 8, True, False),
    (300, 3072, 8, False, True),
    (300, 192, 200, True, True),
    (4000, 320, 200, True, False),
    (4000, 3072, 72, False, False),
    (4000, 64, 1000, False, True),
]


@pytest.mark.parametrize("kind", ["bf16", "f32"])
@pytest.mark.parametrize("M,N,K,ta,tb", RAGGED)
def test_gemm_exact_ragged_shapes(M, N, K, ta, tb, kind):
    """Ragged shapes at the tile width the planner picks, contiguous operands (padded to a 16-byte row stride where
    the transposed layout needs it, e.g. M = 127 stored [K, M])."""
    _check_gemm(M, N, K, kind, ta, tb)


@pytest.mark.parametrize("kind", ["bf16", "gelu", "f32", "resid"])
@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("K", [72, 300])
def test_gemm_exact_persistent_tiles(K, bn, kind):
    """More tiles than SMs with a short K: every persistent CTA walks several tiles, so each epilogue overlaps the
    next tile's main loop, and with 2 or 5 K-blocks per tile the operand ring (8, 5 or 4 stages at BN = 64, 128,
    256) wraps inside a tile."""
    M, N = 4000, 2048
    with _forced(bn=bn):
        p = _plan(M, N, K, *KINDS[kind])
        assert p["BN"] == bn and p["mt"] * p["nt"] > torch.cuda.get_device_properties(0).multi_processor_count
        _check_gemm(M, N, K, kind, strided=(K == 300))


@pytest.mark.parametrize("kind", ["bf16", "f32"])
@pytest.mark.parametrize("M", [300, 1100])
def test_gemm_exact_grouped_rasterisation(M, kind):
    """B too large for L2 (N K 2 > 40 MB): tiles are rasterised in groups of 8 row blocks; M = 1100 leaves a last
    group of one row block, M = 300 a single group of three."""
    N, K = 8192, 4096
    assert _plan(M, N, K, *KINDS[kind])["group_m"] == 8
    _check_gemm(M, N, K, kind, ta=(M == 300))


@pytest.mark.parametrize("splits", [2, 3, 7])
@pytest.mark.parametrize("M,N,K,ta,tb", [(300, 320, 1000, True, True), (129, 1024, 2050, False, False)])
def test_gemm_exact_split_k(M, N, K, ta, tb, splits):
    """Classic split-K (forced): fp32 atomics of integer partial tiles are exact, so the result is bit-exact; the
    last split is shorter than the others."""
    with _forced(splits=splits):
        assert _plan(M, N, K, *KINDS["wgrad"])["splits"] > 1
        _check_gemm(M, N, K, "wgrad", ta, tb, strided=(M == 300))


@pytest.mark.parametrize("M,N,K,ta,tb", [(1000, 1024, 1300, True, True), (300, 1024, 3000, True, True),
                                          (4000, 192, 1000, False, False), (129, 3072, 1000, True, False)])
def test_gemm_exact_stream_k(M, N, K, ta, tb):
    """Planner-chosen stream-K on ragged shapes: the per-CTA unit ranges do not align with the tiles, so tiles
    straddle ranges and are completed with fp32 atomics."""
    p = _plan(M, N, K, *KINDS["wgrad"])
    num_kb = -(-K // 64)
    assert p["sk_units"] > 0 and num_kb % p["sk_units"] != 0
    _check_gemm(M, N, K, "wgrad", ta, tb, strided=(M == 1000))


@pytest.mark.parametrize("M,rows_per_group", [(4000, 37), (4000, 300), (3136, 1568)])
def test_gemm_exact_row_groups(M, rows_per_group):
    """DropPath row scales whose groups do not line up with the epilogue: 37 and 300 rows are not multiples of its
    32-row chunks, and 1568 (the tokens of one 896 x 448 image) is not a multiple of its 128-row tiles."""
    _check_gemm(M, 1024, 200, "resid", rows_per_group=rows_per_group)


# ------------------------------------------------------ exact convolution probes ---------------------------------
def _im2col64(x):
    """[B, H, W, C] -> float64 [B*H*W, 9*C]: every pixel's 3x3 neighbourhood (zero padding), taps (dy, dx)
    row-major, channels innermost"""
    B, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[:, dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], dim=-1).reshape(-1, 9 * C)


def _conv_fwd64(g, w, bias):
    """conv2d(g, w, bias, padding=1) of NHWC g as float64 [B*H*W, 64]"""
    return _im2col64(g) @ w.double().permute(0, 2, 3, 1).reshape(64, 576).t() + bias.double()


def _conv_dgrad64(dc1, w):
    """conv_transpose2d(dc1, w, padding=1) (the input gradient of the convolution) of NHWC dc1, float64 [B*H*W, 64]:
    the same 3x3 neighbourhoods against the taps flipped and the channels swapped"""
    return _im2col64(dc1) @ w.double().flip(2, 3).permute(1, 2, 3, 0).reshape(64, 576).t()


def _conv_wgrad64(g, dc1):
    """the weight gradient of the convolution in the kernel's accumulator layout [tap * 64 + c, o], float64"""
    return _im2col64(g).t() @ dc1.reshape(-1, 64).double()


def test_conv_reference_is_torch_conv():
    """The im2col restatements above are torch's conv2d, conv_transpose2d and conv2d weight gradient (computed on
    the CPU, where torch sums these integer products exactly)."""
    F = torch.nn.functional
    B, H, W = 2, 12, 8
    g, dc1 = _ints((B, H, W, 64), 2, device="cpu"), _ints((B, H, W, 64), 2, device="cpu")
    w, bias = _ints((64, 64, 3, 3), 2, F32, "cpu"), _ints((64,), 16, F32, "cpu")
    nchw = lambda t: t.double().permute(0, 3, 1, 2)
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(-1, 64)
    assert torch.equal(_conv_fwd64(g, w, bias), nhwc(F.conv2d(nchw(g), w.double(), bias.double(), padding=1)))
    assert torch.equal(_conv_dgrad64(dc1, w), nhwc(F.conv_transpose2d(nchw(dc1), w.double(), padding=1)))
    dw = torch.nn.grad.conv2d_weight(nchw(g), (64, 64, 3, 3), nchw(dc1), padding=1)
    assert torch.equal(_conv_wgrad64(g, dc1), dw.permute(2, 3, 1, 0).reshape(576, 64))


CONV_GEOMETRIES = [(1, 128, 64), (3, 64, 32), (1, 896, 448)]   # 64 / 32 / 64 pixels per tile row


@pytest.mark.parametrize("entry", ["head_c1", "dgrad_unshuffle", "wgrad"])
@pytest.mark.parametrize("B,H,W", CONV_GEOMETRIES)
def test_conv3x3_exact(B, H, W, entry):
    """The implicit-GEMM convolutions: the decoder head's bf16 conv output c1 = bf16(conv + bias), the input gradient
    with the inverse pixel shuffle (bf16) and the fp32 weight gradient (split-K atomics, partial sums < 2^24)."""
    from painter_b200 import ops
    p = 16
    h, w = H // p, W // p
    lib, st = _lib(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    g, dc1 = _ints((B, H, W, 64), 2), _ints((B, H, W, 64), 2)
    wc, bias = _ints((64, 64, 3, 3), 2, F32), _ints((64,), 16, F32)
    wf, wd = ops.conv3x3_pack(wc)
    what = f"{entry} B={B} H={H} W={W}"
    if entry == "head_c1":
        hp = torch.cat([bias, 1 + 0.1 * torch.randn(64, device=DEV), 0.1 * torch.randn(64, device=DEV),
                        0.2 * torch.randn(195, device=DEV), torch.zeros(5, device=DEV)])
        tgts = torch.randn(B, 3, H, W, device=DEV)
        mask = (torch.rand(B, h * w, device=DEV) < 0.5).to(torch.uint8)
        valid = torch.ones(B, 3, H, W, device=DEV)
        patch = torch.empty(B, h * w, p * p * 3, device=DEV)
        num = torch.zeros(B, device=DEV)
        buf, got, region = _nan_flat((B, H, W, 64), BF16)
        assert lib.pk_decoder_head_fwd(ptr(g), ptr(wf), ptr(hp), ptr(tgts), ptr(mask), B, ptr(valid), ptr(got),
                                       ptr(patch), ptr(num), B, H, W, p, 0, st) == 0
        want = _conv_fwd64(g, wc, bias).float().bfloat16().view(B, H, W, 64)
    elif entry == "dgrad_unshuffle":
        buf, got, region = _nan_flat((B * h * w, p * p * 64), BF16)
        assert lib.pk_conv3x3_dgrad_unshuffle(ptr(dc1), ptr(wd), ptr(got), B, H, W, p, st) == 0
        want = _conv_dgrad64(dc1, wc).float().bfloat16().reshape(B, h, p, w, p, 64).permute(0, 1, 3, 2, 4, 5)
        want = want.reshape(B * h * w, p * p * 64)
    else:
        ref = _conv_wgrad64(g, dc1)
        assert ref.abs().max() < 2 ** 24
        buf = torch.full((64 + 640 + 64, 64), float("nan"), device=DEV)   # 576 rows, padded to 5 row blocks
        region = (slice(64, 704),)
        got = buf[region]
        got.zero_()
        assert lib.pk_conv3x3_wgrad(ptr(g), ptr(dc1), ptr(got), B, H, W, st) == 0
        want = torch.cat([ref.float(), torch.zeros(64, 64, device=DEV)])   # the padding rows stay zero
    torch.cuda.synchronize()
    _assert_equal(got, want, what)
    _assert_sentinels(buf, region, what)
    if entry == "wgrad":
        dw = torch.empty(64, 64, 3, 3, device=DEV)
        assert lib.pk_conv3x3_wgrad_unpack(ptr(got), ptr(dw), st) == 0
        _assert_equal(dw, want[:576].view(3, 3, 64, 64).permute(3, 2, 0, 1), f"{what}: unpacked [o, c, dy, dx]")


# ------------------------------------------------------ GELU / GELU' sweep -----------------------------------------
def _bf16_sweep(lo, hi):
    """every bf16 value in [lo, hi], ascending (one zero)"""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF16).float()
    return torch.unique(x[torch.isfinite(x) & (x >= lo) & (x <= hi)]).to(DEV)


def _report(name, got, x, grad):
    """print the worst error: in bf16 ulps where one ulp of the result is at least the slack, absolute elsewhere"""
    err, bar, ref = _gelu_errors(got, x, grad)
    ulp = _ulp_bf16(ref)
    coarse = ulp >= (GELU_GRAD_SLACK if grad else GELU_SLACK)   # the stored result's rounding dominates the bar
    ulps = torch.where(coarse, err / ulp, 0.0)
    absf = torch.where(coarse, 0.0, err)
    iu, ia, ib = int(ulps.argmax()), int(absf.argmax()), int((err / bar).argmax())
    slack = GELU_GRAD_SLACK if grad else GELU_SLACK
    print(f"\n{name}: worst {ulps[iu].item():.2f} bf16 ulp at x = {x[iu].item()} (where 1 ulp >= {slack:.3g}); worst "
          f"{absf[ia].item():.3g} absolute at x = {x[ia].item()} (elsewhere); worst {(err / bar)[ib].item():.2f} of "
          f"the bar at x = {x[ib].item()}; {int((err > bar).sum())} of {x.numel()} values beyond it")


def test_gelu_epilogue_every_bf16_value():
    """EPI_GELU with A = 0 and bias = every bf16 value in [-10, 10]: z is exactly the sweep value, and gelu(z) is
    within 1 bf16 ulp + 2^-15 of float64 z Phi(z)."""
    from painter_b200 import ops
    x = _bf16_sweep(-10.0, 10.0)
    n = x.numel()
    N = -(-n // 64) * 64
    bias = torch.zeros(N, device=DEV)
    bias[:n] = x
    z, hact = ops.gemm(torch.zeros(128, 64, dtype=BF16, device=DEV), torch.zeros(N, 64, dtype=BF16, device=DEV),
                       kind=ops.EPI_GELU, bias=bias)
    _assert_equal(z, bias.bfloat16().expand(128, N), "GELU epilogue: z")
    got = hact[:, :n]
    _report("GELU", got[0], x, grad=False)
    _assert_gelu_within_bar(got, x.expand(128, n), False, "GELU epilogue")


def test_gelu_grad_epilogue_every_bf16_value():
    """EPI_DGELU with acc = 1 exactly and aux = every bf16 value in [-10, 10]: the output is within 1 bf16 ulp +
    2^-13 of float64 Phi(x) + x phi(x)."""
    from painter_b200 import ops
    x = _bf16_sweep(-10.0, 10.0)
    n = x.numel()
    M = 128
    N = -(-(-(-n // M)) // 64) * 64   # ceil(n / M) columns, rounded up to a multiple of 64
    aux = torch.zeros(M * N, dtype=BF16, device=DEV)
    aux[:n] = x.bfloat16()
    a = torch.zeros(M, 64, dtype=BF16, device=DEV)
    b = torch.zeros(N, 64, dtype=BF16, device=DEV)
    a[:, 0] = 1
    b[:, 0] = 1
    got = ops.gemm(a, b, kind=ops.EPI_DGELU, aux=aux.view(M, N)).flatten()[:n]
    _report("GELU'", got, x, grad=True)
    _assert_gelu_within_bar(got, x, True, "GELU' epilogue")
