"""Host-side checks of the derain / SIDD scoring (no GPU): the CPU restatement of MATLAB's rgb2ycbcr, fspecial,
filter2 and ssim in oracle/matlab_ref.py against closed forms and brute force, the exact ties of the luma, the refusal
of bad inputs before any device work, and ptxas's report on the kernels."""
import os
import re
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest
from scipy import ndimage, signal

from oracle import matlab_ref as mr
from painter_b200 import build, task_metrics as tm


def _all_colours():
    c = np.arange(1 << 24, dtype=np.int64)
    return np.stack([c >> 16, (c >> 8) & 255, c & 255], -1)


def test_luma_anchors():
    rgb = np.array([[0, 0, 0], [255, 255, 255], [255, 0, 0], [0, 255, 0], [0, 0, 255]], np.uint8)
    np.testing.assert_array_equal(mr.rgb2ycbcr_y(rgb), [16, 235, 81, 145, 41])


def test_luma_is_the_rounded_rational_value_except_at_ties():
    rgb = _all_colours()
    # 255 * 1000 * (Y - 16) = 65481 R + 128553 G + 24966 B: the rational value of Y is N / 255000
    N = rgb @ np.array([65481, 128553, 24966], np.int64) + 16 * 255000
    rem = N % 255000
    tie = rem == 127500
    y = mr.rgb2ycbcr_y(rgb.astype(np.uint8)).astype(np.int64)
    rounded = N // 255000 + (rem > 127500)
    np.testing.assert_array_equal(y[~tie], rounded[~tie])
    assert np.all((y[tie] == N[tie] // 255000) | (y[tie] == N[tie] // 255000 + 1))


def test_the_194_exact_ties():
    rgb = _all_colours()
    N = rgb @ np.array([65481, 128553, 24966], np.int64) + 16 * 255000
    ties = rgb[N % 255000 == 127500]
    assert len(ties) == 194
    k = [Fraction(c).limit_denominator(1000) / 255 for c in mr.YCBCR_Y]
    inv = 1.0 / 255.0
    kf = [inv * c for c in mr.YCBCR_Y]
    ours = mr.rgb2ycbcr_y(ties.astype(np.uint8))
    for (r, g, b), y in zip(ties.tolist(), ours.tolist()):
        exact = k[0] * r + k[1] * g + k[2] * b + 16
        assert exact.denominator == 2                                   # k + 1/2
        v = ((kf[0] * r + kf[1] * g) + kf[2] * b) + 16.0                # the pinned order, scalar fp64
        assert y == (int(v) + 1 if v - int(v) >= 0.5 else int(v)), (r, g, b)
        assert y in (exact.numerator // 2, exact.numerator // 2 + 1)
    # The one point only MATLAB can settle: adding the offset first changes Y for 15 of these colours, and no other.
    alt = mr.rgb2ycbcr_y(ties.astype(np.uint8), offset_first=True)
    assert int(np.sum(alt != ours)) == 15
    rest = _all_colours()[np.arange(1 << 24)[N % 255000 != 127500][::97]].astype(np.uint8)
    np.testing.assert_array_equal(mr.rgb2ycbcr_y(rest, offset_first=True), mr.rgb2ycbcr_y(rest))


def test_fspecial_window():
    w = mr.fspecial_gaussian(11, 1.5)
    x = np.arange(11) - 5.0
    closed = np.exp(-(x[:, None] ** 2 + x[None, :] ** 2) / 4.5)
    np.testing.assert_allclose(w, closed / closed.sum(), rtol=1e-15, atol=0)
    assert abs(w.sum() - 1.0) < 1e-15
    np.testing.assert_allclose(w, np.outer(mr.gaussian_taps(), mr.gaussian_taps()), rtol=1e-14, atol=0)
    # the factor the kernels use
    np.testing.assert_array_equal(tm._gauss_taps(), mr.gaussian_taps())


def test_filter2_valid_is_a_correlation():
    rng = np.random.RandomState(0)
    h = rng.rand(11, 11)
    for shape in [(11, 11), (12, 40), (37, 23)]:
        x = rng.rand(*shape) * 255
        np.testing.assert_allclose(mr.filter2_valid(h, x), signal.correlate2d(x, h, mode="valid"), rtol=1e-13)


def test_depth_matrix():
    M = mr.depth_mix_matrix(mr.gaussian_taps())
    np.testing.assert_allclose(M, [[0.6330, 0.2130, 0.1540], [0.3670, 0.2660, 0.3670], [0.1540, 0.2130, 0.6330]],
                               atol=5e-5)
    np.testing.assert_allclose(M.sum(1), 1.0, rtol=1e-15)
    np.testing.assert_array_equal(tm._depth_matrix(tm._gauss_taps()), M)


def _ssim3_brute(x, y):
    """MATLAB ssim on a volume, brute force: the 11 x 11 x 11 Gaussian as one correlation with replicate padding."""
    g = mr.gaussian_taps()
    k = g[:, None, None] * g[None, :, None] * g[None, None, :]
    f = lambda v: ndimage.correlate(v, k, mode="nearest")
    mux, muy = f(x), f(y)
    sx, sy, sxy = f(x * x) - mux * mux, f(y * y) - muy * muy, f(x * y) - mux * muy
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return np.mean(((2 * mux * muy + C1) * (2 * sxy + C2)) / ((mux * mux + muy * muy + C1) * (sx + sy + C2)))


@pytest.mark.parametrize("shape", [(1, 1, 3), (5, 7, 3), (13, 16, 3), (24, 19, 3)])
def test_sidd_mixing_shortcut_equals_the_brute_force_volume(shape):
    rng = np.random.RandomState(sum(shape))
    y = rng.rand(*shape)
    x = np.clip(y + 0.1 * rng.randn(*shape), 0, 1)
    assert abs(mr.sidd_ssim(x, y) - _ssim3_brute(x, y)) < 1e-13
    # and the same 3-D filter by planes: the separable 2-D pass, then the 3 x 3 matrix
    g = mr.gaussian_taps()
    two_d = mr._replicate_filter(mr._replicate_filter(x, g, 0), g, 1)
    mixed = np.einsum("cd,hwd->hwc", mr.depth_mix_matrix(g), two_d)
    np.testing.assert_allclose(mixed, mr.gauss3(x, g), rtol=0, atol=1e-15)


def test_identical_images():
    rng = np.random.RandomState(1)
    g = rng.randint(0, 256, size=(20, 31, 3)).astype(np.uint8)
    p, s = mr.derain_scores_u8(g, g)
    assert p == np.inf and s == pytest.approx(1.0, abs=1e-15)
    p, s = mr.sidd_scores(g.astype(np.float32) / np.float32(255), g)
    assert p == np.inf and s == pytest.approx(1.0, abs=1e-15)


def test_derain_prediction_truncates():
    x = np.array([[[-0.5, 0.0, 1.0], [1.5, 0.999, 0.5]]])
    np.testing.assert_array_equal(mr.derain_prediction(x), [[[0, 0, 255], [255, 254, 127]]])


def test_derain_psnr_closed_form():
    a = np.full((11, 12), 100, np.uint8)
    b = a.copy()
    b[0, 0] = 110
    assert mr.compute_psnr(a, b) == pytest.approx(20 * np.log10(255 / np.sqrt(100 / 132)), rel=1e-15)


@pytest.fixture
def no_device(monkeypatch):
    """Any upload or library call fails the test: the inputs must be refused before."""
    def fail(*_a, **_k):
        raise AssertionError("device work before validation")
    monkeypatch.setattr(tm._se, "upload", fail)
    monkeypatch.setattr(tm, "lib", fail)


@pytest.mark.parametrize("fn", [tm.derain_scores, tm.sidd_scores])
def test_bad_inputs_are_refused(no_device, fn):
    x, g = np.zeros((12, 13, 3)), np.zeros((12, 13, 3), np.uint8)
    with pytest.raises(ValueError):
        fn([], [])
    with pytest.raises(ValueError):
        fn([x, x], [g])
    with pytest.raises(ValueError, match="disagree"):
        fn([x], [np.zeros((12, 14, 3), np.uint8)])
    with pytest.raises(ValueError, match="float64"):
        fn([x.astype(np.float32)], [g])
    with pytest.raises(ValueError, match="uint8"):
        fn([x], [g.astype(np.uint16)])
    with pytest.raises(ValueError, match="disagree"):
        fn([np.zeros((12, 13))], [np.zeros((12, 13), np.uint8)])            # not RGB
    with pytest.raises(ValueError, match="disagree"):
        fn([np.zeros((12, 13, 4))], [np.zeros((12, 13, 4), np.uint8)])
    with pytest.raises(ValueError, match="CUDA"):
        fn([x], [g], device="cpu")
    with pytest.raises(ValueError, match="65535"):
        fn([np.zeros((11, 11, 3))] * 65536, [np.zeros((11, 11, 3), np.uint8)] * 65536)


def test_derain_small_images_are_refused(no_device):
    for h, w in [(10, 11), (11, 10), (1, 1)]:
        with pytest.raises(ValueError, match="11 x 11"):
            tm.derain_scores([np.zeros((12, 12, 3)), np.zeros((h, w, 3))],
                             [np.zeros((12, 12, 3), np.uint8), np.zeros((h, w, 3), np.uint8)])


def test_ycbcr_y_refuses_host_and_bad_tensors(no_device):
    import torch
    for bad in [np.zeros((4, 4, 3), np.uint8), torch.zeros((4, 4, 3), dtype=torch.uint8),
                torch.zeros((4, 4), dtype=torch.uint8)]:
        with pytest.raises(ValueError):
            tm.ycbcr_y(bad)


def test_kernels_do_not_spill():
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    if not nvcc:
        pytest.skip("nvcc (CUDA toolkit) not found")
    r = subprocess.run([nvcc, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "restoration_matlab.cu"),
                        "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    report, name = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(_ZN2pk[^']*)'", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            report[name] = tuple(int(g) for g in m.groups())
            name = None
    # luma, derain scores, SIDD scores
    assert len(report) == 3, report
    assert all(v == (0, 0, 0) for v in report.values()), report
