"""TEST INFRASTRUCTURE: a CPU restatement of the MATLAB scoring of Painter's derain and SIDD evaluations, which this
environment cannot run (no MATLAB).  Written from the two scripts and from MATLAB's documented algorithms, and
unverified against MATLAB itself:

    rgb2ycbcr_y         rgb2ycbcr on uint8 RGB, the Y channel: K1 R + K2 G + K3 B + 16 in fp64 (Ki = (1/255) *
                        [65.481, 128.553, 24.966]_i), summed left to right with no FMA, rounded half away from zero
    fspecial_gaussian   fspecial('gaussian', n, sigma)
    filter2_valid       filter2(h, x, 'valid') (a correlation)
    derain_prediction   the uint8 image painter_inference_derain.py writes: trunc(clip(x, 0, 1) * 255)
    compute_psnr        Painter/eval/derain/evaluate_PSNR_SSIM.m compute_psnr: on the Y channels, peak 255
    ssim_index          its SSIM_index with the default window and constants: on the Y channels
    sidd_psnr           MATLAB psnr(x, y) on single images in [0, 1] (peak 1), accumulated in fp64
    sidd_ssim           MATLAB ssim(x, y) on an H x W x 3 single array: a 3-D volume, Gaussian sigma 1.5 with 11 taps
                        and replicate padding, C1 = 0.01^2, C2 = 0.03^2, the mean of the map (fp64 here)

Used by tests/test_restoration_matlab_host.py, tests/test_gpu_restoration_matlab.py and scripts/task_metrics.py;
nothing in painter_b200/ imports it.
"""
import numpy as np

YCBCR_Y = (65.481, 128.553, 24.966)


def ycbcr_coefficients():
    inv = 1.0 / 255.0
    return tuple(inv * c for c in YCBCR_Y)


def round_half_away(v):
    """Round half away from zero, exactly (np.round rounds half to even; floor(v + 0.5) can round the sum)."""
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(v)
    f = np.floor(a)
    return np.sign(v) * (f + (a - f >= 0.5))


def rgb2ycbcr_y(rgb_u8, offset_first=False):
    """uint8 [..., 3] -> uint8 [...]: the Y channel of MATLAB rgb2ycbcr.  offset_first=True adds the 16 first (the
    alternative summation order; it changes Y for 15 of the 2^24 colours)."""
    rgb = np.asarray(rgb_u8)
    if rgb.dtype != np.uint8 or rgb.shape[-1] != 3:
        raise ValueError("rgb2ycbcr_y expects uint8 [..., 3]")
    k1, k2, k3 = ycbcr_coefficients()
    r, g, b = (rgb[..., i].astype(np.float64) for i in range(3))
    if offset_first:
        v = ((16.0 + k1 * r) + k2 * g) + k3 * b
    else:
        v = ((k1 * r + k2 * g) + k3 * b) + 16.0
    return np.clip(round_half_away(v), 0, 255).astype(np.uint8)


def fspecial_gaussian(n=11, sigma=1.5):
    """fspecial('gaussian', n, sigma): exp(-(x^2 + y^2) / (2 sigma^2)) on the n x n grid centred on 0, values below
    eps * max set to 0, normalised to sum 1."""
    x = np.arange(n, dtype=np.float64) - (n - 1) / 2.0
    xx, yy = np.meshgrid(x, x)
    h = np.exp(-(xx * xx + yy * yy) / (2.0 * sigma * sigma))
    h[h < np.finfo(np.float64).eps * h.max()] = 0
    s = h.sum()
    return h / s if s != 0 else h


def gaussian_taps(n=11, sigma=1.5):
    """The normalised 1-D Gaussian of n taps (imgaussfilt's kernel; fspecial's window is its outer product)."""
    x = np.arange(n, dtype=np.float64) - (n - 1) / 2.0
    g = np.exp(-(x * x) / (2.0 * sigma * sigma))
    return g / g.sum()


def filter2_valid(h, x):
    """filter2(h, x, 'valid'): out[i, j] = sum_{a, b} h[a, b] x[i + a, j + b]."""
    h = np.asarray(h, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    m, n = h.shape
    H, W = x.shape
    out = np.zeros((H - m + 1, W - n + 1))
    for a in range(m):
        for b in range(n):
            out += h[a, b] * x[a:a + H - m + 1, b:b + W - n + 1]
    return out


def derain_prediction(restored):
    """The PNG painter_inference_derain.py writes from run_one_image's output: (clip(x, 0, 1) * 255).astype(uint8)."""
    return (np.clip(np.asarray(restored, dtype=np.float64), 0, 1) * 255).astype(np.uint8)


def compute_psnr(y1, y2):
    """evaluate_PSNR_SSIM.m compute_psnr on two uint8 Y images: 20 log10(255 / rmse).  +Inf for identical images."""
    d = y1.astype(np.int64) - y2.astype(np.int64)
    sse = int(np.sum(d * d))
    rmse = np.sqrt(sse / d.size)
    with np.errstate(divide="ignore"):
        return float(20.0 * np.log10(255.0 / rmse))


def ssim_index(y1, y2):
    """evaluate_PSNR_SSIM.m SSIM_index(img1, img2) with its defaults: an 11 x 11 Gaussian window (sigma 1.5),
    K = (0.01, 0.03), L = 255, 'valid' filtering, the mean of the map.  Images under 11 x 11 are refused (the
    script returns -Inf)."""
    M, N = y1.shape
    if M < 11 or N < 11:
        raise ValueError("SSIM_index needs at least 11 x 11")
    w = fspecial_gaussian(11, 1.5)
    w = w / np.sum(w)
    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
    a, b = y1.astype(np.float64), y2.astype(np.float64)
    mu1, mu2 = filter2_valid(w, a), filter2_valid(w, b)
    mu1_sq, mu2_sq, mu1_mu2 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = filter2_valid(w, a * a) - mu1_sq
    s2 = filter2_valid(w, b * b) - mu2_sq
    s12 = filter2_valid(w, a * b) - mu1_mu2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2))
    return float(np.mean(ssim_map))


def derain_scores(restored, gt_u8):
    """(psnr, ssim) of one image as evaluate_PSNR_SSIM.m scores the PNG the derain script writes."""
    return derain_scores_u8(derain_prediction(restored), gt_u8)


def derain_scores_u8(pred_u8, gt_u8):
    y1, y2 = rgb2ycbcr_y(pred_u8), rgb2ycbcr_y(gt_u8)
    return compute_psnr(y1, y2), ssim_index(y1, y2)


def sidd_inputs(restored, gt_u8):
    """x = single(clip(r, 0, 1)) (Idenoised.mat holds float32), y = im2single(gt) = single(g) / 255 in float32."""
    x = np.clip(np.asarray(restored, dtype=np.float64), 0, 1).astype(np.float32)
    y = np.asarray(gt_u8).astype(np.float32) / np.float32(255)
    return x, y


def sidd_psnr(x, y):
    """MATLAB psnr(x, y) for floating images: 10 log10(1 / mean((x - y)^2)), in fp64."""
    d = x.astype(np.float64) - y.astype(np.float64)
    with np.errstate(divide="ignore"):
        return float(10.0 * np.log10(1.0 / np.mean(d * d)))


def _replicate_filter(v, taps, axis):
    """'same' correlation along one axis with replicate padding."""
    r = len(taps) // 2
    n = v.shape[axis]
    out = np.zeros_like(v)
    for k, t in enumerate(taps):
        idx = np.clip(np.arange(n) + k - r, 0, n - 1)
        out += t * np.take(v, idx, axis=axis)
    return out


def gauss3(v, taps):
    """imgaussfilt3(v, 1.5) on H x W x D: the separable Gaussian along rows, columns and depth, replicate padding."""
    for axis in range(3):
        v = _replicate_filter(v, taps, axis)
    return v


def depth_mix_matrix(taps, depth=3):
    """The depth pass of gauss3 on D = depth planes, as a D x D matrix: M[c, d] = sum of the taps whose replicate-
    clamped source plane is d."""
    r = len(taps) // 2
    M = np.zeros((depth, depth))
    for c in range(depth):
        for k, t in enumerate(taps):
            M[c, min(max(c + k - r, 0), depth - 1)] += t
    return M


def sidd_ssim(x, y):
    """MATLAB ssim(x, y) on H x W x 3 arrays (a volume): mean of the SSIM map with C1 = 0.01^2, C2 = 0.03^2."""
    taps = gaussian_taps(11, 1.5)
    a, b = x.astype(np.float64), y.astype(np.float64)
    mux, muy = gauss3(a, taps), gauss3(b, taps)
    mux2, muy2, muxy = mux * mux, muy * muy, mux * muy
    sx = gauss3(a * a, taps) - mux2
    sy = gauss3(b * b, taps) - muy2
    sxy = gauss3(a * b, taps) - muxy
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    m = ((2 * muxy + C1) * (2 * sxy + C2)) / ((mux2 + muy2 + C1) * (sx + sy + C2))
    return float(np.mean(m))


def sidd_scores(restored, gt_u8):
    """(psnr, ssim) of one block as eval_sidd.m scores the Idenoised.mat painter_inference_sidd.py saves."""
    x, y = sidd_inputs(restored, gt_u8)
    return sidd_psnr(x, y), sidd_ssim(x, y)
