"""Task metrics on the GPU: the scores of the Painter evaluators, computed from the outputs of
painter_inference.run_batch without writing or reading PNG files (kernels in csrc/metrics.cu).

    palette_classes     SemSegEvaluatorCustom.post_process_segm_output (Painter/eval/ade20k_semantic/
                        ADE20kSemSegEvaluatorCustom.py, coco_panoptic/COCOPanoSemSegEvaluatorCustom.py)
    SemSegMeter         their confusion matrix (np.bincount) and detectron2 SemSegEvaluator.evaluate's mIoU, fwIoU,
                        mACC, pACC
    DepthMeter          Painter/eval/nyuv2_depth/eval_with_pngs.py as eval/nyuv2_depth/eval.sh runs it
    restoration_scores  the PSNR / SSIM of Painter/eval/lol/painter_inference_lol.py (skimage 0.19)
    derain_scores       the PSNR / SSIM of Painter/eval/derain/evaluate_PSNR_SSIM.m (MATLAB; csrc/restoration_matlab.cu)
    sidd_scores         the PSNR / SSIM of Painter/eval/sidd/eval_sidd.m (MATLAB psnr / ssim)
    ycbcr_y             MATLAB rgb2ycbcr's Y channel of uint8 RGB, as derain_scores computes it

Every update / call validates its host-side inputs on the host (ValueError) before any device work, then makes one
upload (the host arrays and a descriptor table of every image's device address and size) and one launch for the whole
batch, with no device-to-host synchronisation except where a result is returned to the host.  Results are bitwise
reproducible from run to run.
"""
import ctypes

import numpy as np
import torch

from . import seggpt_engine as _se
from ._lib import check, lib
from .seggpt_engine import _stream

DIST_TYPES = {"abs": 0, "square": 1, "mean": 2}       # include/painter_b200.h PK_DIST_*
MAX_CLASSES = 200
DEPTH_COLUMNS = ("d1", "d2", "d3", "AbsRel", "SqRel", "RMSE", "RMSElog", "SILog", "log10")
_FIELDS = 5                                            # PK_METRIC_FIELDS


def _check_palette(palette):
    p = np.asarray(palette)
    if p.ndim != 2 or p.shape[1] != 3 or not 1 <= p.shape[0] <= MAX_CLASSES:
        raise ValueError(f"palette must be [K, 3] with 1 <= K <= {MAX_CLASSES}, got shape {p.shape}")
    if not (np.issubdtype(p.dtype, np.integer) or np.issubdtype(p.dtype, np.floating)):
        raise ValueError(f"palette must hold numbers, got {p.dtype}")
    pf = p.astype(np.float64)
    if not np.all((pf == np.round(pf)) & (pf >= 0) & (pf <= 255)):
        raise ValueError("palette colours must be integers in 0..255")
    return pf.astype(np.uint8)


def _check_dist(dist_type):
    if dist_type not in DIST_TYPES:
        raise ValueError(f"dist_type must be one of {sorted(DIST_TYPES)}, got {dist_type!r}")
    return DIST_TYPES[dist_type]


def _pad16(n):
    return (n + 15) // 16 * 16


def _as_host(a, dtype, what):
    if torch.is_tensor(a):
        a = a.numpy()
    a = np.ascontiguousarray(a)
    if a.dtype != dtype:
        raise ValueError(f"{what} must be {np.dtype(dtype).name}, got {a.dtype}")
    return a


def _batch(preds, gts, pred_dtype, gt_dtype, pred_ndim, gt_ndim, device, what, extra=()):
    """Validate one batch and lay out its upload: the descriptor table first, then every host prediction, ground truth
    and extra array at the 16-byte-aligned offsets seggpt_engine.upload gives them.  Device predictions (CUDA tensors
    on `device`) are read in place.  Returns (the upload function, largest H, largest W); nothing
    touches the device before the upload function is called."""
    n = len(preds)
    if n < 1 or len(gts) != n or n > 65535:
        raise ValueError(f"{what}: {n} predictions and {len(gts)} ground truths (1 .. 65535 images)")
    tdt = {np.uint8: torch.uint8, np.int32: torch.int32, np.float64: torch.float64}[pred_dtype]
    rows = np.zeros((n, _FIELDS), dtype=np.int64)
    arrays, offs, end = [rows], [0], _pad16(rows.nbytes)

    def add(a):
        nonlocal end
        arrays.append(a)
        offs.append(end)
        end += _pad16(a.nbytes)
        return offs[-1]

    max_h = max_w = 0
    for i, (p, g) in enumerate(zip(preds, gts)):
        g = _as_host(g, gt_dtype, f"{what}: ground truth {i}")
        if torch.is_tensor(p) and p.is_cuda:
            if device.index is None:
                device = torch.device("cuda", torch.cuda.current_device())
            if p.dtype != tdt or not p.is_contiguous() or p.device != device:
                raise ValueError(f"{what}: prediction {i} must be a contiguous {tdt} tensor on {device}, got "
                                 f"{p.dtype} on {p.device}")
            shape, addr, staged = tuple(p.shape), p.data_ptr(), 0
        else:
            p = _as_host(p, pred_dtype, f"{what}: prediction {i}")
            shape, addr, staged = p.shape, None, 1
        if len(shape) != pred_ndim or g.ndim != gt_ndim or shape[:2] != g.shape[:2] or \
                (pred_ndim == 3 and shape[2] != 3) or (gt_ndim == 3 and g.shape[2] != 3) or min(shape[:2]) < 1:
            raise ValueError(f"{what}: image {i}: prediction {tuple(shape)} and ground truth {g.shape} disagree")
        if staged:
            addr = add(p)
        rows[i] = (addr, staged, add(g), shape[0], shape[1])
        max_h, max_w = max(max_h, shape[0]), max(max_w, shape[1])
    for e in extra:
        add(e)

    def upload():
        views = _se.upload(arrays, device)
        base = views[0].data_ptr()
        assert [v.data_ptr() - base for v in views] == offs, "upload layout"
        return views

    return upload, max_h, max_w


def _device(device):
    d = torch.device(device)
    if d.type != "cuda":
        raise ValueError(f"task metrics run on a CUDA device, got {d}")
    return d


def palette_classes(segm_u8, palette, dist_type="abs"):
    """segm_u8: device uint8 [H, W, 3] -> device uint8 [H, W]: the index of the nearest palette colour (the first of
    equally near ones), as post_process_segm_output computes it with the same palette and dist_type."""
    pal = _check_palette(palette)
    dist = _check_dist(dist_type)
    if not (torch.is_tensor(segm_u8) and segm_u8.is_cuda and segm_u8.dtype == torch.uint8 and segm_u8.dim() == 3
            and segm_u8.shape[2] == 3 and segm_u8.is_contiguous() and segm_u8.numel() > 0):
        raise ValueError("palette_classes: segm must be a contiguous device uint8 [H, W, 3] tensor")
    pal_d = torch.from_numpy(pal).to(segm_u8.device, non_blocking=True)
    out = torch.empty(segm_u8.shape[:2], dtype=torch.uint8, device=segm_u8.device)
    check(lib().pk_palette_classes(ctypes.c_void_p(segm_u8.data_ptr()), ctypes.c_longlong(out.numel()),
                                   ctypes.c_void_p(pal_d.data_ptr()), pal.shape[0], dist,
                                   ctypes.c_void_p(out.data_ptr()), _stream()), "pk_palette_classes")
    return out


class SemSegMeter:
    """Confusion matrix and scores of the semantic-segmentation evaluators (ADE20K with its 150-colour palette, COCO
    panoptic semseg with its 133-colour one).  The palette is the [K, 3] list the evaluator is given; a ground-truth
    value equal to ignore_label counts as class K, as in the evaluator; any other value >= K is refused."""

    def __init__(self, palette, ignore_label=255, dist_type="abs", device="cuda"):
        self._pal = _check_palette(palette)
        self._dist = _check_dist(dist_type)
        if not (isinstance(ignore_label, (int, np.integer)) and 0 <= ignore_label <= 255):
            raise ValueError(f"ignore_label must be an integer in 0..255 (labels are uint8), got {ignore_label!r}")
        self.num_classes = self._pal.shape[0]
        self.ignore_label = int(ignore_label)
        self.device = _device(device)
        self._pal_d = self._conf = None        # allocated by the first update

    def reset(self):
        if self._conf is not None:
            self._conf.zero_()

    def update(self, preds, gts):
        """preds: uint8 [H, W, 3] images (device tensors, as run_batch(task="segm") returns them, or host arrays);
        gts: uint8 [H, W] label maps on the host.  One upload and one launch."""
        K = self.num_classes
        for i, g in enumerate(gts):
            g = np.asarray(g)
            if g.dtype == np.uint8 and np.any((g >= K) & (g != self.ignore_label)):
                raise ValueError(f"SemSegMeter.update: ground truth {i} has labels >= {K} other than the ignore "
                                 f"label {self.ignore_label}")
        upload, max_h, max_w = _batch(preds, gts, np.uint8, np.uint8, 3, 2, self.device, "SemSegMeter.update")
        views = upload()
        if self._conf is None:
            self._pal_d = torch.from_numpy(self._pal).to(self.device)
            self._conf = torch.zeros((K + 1) ** 2, dtype=torch.int64, device=self.device)
        check(lib().pk_semseg_confusion(ctypes.c_void_p(views[0].data_ptr()), ctypes.c_void_p(views[0].data_ptr()),
                                        len(views[0]), ctypes.c_longlong(max_h * max_w),
                                        ctypes.c_void_p(self._pal_d.data_ptr()), K, self._dist, self.ignore_label,
                                        ctypes.c_void_p(self._conf.data_ptr()), _stream()), "pk_semseg_confusion")

    @property
    def conf_matrix(self):
        """int64 numpy [K+1, K+1]; entry [pred, gt]."""
        K = self.num_classes
        if self._conf is None:
            return np.zeros((K + 1, K + 1), dtype=np.int64)
        return self._conf.cpu().numpy().reshape(K + 1, K + 1)

    def evaluate(self):
        return semseg_scores(self.conf_matrix)


def semseg_scores(conf):
    """detectron2 SemSegEvaluator.evaluate on a [K+1, K+1] confusion matrix (rows: prediction, columns: ground truth,
    last row / column: the ignore label), x 100.  These formulas are restated from detectron2's evaluator, which is not
    a dependency of this project.  IoU / ACC are per class, NaN for classes absent from the ground truth."""
    conf = np.asarray(conf)
    K = conf.shape[0] - 1
    acc = np.full(K, np.nan, dtype=np.float64)
    iou = np.full(K, np.nan, dtype=np.float64)
    tp = conf.diagonal()[:-1].astype(np.float64)
    pos_gt = np.sum(conf[:-1, :-1], axis=0).astype(np.float64)
    class_weights = pos_gt / np.sum(pos_gt)
    pos_pred = np.sum(conf[:-1, :-1], axis=1).astype(np.float64)
    acc_valid = pos_gt > 0
    acc[acc_valid] = tp[acc_valid] / pos_gt[acc_valid]
    union = pos_gt + pos_pred - tp
    iou_valid = np.logical_and(acc_valid, union > 0)
    iou[iou_valid] = tp[iou_valid] / union[iou_valid]
    macc = np.sum(acc[acc_valid]) / np.sum(acc_valid)
    miou = np.sum(iou[iou_valid]) / np.sum(iou_valid)
    fiou = np.sum(iou[iou_valid] * class_weights[iou_valid])
    pacc = np.sum(tp) / np.sum(pos_gt)
    return {"mIoU": 100 * miou, "fwIoU": 100 * fiou, "mACC": 100 * macc, "pACC": 100 * pacc,
            "IoU": 100 * iou, "ACC": 100 * acc}


class DepthMeter:
    """NYUv2 depth errors of eval_with_pngs.py (--dataset nyu --min_depth_eval 1e-3 --max_depth_eval 10 --eigen_crop,
    as eval/nyuv2_depth/eval.sh runs it).  Predictions are depth in units of 1e-3 (the PNG values; run_batch's int32
    maps hold the same values the PNG stores), ground truths the uint16 NYUv2 PNG arrays (units of 1e-3)."""

    def __init__(self, min_depth=1e-3, max_depth=10.0, eigen_crop=True, device="cuda"):
        # the script compares and clamps float32 arrays with these values: as float32
        self.min_depth, self.max_depth = float(np.float32(min_depth)), float(np.float32(max_depth))
        if not self.min_depth < self.max_depth:
            raise ValueError(f"DepthMeter: min_depth {min_depth} must be below max_depth {max_depth}")
        self.eigen_crop = bool(eigen_crop)
        self.device = _device(device)
        self._out = []

    def reset(self):
        self._out = []

    def update(self, preds, gts):
        """preds: int32 [H, W] depth maps (device tensors, as run_batch(task="depth") returns them, or host arrays);
        gts: uint16 [H, W] host arrays.  One upload and one launch."""
        upload, _, _ = _batch(preds, gts, np.int32, np.uint16, 2, 2, self.device, "DepthMeter.update")
        views = upload()
        out = torch.empty((len(views[0]), 9), dtype=torch.float64, device=self.device)
        check(lib().pk_depth_errors(ctypes.c_void_p(views[0].data_ptr()), ctypes.c_void_p(views[0].data_ptr()),
                                    len(views[0]), ctypes.c_float(self.min_depth), ctypes.c_float(self.max_depth),
                                    int(self.eigen_crop), ctypes.c_void_p(out.data_ptr()), _stream()),
              "pk_depth_errors")
        self._out.append(out)

    def per_image(self):
        """float64 [n, 9], columns DEPTH_COLUMNS, one row per image in update order."""
        if not self._out:
            return np.zeros((0, 9))
        return torch.cat(self._out).cpu().numpy()

    def evaluate(self):
        """The means the script prints, under its column names."""
        return dict(zip(DEPTH_COLUMNS, self.per_image().mean(axis=0)))


# skimage 0.19 structural_similarity with data_range=None on float64 images uses the dtype's range, (-1, 1): R = 2
_SSIM_R = 2.0
_SSIM_C1 = (0.01 * _SSIM_R) ** 2
_SSIM_C2 = (0.03 * _SSIM_R) ** 2


def restoration_scores(restored, gts, device="cuda"):
    """Per-image PSNR and SSIM of painter_inference_lol.py: x = clip(restored, 0, 1), y = gt / 255.,
    peak_signal_noise_ratio(x, y) and structural_similarity(x, y, multichannel=True) of skimage 0.19.

    restored: float64 [H, W, 3] arrays (as run_batch(task="restore") returns them, or device tensors); gts: uint8
    [H, W, 3] host arrays; every image at least 7 x 7.  Returns (psnr, ssim), float64 numpy [n] each.

    The skimage semantics are restated here without skimage (not a dependency of this project): PSNR =
    10 log10(1 / mean((x - y)^2)) (data_range 1: x is a float image with minimum >= 0); SSIM per channel with a 7 x 7
    uniform window (scipy reflect border), sample covariance (49 / 48), C1 = (0.01 R)^2, C2 = (0.03 R)^2 with R = 2
    (the float64 dtype range), the mean of the S map without 3 pixels at each border, averaged over the channels."""
    dev = _device(device)
    n = len(restored)
    for i, g in enumerate(gts):
        if min(np.shape(g)[:2]) < 7:
            raise ValueError(f"restoration_scores: image {i} is {np.shape(g)[:2]}; SSIM needs at least 7 x 7")
    counters = np.zeros(n, dtype=np.uint32)
    upload, max_h, max_w = _batch(restored, gts, np.float64, np.uint8, 3, 3, dev, "restoration_scores",
                                  extra=(counters,))
    views = upload()
    lib().pk_restoration_ws_doubles.restype = ctypes.c_longlong
    ws = int(lib().pk_restoration_ws_doubles(max_h, max_w))
    partials = torch.empty(n * ws, dtype=torch.float64, device=dev)
    res = torch.empty((2, n), dtype=torch.float64, device=dev)
    check(lib().pk_restoration_scores(ctypes.c_void_p(views[0].data_ptr()), ctypes.c_void_p(views[0].data_ptr()), n,
                                      max_h, max_w, ctypes.c_void_p(views[-1].data_ptr()),
                                      ctypes.c_void_p(partials.data_ptr()), ctypes.c_double(_SSIM_C1),
                                      ctypes.c_double(_SSIM_C2), ctypes.c_void_p(res[0].data_ptr()),
                                      ctypes.c_void_p(res[1].data_ptr()), _stream()), "pk_restoration_scores")
    host = res.cpu().numpy()
    return host[0].copy(), host[1].copy()


# ---------------------------------------------------------------------------------------------------------------------
# The two benchmarks the reference scores in MATLAB.  Restated from the scripts and MATLAB's documented algorithms,
# unverified against MATLAB itself (DESIGN.md, Task metrics).
_GAUSS_TAPS, _GAUSS_SIGMA = 11, 1.5
_DERAIN_C1, _DERAIN_C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2
_SIDD_C1, _SIDD_C2 = 0.01 ** 2, 0.03 ** 2


def _gauss_taps():
    """The normalised 1-D Gaussian of 11 taps, sigma 1.5: imgaussfilt's kernel, and the factor of fspecial('gaussian',
    11, 1.5) (its outer product with itself; the values fspecial zeroes, below eps * max, do not occur here)."""
    x = np.arange(_GAUSS_TAPS, dtype=np.float64) - _GAUSS_TAPS // 2
    g = np.exp(-(x * x) / (2.0 * _GAUSS_SIGMA * _GAUSS_SIGMA))
    return g / g.sum()


def _depth_matrix(taps, depth=3):
    """The depth pass of the separable Gaussian with replicate padding on `depth` planes, as a matrix: M[c, d] = the
    sum of the taps whose clamped source plane is d."""
    r = len(taps) // 2
    M = np.zeros((depth, depth))
    for c in range(depth):
        for k, t in enumerate(taps):
            M[c, min(max(c + k - r, 0), depth - 1)] += t
    return M


def ycbcr_y(img_u8):
    """img_u8: device uint8 [H, W, 3] -> device uint8 [H, W]: the Y channel of MATLAB rgb2ycbcr, K1 R + K2 G + K3 B + 16
    with Ki = (1/255) * (65.481, 128.553, 24.966)_i in fp64, summed left to right, rounded half away from zero."""
    if not (torch.is_tensor(img_u8) and img_u8.is_cuda and img_u8.dtype == torch.uint8 and img_u8.dim() == 3
            and img_u8.shape[2] == 3 and img_u8.is_contiguous() and img_u8.numel() > 0):
        raise ValueError("ycbcr_y: img must be a contiguous device uint8 [H, W, 3] tensor")
    out = torch.empty(img_u8.shape[:2], dtype=torch.uint8, device=img_u8.device)
    check(lib().pk_ycbcr_y(ctypes.c_void_p(img_u8.data_ptr()), ctypes.c_longlong(out.numel()),
                           ctypes.c_void_p(out.data_ptr()), _stream()), "pk_ycbcr_y")
    return out


def _matlab_scores(name, restored, gts, device, consts, c1, c2):
    dev = _device(device)
    n = len(restored)
    counters = np.zeros(n, dtype=np.uint32)
    upload, max_h, max_w = _batch(restored, gts, np.float64, np.uint8, 3, 3, dev, f"{name}_scores",
                                  extra=(consts, counters))
    views = upload()
    ws_fn = getattr(lib(), f"pk_{name}_ws_doubles")
    ws_fn.restype = ctypes.c_longlong
    ws = int(ws_fn(max_h, max_w))
    partials = torch.empty(n * ws, dtype=torch.float64, device=dev)
    res = torch.empty((2, n), dtype=torch.float64, device=dev)
    check(getattr(lib(), f"pk_{name}_scores")(
        ctypes.c_void_p(views[0].data_ptr()), ctypes.c_void_p(views[0].data_ptr()), n, max_h, max_w,
        ctypes.c_void_p(views[-2].data_ptr()), ctypes.c_void_p(views[-1].data_ptr()),
        ctypes.c_void_p(partials.data_ptr()), ctypes.c_double(c1), ctypes.c_double(c2),
        ctypes.c_void_p(res[0].data_ptr()), ctypes.c_void_p(res[1].data_ptr()), _stream()), f"pk_{name}_scores")
    host = res.cpu().numpy()
    return host[0].copy(), host[1].copy()


def derain_scores(restored, gts, device="cuda"):
    """Per-image PSNR and SSIM of Painter/eval/derain/evaluate_PSNR_SSIM.m on the PNGs painter_inference_derain.py
    writes from run_one_image's output.

    restored: float64 [H, W, 3] arrays (as run_batch(task="restore") returns them, or device tensors); gts: the uint8
    [H, W, 3] decoded targets on the host; every image at least 11 x 11.  Returns (psnr, ssim), float64 numpy [n] each.

    Prediction u = uint8(trunc(clip(x, 0, 1) * 255)) in fp64 (the script's PNG); both images go to the Y channel of
    rgb2ycbcr (ycbcr_y).  PSNR = 20 log10(255 / sqrt(mean((Yp - Yg)^2))), the sum of squares exact in int64, +Inf for
    identical images.  SSIM = SSIM_index's defaults: fspecial('gaussian', 11, 1.5) window, 'valid' filtering of Y, Y^2
    and Yp Yg in fp64, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2, the mean of the (H - 10) x (W - 10) map.  The script
    averages per set and then over the five sets; that aggregation is the caller's (INTEGRATION.md)."""
    for i, g in enumerate(gts):
        if len(np.shape(g)) >= 2 and min(np.shape(g)[:2]) < _GAUSS_TAPS:
            raise ValueError(f"derain_scores: image {i} is {np.shape(g)[:2]}; SSIM_index needs at least 11 x 11")
    return _matlab_scores("derain", restored, gts, device, _gauss_taps(), _DERAIN_C1, _DERAIN_C2)


def sidd_scores(restored, gts, device="cuda"):
    """Per-block PSNR and SSIM of Painter/eval/sidd/eval_sidd.m on the Idenoised.mat painter_inference_sidd.py saves.

    restored: float64 [H, W, 3] arrays (as run_batch(task="restore") returns them, or device tensors); gts: uint8
    [H, W, 3] host arrays.  Returns (psnr, ssim), float64 numpy [n] each; eval_sidd.m reports their means.

    x = single(clip(r, 0, 1)) (the .mat holds float32), y = im2single(g) = single(g) / 255.  PSNR =
    10 log10(1 / mean((x - y)^2)) over the 3 H W values (peak 1), in fp64.  SSIM = MATLAB ssim on the H x W x 3 array,
    which it filters as a volume: a separable Gaussian (sigma 1.5, 11 taps) with replicate padding along rows, columns
    and depth ('same' output), C1 = 0.01^2, C2 = 0.03^2, the mean of the map; the depth pass on 3 planes is a 3 x 3
    matrix applied after the 2-D passes.  MATLAB computes in single precision, this in fp64."""
    taps = _gauss_taps()
    consts = np.concatenate([taps, _depth_matrix(taps).reshape(-1)])
    return _matlab_scores("sidd", restored, gts, device, consts, _SIDD_C1, _SIDD_C2)
