"""COCO panoptic post-processing on the GPU (kernels in csrc/panoptic.cu): the steps Painter/eval/coco_panoptic/eval.sh
runs on the painted instance and semantic images, computed from painter_inference.run_batch's device outputs without
writing or reading PNG files.

    instance_palette     define_colors_per_location_r_gb (COCOCAInstSegEvaluatorCustom.py): the 6400 location colours
    decode_instances     COCOEvaluatorCustom.post_process_segm_output_by_threshold (candidate masks per colour and
                         threshold, maskness, top 2000, util/matrix_nms.mask_matrix_nms, top 100) and
                         post_process_segm_output_by_minmax
    classify_instances   COCOInstanceEvaluatorCustom.merge_inst_semseg_result (COCOInstSegEvaluatorCustom.py,
                         dist_type 'abs'): the class vote over the semantic prediction, and with_nms its class-aware
                         matrix NMS
    panoptic_merge       combine_semantic_and_instance_outputs_custom (COCOPanoEvaluatorCustom.py)

Every call validates its host-side inputs (ValueError) before any device work.  Per batch the number of launches does
not depend on how many images or candidates it holds; the only device-to-host copies are decode_instances' instance
counts (which size the returned masks) and panoptic_merge's segments.  Masks, areas, intersection counts and the
panoptic maps are exact; scores are the reference's fp32 expressions on exact sums.  Results are bitwise reproducible.
"""
import ctypes

import numpy as np
import torch

from . import seggpt_engine as _se
from ._lib import check, lib
from .seggpt_engine import _stream
from .task_metrics import _check_palette

MAX_THRESHOLDS = 4                     # include/painter_b200.h PK_PANO_MAX_THR
PRE_NMS_TOPK = 2000                    # the reference's first sort keeps 2000 candidates
NMS_MAX_NUM = 100                      # mask_matrix_nms(max_num=100)
NMS_SIGMA = 2.0
VOTE_CLASSES = 80                      # the vote reads the first 80 (thing) colours of the semantic palette
POST_TYPES = ("threshold", "minmax")
_FIELDS = 4                            # PK_PANO_FIELDS


def instance_palette():
    """uint8 [6400, 3]: the location colours of define_colors_per_location_r_gb() in its dict order.  The 16 global
    cells step R down from 255 by 255 // 16; the 20 x 20 local cells step G (rows) and B (columns) down from 255 by
    256 // 20 + 1."""
    r = 255 - np.arange(16) * (255 // 16)
    gb = 255 - np.arange(20) * (256 // 20 + 1)
    R, G, B = np.meshgrid(r, gb, gb, indexing="ij")     # global cell, then local row, then local column
    return np.stack([R, G, B], axis=-1).reshape(-1, 3).astype(np.uint8)


class Instances:
    """The instances of one image: masks (device bool [n, H, W]), scores (fp32 [n]), classes (int64 [n]) and
    image_size (H, W), the fields of the reference's detectron2 Instances (pred_masks, scores, pred_classes)."""

    def __init__(self, image_size, masks, scores, classes):
        self.image_size = tuple(int(v) for v in image_size)
        self.masks, self.scores, self.classes = masks, scores, classes

    def __len__(self):
        return int(self.masks.shape[0])

    def __repr__(self):
        return f"Instances(n={len(self)}, image_size={self.image_size})"


def _device_of(device):
    d = torch.device(device)
    if d.type != "cuda":
        raise ValueError(f"panoptic post-processing runs on a CUDA device, got {d}")
    if d.index is None:
        d = torch.device("cuda", torch.cuda.current_device())
    return d


def _pad16(n):
    return (n + 15) // 16 * 16


def _images(preds, device, what, sizes=None):
    """Validate uint8 [H, W, 3] images (device tensors read in place, or host arrays staged in the upload).  Returns
    (table rows int64 [n, 4], staged arrays with their offsets relative to the table's upload, sizes)."""
    n = len(preds)
    if n < 1 or n > 65535:
        raise ValueError(f"{what}: {n} images (1 .. 65535)")
    rows = np.zeros((n, _FIELDS), dtype=np.int64)
    staged, out_sizes = [], []
    for i, p in enumerate(preds):
        if torch.is_tensor(p) and p.is_cuda:
            if p.dtype != torch.uint8 or not p.is_contiguous() or p.device != device:
                raise ValueError(f"{what}: image {i} must be a contiguous uint8 tensor on {device}, got {p.dtype} on "
                                 f"{p.device}")
            shape = tuple(p.shape)
        else:
            p = p.numpy() if torch.is_tensor(p) else np.asarray(p)
            if p.dtype != np.uint8:
                raise ValueError(f"{what}: image {i} must be uint8, got {p.dtype}")
            shape = p.shape
        if len(shape) != 3 or shape[2] != 3 or min(shape[:2]) < 1:
            raise ValueError(f"{what}: image {i} must be [H, W, 3], got {tuple(shape)}")
        if sizes is not None and tuple(shape[:2]) != tuple(sizes[i]):
            raise ValueError(f"{what}: image {i} is {tuple(shape[:2])}, its instances are {tuple(sizes[i])}")
        rows[i, 2:] = shape[:2]
        if torch.is_tensor(p):
            rows[i, 0], rows[i, 1] = p.data_ptr(), 0
        else:
            rows[i, 1] = 1
            staged.append((i, np.ascontiguousarray(p)))
        out_sizes.append(tuple(int(v) for v in shape[:2]))
    return rows, staged, out_sizes


def _upload(device, tables, staged=(), extra=()):
    """One transfer: the tables, then the staged images (their table rows get byte offsets from the first table's
    start), then the extra arrays.  Returns the device views of the tables and extras."""
    arrays, offs, end = [], [], 0

    def add(a):
        nonlocal end
        arrays.append(a)
        offs.append(end)
        end += _pad16(a.nbytes)
        return offs[-1]

    for t in tables:
        add(t)
    for rows, items in staged:
        for i, a in items:
            rows[i, 0] = add(a)
    for e in extra:
        add(e)
    views = _se.upload(arrays, device)
    base = views[0].data_ptr()
    assert [v.data_ptr() - base for v in views] == offs, "upload layout"
    return views[:len(tables)], views[len(arrays) - len(extra):]


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def _words(max_pix):
    return (max_pix + 1023) // 1024 * 32


def _round128(n):
    return max(128, (n + 127) // 128 * 128)


def _thresholds(dist_thr):
    thr = list(dist_thr) if isinstance(dist_thr, (list, tuple)) else [dist_thr]
    if not 1 <= len(thr) <= MAX_THRESHOLDS:
        raise ValueError(f"dist_thr: 1 .. {MAX_THRESHOLDS} thresholds, got {len(thr)}")
    out = []
    for t in thr:
        if isinstance(t, bool) or not isinstance(t, (int, float, np.integer, np.floating)) or not np.isfinite(t) \
                or not t > 0:
            raise ValueError(f"dist_thr must hold positive finite numbers, got {t!r}")
        out.append(float(t))
    return out


def _bounds(thresholds):
    """The mask dist < thr, with dist = fp32(L1) * fp32(1/3) as torch computes `fp32 / 3.` on the device (L1 = 0..765),
    is L1 < bound: the count of L1 values whose dist is below fp32(thr)."""
    d = np.arange(766, dtype=np.float32) * np.float32(1.0 / 3.0)
    b = np.zeros(MAX_THRESHOLDS, dtype=np.int32)
    for i, t in enumerate(thresholds):
        b[i] = np.count_nonzero(d < np.float32(t))
    return b


def _instances_out(dev, sizes, counts, fill):
    """Allocate every image's bool [n_i, H, W] masks in one buffer and run `fill(table, max_rows, max_pix)`."""
    npix = [h * w for h, w in sizes]
    flat = torch.empty(sum(c * p for c, p in zip(counts, npix)), dtype=torch.bool, device=dev)
    table = np.zeros((len(sizes), _FIELDS), dtype=np.int64)
    masks, off = [], 0
    for i, ((h, w), c) in enumerate(zip(sizes, counts)):
        m = flat[off:off + c * h * w].view(c, h, w)
        table[i] = (flat.data_ptr() + off, c, h, w)
        masks.append(m)
        off += c * h * w
    if max(counts) > 0:
        (tab,), _ = _upload(dev, [table])
        fill(tab, max(counts), max(npix))
    return masks


def decode_instances(preds, dist_thr=19.0, post_type="threshold", topk=100, keep_all=False, device="cuda",
                     _timer=None):
    """The instances painted in each uint8 [H, W, 3] image (device tensors, as run_batch(task="nearest") returns them,
    or host arrays), as post_process_segm_output_by_threshold(pred, dist_thr_list, keep_all) computes them with the
    6400 location colours; with post_type="minmax", as post_process_segm_output_by_minmax.  Returns one Instances per
    image, in descending score order for "threshold" (top min(topk, 100) after matrix NMS; every kept candidate, up to
    2000, with keep_all) and in colour order for "minmax".  An image without a candidate gives one empty mask with
    score 0 and class 0, as the reference does."""
    if post_type not in POST_TYPES:
        raise ValueError(f"post_type must be one of {POST_TYPES}, got {post_type!r}")
    thr = _thresholds(dist_thr)
    if isinstance(topk, bool) or not isinstance(topk, (int, np.integer)) or topk < 1:
        raise ValueError(f"topk must be a positive integer, got {topk!r}")
    dev = _device_of(device)
    rows, staged, sizes = _images(preds, dev, "decode_instances")
    pal = instance_palette()
    P = pal.shape[0]
    n = len(sizes)
    max_pix = max(h * w for h, w in sizes)
    tick = _timer or (lambda name: None)
    tick("upload")
    (tab,), (pal_d,) = _upload(dev, [rows], [(rows, staged)], extra=[pal])
    st = _stream()
    L = lib()
    if post_type == "minmax":
        pred = torch.empty((n, max_pix), dtype=torch.int16, device=dev)
        cs = torch.zeros((2, n, P + 1), dtype=torch.int64, device=dev)     # counts (int32 view) and sums
        cnt = cs[0].view(torch.int32)[:, :P + 1]
        cols = torch.empty((n, P + 1), dtype=torch.int32, device=dev)
        scores = torch.empty((n, P + 1), dtype=torch.float32, device=dev)
        classes = torch.empty((n, P + 1), dtype=torch.int64, device=dev)
        count = torch.empty(n, dtype=torch.int32, device=dev)
        tick("candidates")
        check(L.pk_pano_minmax(_ptr(tab), _ptr(tab), n, ctypes.c_longlong(max_pix), _ptr(pal_d), P, _ptr(pred),
                               _ptr(cnt), _ptr(cs[1]), _ptr(cols), _ptr(scores), _ptr(classes), _ptr(count), st),
              "pk_pano_minmax")
        tick("masks")
        counts = count.cpu().tolist()
        masks = _instances_out(dev, sizes, counts, lambda t, mr, mp: check(L.pk_pano_minmax_masks(
            _ptr(pred), n, ctypes.c_longlong(max_pix), _ptr(cols), P + 1, mr, _ptr(t), st), "pk_pano_minmax_masks"))
        tick("end")
        return [Instances(s, m, scores[i, :c], classes[i, :c]) for i, (s, m, c) in
                enumerate(zip(sizes, masks, counts))]

    T = len(thr)
    bounds = _bounds(thr)
    NC = T * P
    ncap = _round128(PRE_NMS_TOPK)
    words = _words(max_pix)
    b_ptr = bounds.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    area = torch.zeros((n, T, P), dtype=torch.int32, device=dev)
    sumfx = torch.zeros((n, T, P), dtype=torch.int64, device=dev)
    tick("candidates")
    check(L.pk_pano_candidates(_ptr(tab), _ptr(tab), n, ctypes.c_longlong(max_pix), _ptr(pal_d), P, b_ptr, T,
                               _ptr(area), _ptr(sumfx), st), "pk_pano_candidates")
    L.pk_pano_select_ws_bytes.restype = ctypes.c_longlong
    ws_bytes = int(L.pk_pano_select_ws_bytes(n, NC))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    count = torch.empty(n, dtype=torch.int32, device=dev)
    cand = torch.empty((n, ncap), dtype=torch.int32, device=dev)
    sel_scores = torch.empty((n, ncap), dtype=torch.float32, device=dev)
    tick("select")
    check(L.pk_pano_select(_ptr(area), _ptr(sumfx), n, NC, PRE_NMS_TOPK, ncap, _ptr(ws), ctypes.c_longlong(ws_bytes),
                           _ptr(count), _ptr(cand), _ptr(sel_scores), st), "pk_pano_select")
    bits = torch.empty((n, ncap, words), dtype=torch.int32, device=dev)
    tick("pack")
    check(L.pk_pano_pack_candidates(_ptr(tab), _ptr(tab), n, _ptr(pal_d), P, b_ptr, T, _ptr(cand), _ptr(count), ncap,
                                    words, _ptr(bits), st), "pk_pano_pack_candidates")
    max_num = ncap if keep_all else min(topk, NMS_MAX_NUM)
    gram = None
    if not keep_all:
        gram = torch.empty((n, ncap, ncap), dtype=torch.int32, device=dev)
        tick("gram")
        check(L.pk_pano_gram(_ptr(bits), n, ncap, words, _ptr(count), _ptr(gram), st), "pk_pano_gram")
    # classes: 1 for every decoded instance, 0 for the empty one
    out_classes = torch.empty((n, max_num), dtype=torch.int64, device=dev)
    out_rows, out_scores, out_count = _nms(gram, None, sel_scores, count, n, ncap, max_num, True, dev, tick,
                                           out_labels=out_classes)
    tick("masks")
    counts = out_count.cpu().tolist()
    masks = _instances_out(dev, sizes, counts, lambda t, mr, mp: check(L.pk_pano_unpack(
        _ptr(bits), n, ncap, words, _ptr(out_rows), max_num, mr, ctypes.c_longlong(mp), _ptr(t), st),
        "pk_pano_unpack"))
    tick("end")
    return [Instances(s, m, out_scores[i, :c], out_classes[i, :c]) for i, (s, m, c) in
            enumerate(zip(sizes, masks, counts))]


def _nms(gram, labels, scores, count, n, ncap, max_num, empty_one, dev, tick, out_labels=None):
    ws = torch.empty(4 * n * ncap, dtype=torch.int32, device=dev)
    rows = torch.empty((n, max_num), dtype=torch.int32, device=dev)
    out_scores = torch.empty((n, max_num), dtype=torch.float32, device=dev)
    out_count = torch.empty(n, dtype=torch.int32, device=dev)
    tick("nms")
    check(lib().pk_pano_nms(_ptr(gram) if gram is not None else None, _ptr(labels) if labels is not None else None,
                            _ptr(scores), _ptr(count), n, ncap, ctypes.c_float(NMS_SIGMA), max_num, int(empty_one),
                            _ptr(ws), _ptr(rows), _ptr(out_scores), _ptr(out_count),
                            _ptr(out_labels) if out_labels is not None else None, _stream()), "pk_pano_nms")
    return rows, out_scores, out_count


def _check_instances(instances, dev, what):
    if len(instances) < 1 or len(instances) > 65535:
        raise ValueError(f"{what}: {len(instances)} images (1 .. 65535)")
    for i, inst in enumerate(instances):
        m, s, c = inst.masks, inst.scores, inst.classes
        ok = torch.is_tensor(m) and m.is_cuda and m.device == dev and m.dtype == torch.bool and m.dim() == 3 and \
            m.is_contiguous() and tuple(m.shape[1:]) == tuple(inst.image_size) and m.shape[0] >= 1
        ok = ok and torch.is_tensor(s) and s.is_cuda and s.device == dev and s.dtype == torch.float32 and \
            s.is_contiguous() and tuple(s.shape) == (m.shape[0],)
        ok = ok and (c is None or (torch.is_tensor(c) and c.is_cuda and c.device == dev and c.dtype == torch.int64
                                   and c.is_contiguous() and tuple(c.shape) == (m.shape[0],)))
        if not ok:
            raise ValueError(f"{what}: instances {i} must hold contiguous device bool masks [n >= 1, H, W] on {dev}, "
                             f"fp32 scores [n] and int64 classes [n]")


def _sem_palette(palette):
    pal = _check_palette(palette)
    if not VOTE_CLASSES <= pal.shape[0] <= 200:
        raise ValueError(f"semantic palette must be [K, 3] with {VOTE_CLASSES} <= K <= 200, got {pal.shape}")
    return pal


def _pack(instances, dev, with_classes):
    """Bit rows of every image's masks, its scores and classes as [n, ncap] batch arrays (one upload, one launch)."""
    n = len(instances)
    counts = [len(x) for x in instances]
    sizes = [x.image_size for x in instances]
    ncap = _round128(max(counts))
    words = _words(max(h * w for h, w in sizes))
    table = np.zeros((n, _FIELDS), dtype=np.int64)
    aux = np.zeros((n, 2), dtype=np.int64)
    for i, x in enumerate(instances):
        table[i] = (x.masks.data_ptr(), counts[i], sizes[i][0], sizes[i][1])
        aux[i] = (x.scores.data_ptr(), x.classes.data_ptr() if with_classes else 0)
    return table, aux, np.asarray(counts, dtype=np.int32), ncap, words


def _run_pack(tab, aux, count_d, n, max_rows, ncap, words, dev, with_classes):
    bits = torch.empty((n, ncap, words), dtype=torch.int32, device=dev)
    scores = torch.empty((n, ncap), dtype=torch.float32, device=dev)
    classes = torch.empty((n, ncap), dtype=torch.int64, device=dev) if with_classes else None
    check(lib().pk_pano_pack_masks(_ptr(tab), n, max_rows, ncap, words, _ptr(bits), _ptr(aux), _ptr(scores),
                                   _ptr(classes) if classes is not None else None, _stream()), "pk_pano_pack_masks")
    return bits, scores, classes


def classify_instances(instances, semseg_preds, palette, with_nms=False, device="cuda"):
    """merge_inst_semseg_result of COCOInstSegEvaluatorCustom.py with dist_type 'abs': each instance's class is the
    argmax of the vote sum over its pixels of 1 - d / max d over the first 80 semantic colours (d the L1 distance of
    the semantic prediction's pixel to the colour, max d over the image), the first on ties.  semseg_preds: uint8
    [H, W, 3] images (run_batch(task="segm") outputs or host arrays), one per Instances, of its size; palette: the
    [K, 3] semantic palette, 80 <= K <= 200.  with_nms (instances decoded with keep_all=True): then a class-aware
    matrix NMS and the top 100, in descending score order.  Returns new Instances."""
    pal = _sem_palette(palette)
    dev = _device_of(device)
    _check_instances(instances, dev, "classify_instances")
    if len(semseg_preds) != len(instances):
        raise ValueError(f"classify_instances: {len(instances)} instances and {len(semseg_preds)} semantic images")
    sizes = [x.image_size for x in instances]
    rows, staged, _ = _images(semseg_preds, dev, "classify_instances", sizes=sizes)
    table, aux, counts, ncap, words = _pack(instances, dev, False)
    n = len(instances)
    max_pix = max(h * w for h, w in sizes)
    (tab, mtab, auxd), (pal_d, count_d) = _upload(dev, [rows, table, aux], [(rows, staged)], extra=[pal, counts])
    bits, scores, _ = _run_pack(mtab, auxd, count_d, n, int(counts.max()), ncap, words, dev, False)
    dmax = torch.zeros(n, dtype=torch.int32, device=dev)
    classes = torch.empty((n, ncap), dtype=torch.int64, device=dev)
    st = _stream()
    check(lib().pk_pano_vote(_ptr(tab), _ptr(tab), n, ctypes.c_longlong(max_pix), _ptr(pal_d), _ptr(bits), ncap,
                             words, _ptr(count_d), int(counts.max()), _ptr(dmax), _ptr(classes), st), "pk_pano_vote")
    if not with_nms:
        return [Instances(x.image_size, x.masks, x.scores, classes[i, :counts[i]]) for i, x in enumerate(instances)]
    gram = torch.empty((n, ncap, ncap), dtype=torch.int32, device=dev)
    check(lib().pk_pano_gram(_ptr(bits), n, ncap, words, _ptr(count_d), _ptr(gram), st), "pk_pano_gram")
    out_labels = torch.empty((n, NMS_MAX_NUM), dtype=torch.int64, device=dev)
    out_rows, out_scores, _ = _nms(gram, classes, scores, count_d, n, ncap, NMS_MAX_NUM, False, dev,
                                   lambda name: None, out_labels=out_labels)
    kept = [min(int(c), NMS_MAX_NUM) for c in counts]
    masks = _instances_out(dev, sizes, kept, lambda t, mr, mp: check(lib().pk_pano_unpack(
        _ptr(bits), n, ncap, words, _ptr(out_rows), NMS_MAX_NUM, mr, ctypes.c_longlong(mp), _ptr(t), st),
        "pk_pano_unpack"))
    return [Instances(s, m, out_scores[i, :k], out_labels[i, :k]) for i, (s, m, k) in enumerate(zip(sizes, masks, kept))]


def matrix_nms(masks, labels, scores, max_num=NMS_MAX_NUM, sigma=NMS_SIGMA, device="cuda"):
    """util/matrix_nms.mask_matrix_nms(masks, labels, scores, filter_thr=-1, nms_pre=-1, max_num, 'gaussian', sigma)
    for one image: masks device bool [n, H, W], labels int64 [n] or None (class-agnostic), scores fp32 [n].  Returns
    (scores, keep_inds): the decayed scores in stable descending order and the input index of each, top max_num."""
    dev = _device_of(device)
    inst = Instances(tuple(masks.shape[1:]), masks, scores, labels)
    _check_instances([inst], dev, "matrix_nms")
    if isinstance(max_num, bool) or not isinstance(max_num, (int, np.integer)) or max_num < 1:
        raise ValueError(f"max_num must be a positive integer, got {max_num!r}")
    if not (isinstance(sigma, (int, float)) and np.isfinite(sigma)):
        raise ValueError(f"sigma must be a finite number, got {sigma!r}")
    table, aux, counts, ncap, words = _pack([inst], dev, labels is not None)
    (mtab, auxd), (count_d,) = _upload(dev, [table, aux], extra=[counts])
    bits, sc, cl = _run_pack(mtab, auxd, count_d, 1, int(counts[0]), ncap, words, dev, labels is not None)
    gram = torch.empty((1, ncap, ncap), dtype=torch.int32, device=dev)
    st = _stream()
    check(lib().pk_pano_gram(_ptr(bits), 1, ncap, words, _ptr(count_d), _ptr(gram), st), "pk_pano_gram")
    ws = torch.empty(4 * ncap, dtype=torch.int32, device=dev)
    rows = torch.empty((1, max_num), dtype=torch.int32, device=dev)
    out_scores = torch.empty((1, max_num), dtype=torch.float32, device=dev)
    out_count = torch.empty(1, dtype=torch.int32, device=dev)
    check(lib().pk_pano_nms(_ptr(gram), _ptr(cl) if cl is not None else None, _ptr(sc), _ptr(count_d), 1, ncap,
                            ctypes.c_float(sigma), max_num, 0, _ptr(ws), _ptr(rows), _ptr(out_scores),
                            _ptr(out_count), None, st), "pk_pano_nms")
    k = min(int(counts[0]), max_num)
    return out_scores[0, :k], rows[0, :k].to(torch.int64)


def panoptic_merge(instances, semseg_preds, palette, overlap_threshold=0.5, stuff_area_thresh=8192,
                   instances_score_thresh=0.55, device="cuda"):
    """combine_semantic_and_instance_outputs_custom for each image: the instances (classified) in descending score
    order while score >= instances_score_thresh, each claiming its pixels not yet claimed unless more than
    overlap_threshold of it is; then every semantic label >= 80 of the argmin map of semseg_preds (uint8 [H, W, 3],
    palette [K, 3] with 80 <= K <= 200) on the unclaimed pixels, if its area reaches stuff_area_thresh.  Returns
    [(int32 device [H, W] panoptic map, segments_info)], segments_info as the reference's list of dicts."""
    pal = _sem_palette(palette)
    for name, v in (("overlap_threshold", overlap_threshold), ("stuff_area_thresh", stuff_area_thresh),
                    ("instances_score_thresh", instances_score_thresh)):
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or np.isnan(v):
            raise ValueError(f"{name} must be a number, got {v!r}")
    dev = _device_of(device)
    _check_instances(instances, dev, "panoptic_merge")
    if any(x.classes is None for x in instances):
        raise ValueError("panoptic_merge: the instances need classes (classify_instances)")
    if len(semseg_preds) != len(instances):
        raise ValueError(f"panoptic_merge: {len(instances)} instances and {len(semseg_preds)} semantic images")
    sizes = [x.image_size for x in instances]
    rows, staged, _ = _images(semseg_preds, dev, "panoptic_merge", sizes=sizes)
    table, aux, counts, ncap, words = _pack(instances, dev, True)
    L = lib()
    L.pk_pano_merge_smem.restype = ctypes.c_longlong
    if int(L.pk_pano_merge_smem(words, ncap)) > 200 * 1024:
        raise ValueError("panoptic_merge: images or instance counts too large for one CTA's claimed-pixel bitmap")
    n = len(instances)
    npix = [h * w for h, w in sizes]
    max_pix = max(npix)
    flat = torch.zeros(sum(npix), dtype=torch.int32, device=dev)
    maps = np.zeros((n, _FIELDS), dtype=np.int64)
    off = 0
    for i, (h, w) in enumerate(sizes):
        maps[i] = (flat.data_ptr() + 4 * off, 0, h, w)
        off += h * w
    K = pal.shape[0]
    max_seg = ncap + K
    (tab, mtab, auxd, maps_d), (pal_d, count_d) = _upload(dev, [rows, table, aux, maps], [(rows, staged)],
                                                          extra=[pal, counts])
    bits, scores, classes = _run_pack(mtab, auxd, count_d, n, int(counts.max()), ncap, words, dev, True)
    labels = torch.empty((n, max_pix), dtype=torch.uint8, device=dev)
    out = torch.empty(n * max_seg * 4 + (n + 1) // 2, dtype=torch.int64, device=dev)
    nseg = out[n * max_seg * 4:].view(torch.int32)
    check(L.pk_pano_merge(_ptr(tab), _ptr(tab), _ptr(maps_d), n, ctypes.c_longlong(max_pix), _ptr(pal_d), K,
                          _ptr(labels), _ptr(bits), ncap, words, _ptr(scores), _ptr(classes), _ptr(count_d),
                          ctypes.c_double(float(overlap_threshold)), ctypes.c_double(float(stuff_area_thresh)),
                          ctypes.c_double(float(instances_score_thresh)), max_seg, _ptr(out), _ptr(nseg), _stream()),
          "pk_pano_merge")
    host = out.cpu().numpy()
    segs = host[:n * max_seg * 4].reshape(n, max_seg, 4)
    nsg = host[n * max_seg * 4:].view(np.int32)[:n]
    results, off = [], 0
    for i, (h, w) in enumerate(sizes):
        info = []
        for s in range(int(nsg[i])):
            inst, cat, area, bits_ = (int(v) for v in segs[i, s])
            if inst >= 0:
                score = float(np.array([bits_], dtype=np.uint32).view(np.float32)[0])
                info.append({"id": s + 1, "isthing": True, "score": score, "category_id": cat,
                             "instance_id": inst})
            else:
                info.append({"id": s + 1, "isthing": False, "category_id": cat, "area": area})
        results.append((flat[off:off + h * w].view(h, w), info))
        off += h * w
    return results
